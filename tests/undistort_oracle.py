"""ctypes driver for the undistortion restatement (oracle/liboracle_undistort.so, oracle/undistort.mk) and, where it was built, the
reference's own undistorters (oracle/_ref/libref_undistort_pin.so) — TEST INFRASTRUCTURE ONLY. The product package never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
GOLDEN = os.path.join(ROOT, "tests", "golden")
PIN = os.path.join(ORACLE_DIR, "_ref", "pin_undistort")
CAMERAS = ["fov_crop", "radtan_crop", "equidistant_crop", "kb_crop", "pinhole_crop", "fov_calib", "radtan_calib", "pinhole_none"]
c_fp = C.POINTER(C.c_float)
_lib = None


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(ORACLE_DIR, "liboracle_undistort.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(ORACLE_DIR, "undistort.cc")):
            subprocess.check_call(["make", "-C", ORACLE_DIR, "-s", "-f", "undistort.mk"])
        L = C.CDLL(path)
        L.oracle_undistort.restype = C.c_float
        L.oracle_undistort.argtypes = [C.c_int] * 4 + [c_fp] * 4 + [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_float, c_fp,
                                                                     C.POINTER(C.c_ubyte)]
        _lib = L
    return _lib


def _f(a):
    return None if a is None else np.ascontiguousarray(a, np.float32).ctypes.data_as(c_fp)


def undistort(raw, w, h, remapX, remapY, G, vinv, mode, use_exposure, exposure, factor):
    """The restatement of processFrame<T> + undistort<T> (zero past the end of the raw frame). Returns (image h x w, exposure time,
    past-end mask)."""
    raw = np.ascontiguousarray(raw)
    assert raw.dtype in (np.uint8, np.uint16)
    hOrg, wOrg = raw.shape
    keep = [None if a is None else np.ascontiguousarray(a, np.float32) for a in (remapX, remapY, G, vinv)]
    out = np.zeros((h, w), np.float32)
    past = np.zeros((h, w), np.uint8)
    e = lib().oracle_undistort(wOrg, hOrg, w, h, *[_f(a) for a in keep], int(mode), int(use_exposure), raw.ctypes.data_as(C.c_void_p),
                               raw.itemsize, float(exposure), float(factor), out.ctypes.data_as(c_fp),
                               past.ctypes.data_as(C.POINTER(C.c_ubyte)))
    return out, float(e), past


def tables():
    return dict(np.load(os.path.join(GOLDEN, "undistort_tables.npz")))


def camera(name):
    """One camera's fixture: (remapX, remapY or None, None), and per case (settings row, expected image, past-end mask)."""
    z = np.load(os.path.join(GOLDEN, f"undistort_{name}.npz"))
    remap = (z["remapX"], z["remapY"]) if "remapX" in z else (None, None)
    return remap, [(c, z["out_" + c["name"]], z["past_" + c["name"]]) for c in z["cases"]]


def case_inputs(t, c):
    """The raw frame, G and vignetteMapInv a fixture case ran with (G None when the calibration is invalid)."""
    raw = t["raw8"] if c["bpp"] == 1 else t["raw16"]
    g = int(c["g_entries"])
    G = t[f"G{g}"] if g else None          # in mode 0 the reference's G is a linear ramp that processFrame never reads
    vinv = t["vinv8" if g == 256 else "vinv16"] if g else None
    return raw, G, vinv

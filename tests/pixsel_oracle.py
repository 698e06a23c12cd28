"""ctypes driver for the pixel-selection restatement (oracle/liboracle_pixsel.so, oracle/pixsel.mk) and, where it was built, the
reference's own PixelSelector (oracle/_ref/libref_pixsel_pin.so) — TEST INFRASTRUCTURE ONLY. The product package never imports it.

Fixture images are exact float32 renders from a few integers (image()): corners_oracle's value noise, a flat image, or axis-aligned
steps, whose purely horizontal or vertical gradients make a cell's level-0 pick depend on its search direction.
"""
from __future__ import annotations

import ctypes as C
import glob
import os
import subprocess

import numpy as np

from tests import corners_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
GOLDEN = os.path.join(ROOT, "tests", "golden")
PIN_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_pixsel_pin.so")
FAST_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_pixsel.so")
c_fp = C.POINTER(C.c_float)
c_ip = C.POINTER(C.c_int32)
c_bp = C.POINTER(C.c_uint8)
_lib = None
_pin = {}
# makeMaps' settings: (density, recursions_left, th_factor, minGradHistCut, minGradHistAdd, gradDownweightPerLevel, dirDist)
DEFAULT = dict(density=1500.0, recursions_left=1, th_factor=1.0, minGradHistCut=0.5, minGradHistAdd=7.0, gradDownweightPerLevel=0.75,
               selectDirectionDistribution=1)


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(ORACLE_DIR, "liboracle_pixsel.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(ORACLE_DIR, "pixsel.cc")):
            subprocess.check_call(["make", "-C", ORACLE_DIR, "-s", "-f", "pixsel.mk"])
        L = C.CDLL(path)
        L.oracle_pixsel_new.restype = C.c_void_p
        L.oracle_pixsel_new.argtypes = [C.c_int, C.c_int]
        L.oracle_pixsel_free.argtypes = [C.c_void_p]
        L.oracle_pixsel_get_potential.argtypes = [C.c_void_p]
        L.oracle_pixsel_set_potential.argtypes = [C.c_void_p, C.c_int]
        L.oracle_pixsel_pattern.argtypes = [C.c_void_p, c_bp]
        L.oracle_pixsel_set_frame.argtypes = [C.c_void_p, c_fp, c_fp, C.c_float, C.c_float, c_fp, c_fp]
        L.oracle_pixsel_th.restype = C.c_float
        L.oracle_pixsel_th.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.oracle_pixsel_make_maps.argtypes = [C.c_void_p, C.c_float, C.c_int, C.c_float, C.c_float, C.c_int, c_bp, c_ip]
        _lib = L
    return _lib


def pin(path=PIN_LIB):
    """The reference's own PixelSelector behind a C interface (the pin, or with path=FAST_LIB its Release build), or None where no
    reference checkout was built."""
    if path not in _pin and os.path.exists(path):
        L = C.CDLL(path)
        L.cref_pixsel_new.restype = C.c_void_p
        L.cref_pixsel_new.argtypes = [C.c_int, C.c_int]
        L.cref_pixsel_free.argtypes = [C.c_void_p]
        L.cref_pixsel_pattern.argtypes = [C.c_void_p, C.c_int, c_bp]
        L.cref_pixsel_get_potential.argtypes = [C.c_void_p]
        L.cref_pixsel_set_potential.argtypes = [C.c_void_p, C.c_int]
        L.cref_pixsel_make_maps.argtypes = [C.c_void_p, C.c_int, C.c_int, c_fp, c_fp, C.c_float, C.c_int, C.c_float, C.c_float, C.c_float,
                                            C.c_float, C.c_int, c_fp]
        L.cref_pixsel_time.restype = C.c_double
        L.cref_pixsel_time.argtypes = [C.c_int, C.c_int, c_fp, c_fp, C.c_float, C.c_int, C.c_int, c_ip]
        _pin[path] = L
    return _pin.get(path)


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def image(kind, w, h, seed):
    """A fixture image, exact in float32: 'noise' (corners_oracle.render), 'flat' (all 0) or 'steps' (a sum of axis-aligned steps on a
    seeded grid: every gradient away from the step crossings is purely horizontal or vertical)."""
    if kind == "noise":
        return co.render(w, h, seed)
    if kind == "flat":
        return np.zeros((h, w), np.float32)
    assert kind == "steps"
    rng = np.random.default_rng(seed)
    xs = np.cumsum(rng.integers(5, 17, size=w))
    ys = np.cumsum(rng.integers(5, 17, size=h))
    col = np.searchsorted(xs, np.arange(w), side="right") % 2 * rng.integers(10, 60)
    row = np.searchsorted(ys, np.arange(h), side="right") % 2 * rng.integers(10, 60)
    return np.ascontiguousarray(20 + row[:, None] + col[None, :], np.float32)


class Selector:
    """The restatement's PixelSelector(w, h): currentPotential 3 at construction, carried from call to call."""

    def __init__(self, w, h):
        self.w, self.h = w, h
        self.s = lib().oracle_pixsel_new(w, h)

    def __del__(self):
        if getattr(self, "s", None):
            lib().oracle_pixsel_free(self.s)

    @property
    def potential(self):
        return int(lib().oracle_pixsel_get_potential(self.s))

    @potential.setter
    def potential(self, p):
        lib().oracle_pixsel_set_potential(self.s, int(p))

    def pattern(self):
        out = np.zeros(self.w * self.h, np.uint8)
        lib().oracle_pixsel_pattern(self.s, _p(out, c_bp))
        return out

    def set_frame(self, color, B=None, minGradHistCut=0.5, minGradHistAdd=7.0):
        """makeImages + makeHists; returns absSquaredGrad[0..2] and thsSmoothed."""
        color = np.ascontiguousarray(color, np.float32)
        w, h = self.w, self.h
        ag = np.zeros(w * h + (w >> 1) * (h >> 1) + (w >> 2) * (h >> 2), np.float32)
        ths = np.zeros(max((w // 32) * (h // 32), 1), np.float32)
        Bc = None if B is None else np.ascontiguousarray(B, np.float32)
        lib().oracle_pixsel_set_frame(self.s, _p(color, c_fp), _p(Bc, c_fp), minGradHistCut, minGradHistAdd, _p(ag, c_fp), _p(ths, c_fp))
        n0, n1 = w * h, (w >> 1) * (h >> 1)
        return [ag[:n0].reshape(h, w), ag[n0:n0 + n1].reshape(h >> 1, w >> 1), ag[n0 + n1:].reshape(h >> 2, w >> 2)], ths

    def th(self, xf, yf):
        return float(lib().oracle_pixsel_th(self.s, int(xf), int(yf)))

    def make_maps(self, color, B=None, **kw):
        """makeMaps on `color`; returns the uint8 map, n, (n2, n3, n4) of the final pass, and the mixed cells of that pass."""
        p = dict(DEFAULT, **kw)
        self.set_frame(color, B, p["minGradHistCut"], p["minGradHistAdd"])
        mp = np.zeros((self.h, self.w), np.uint8)
        o = np.zeros(4, np.int32)
        n = lib().oracle_pixsel_make_maps(self.s, p["density"], p["recursions_left"], p["th_factor"], p["gradDownweightPerLevel"],
                                          p["selectDirectionDistribution"], _p(mp, c_bp), _p(o, c_ip))
        return mp, int(n), tuple(int(x) for x in o[:3]), int(o[3])


class RefSelector:
    """The reference's own PixelSelector(w, h) through the pin."""

    def __init__(self, w, h, path=PIN_LIB):
        self.L = pin(path)
        self.w, self.h = w, h
        self.s = self.L.cref_pixsel_new(w, h)

    def __del__(self):
        if getattr(self, "s", None):
            self.L.cref_pixsel_free(self.s)

    @property
    def potential(self):
        return int(self.L.cref_pixsel_get_potential(self.s))

    @potential.setter
    def potential(self, p):
        self.L.cref_pixsel_set_potential(self.s, int(p))

    def pattern(self):
        out = np.zeros(self.w * self.h, np.uint8)
        self.L.cref_pixsel_pattern(self.s, out.size, _p(out, c_bp))
        return out

    def make_maps(self, color, B=None, **kw):
        p = dict(DEFAULT, **kw)
        color = np.ascontiguousarray(color, np.float32)
        Bc = None if B is None else np.ascontiguousarray(B, np.float32)
        mp = np.zeros((self.h, self.w), np.float32)
        n = self.L.cref_pixsel_make_maps(self.s, self.w, self.h, _p(color, c_fp), _p(Bc, c_fp), p["density"], p["recursions_left"],
                                         p["th_factor"], p["minGradHistCut"], p["minGradHistAdd"], p["gradDownweightPerLevel"],
                                         p["selectDirectionDistribution"], _p(mp, c_fp))
        return mp, int(n)


def fixtures():
    return sorted(glob.glob(os.path.join(GOLDEN, "pixsel_*.npz")))


def load(path):
    """One fixture: its arrays, its calls' images re-rendered and checked against the stored SHA-256s, and its parameters."""
    z = dict(np.load(path))
    w, h = int(z["w"]), int(z["h"])
    z["images"] = []
    for kind, seed, sha in zip(z["kind"], z["seed"], z["image_sha256"]):
        img = image(str(kind), w, h, int(seed))
        assert co.image_sha(img) == str(sha), f"{path}: the rendered image is not the one the fixture was made from"
        z["images"].append(img)
    z["B"] = None if int(z["has_B"]) == 0 else z["B"]
    z["params"] = {k: (int(z["p_" + k]) if isinstance(v, int) else float(z["p_" + k])) for k, v in DEFAULT.items()}
    return z

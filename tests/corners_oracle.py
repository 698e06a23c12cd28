"""ctypes driver for the corner-detection restatement (oracle/liboracle_corners.so, oracle/corners.mk) and, where it was built, the
reference's own FeatureDetector (oracle/_ref/libref_corners_pin.so) — TEST INFRASTRUCTURE ONLY. The product package never imports it.

The fixture images are rendered here from a few integers (render()): integer value noise on power-of-two lattices, divided by a power of
two, so every pixel is an exact float32 and the same on every machine. The fixtures keep the render parameters and the image's SHA-256
instead of megabytes of pixels.
"""
from __future__ import annotations

import ctypes as C
import glob
import hashlib
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
GOLDEN = os.path.join(ROOT, "tests", "golden")
PIN_LIB = os.path.join(ORACLE_DIR, "_ref", "libref_corners_pin.so")
c_fp = C.POINTER(C.c_float)
c_ip = C.POINTER(C.c_int32)
c_bp = C.POINTER(C.c_uint8)
_lib = None
_pin = None
FIELDS = ("u", "v", "score", "is_corner", "angle", "descriptor")


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(ORACLE_DIR, "liboracle_corners.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(ORACLE_DIR, "corners.cc")):
            subprocess.check_call(["make", "-C", ORACLE_DIR, "-s", "-f", "corners.mk"])
        L = C.CDLL(path)
        L.oracle_corners_capacity.restype = C.c_longlong
        L.oracle_corners_capacity.argtypes = [C.c_int] * 3
        L.oracle_corners_grid.argtypes = [C.c_int] * 3 + [c_ip, c_fp]
        L.oracle_corners_umax.argtypes = [c_ip]
        L.oracle_corners_level0.argtypes = [C.c_int, C.c_int, c_fp, c_fp]
        L.oracle_detect_corners.argtypes = [C.c_int, C.c_int, c_fp, c_fp, C.c_int, c_ip, C.c_int, c_fp, c_fp, c_fp, c_bp, c_fp, c_bp,
                                            c_ip, c_ip]
        L.oracle_corners_suppress.argtypes = [C.c_int, c_fp, c_fp, c_fp, c_bp, c_bp]
        _lib = L
    return _lib


def pin():
    """The reference's own DetectCorners behind a C interface, or None where no reference checkout was built."""
    global _pin
    if _pin is None and os.path.exists(PIN_LIB):
        L = C.CDLL(PIN_LIB)
        L.cref_pattern.argtypes = [c_ip]
        L.cref_level0.argtypes = [C.c_int, C.c_int, c_fp, c_fp, c_fp, c_fp]
        L.cref_detect.argtypes = [C.c_int, C.c_int, c_fp, c_fp, C.c_int, C.c_int, c_fp, c_fp, c_fp, c_bp, c_fp, c_bp, c_ip]
        _pin = L
    return _pin


def _p(a, t):
    return None if a is None else a.ctypes.data_as(t)


def capacity(w, h, n_features):
    return int(lib().oracle_corners_capacity(int(w), int(h), int(n_features)))


def grid(w, h, n_features):
    """(gs, gridX, gridY, skip, ncx, ncy, kcap), nfeatInGrid; None for a refused configuration."""
    o = np.zeros(7, np.int32)
    f = C.c_float(0)
    if lib().oracle_corners_grid(int(w), int(h), int(n_features), _p(o, c_ip), C.byref(f)) != 0:
        return None
    return tuple(int(x) for x in o), f.value


def umax():
    o = np.zeros(16, np.int32)
    lib().oracle_corners_umax(_p(o, c_ip))
    return o


def level0(color):
    """(I, dx, dy) of FrameHessian::makeImages' level 0, h x w x 3."""
    color = np.ascontiguousarray(color, np.float32)
    h, w = color.shape
    img3 = np.zeros((h, w, 3), np.float32)
    lib().oracle_corners_level0(w, h, _p(color, c_fp), _p(img3, c_fp))
    return img3


def _empty(cap):
    return dict(u=np.zeros(cap, np.float32), v=np.zeros(cap, np.float32), score=np.zeros(cap, np.float32),
                is_corner=np.zeros(cap, np.uint8), angle=np.zeros(cap, np.float32), descriptor=np.zeros((cap, 32), np.uint8))


def detect(color, B, n_features, pattern, img3=None):
    """The restatement of DetectCorners on the image `color` (h x w float32) or a given level 0 `img3`. Returns a dict of arrays
    (FIELDS, plus `cell`), and n_corners."""
    color = np.ascontiguousarray(color, np.float32)
    h, w = color.shape
    img3 = level0(color) if img3 is None else np.ascontiguousarray(img3, np.float32)
    cap = capacity(w, h, n_features)
    assert cap >= 0, "refused configuration"
    o = _empty(max(cap, 1))
    cell = np.zeros(max(cap, 1), np.int32)
    n = C.c_int(0)
    Bc = None if B is None else np.ascontiguousarray(B, np.float32)
    pat = np.ascontiguousarray(pattern, np.int32)
    nc = lib().oracle_detect_corners(w, h, _p(img3, c_fp), _p(Bc, c_fp), int(n_features), _p(pat, c_ip), cap, _p(o["u"], c_fp),
                                     _p(o["v"], c_fp), _p(o["score"], c_fp), _p(o["is_corner"], c_bp), _p(o["angle"], c_fp),
                                     _p(o["descriptor"], c_bp), _p(cell, c_ip), C.byref(n))
    assert nc >= 0
    out = {k: a[:n.value] for k, a in o.items()}
    out["cell"] = cell[:n.value]
    return out, nc


def suppress(u, v, score, initial):
    u, v, score = (np.ascontiguousarray(a, np.float32) for a in (u, v, score))
    ini = np.ascontiguousarray(initial, np.uint8)
    out = np.zeros(len(u), np.uint8)
    lib().oracle_corners_suppress(len(u), _p(u, c_fp), _p(v, c_fp), _p(score, c_fp), _p(ini, c_bp), _p(out, c_bp))
    return out


def ref_pattern():
    pat = np.zeros(1024, np.int32)
    pin().cref_pattern(_p(pat, c_ip))
    return pat


def ref_detect(color, B, n_features):
    """The reference's own makeImages + DetectCorners (the pin library). Returns (dict of arrays, n_corners)."""
    color = np.ascontiguousarray(color, np.float32)
    h, w = color.shape
    cap = max(capacity(w, h, n_features), 1)
    o = _empty(cap)
    n = C.c_int(0)
    Bc = None if B is None else np.ascontiguousarray(B, np.float32)
    nc = pin().cref_detect(w, h, _p(color, c_fp), _p(Bc, c_fp), int(n_features), cap, _p(o["u"], c_fp), _p(o["v"], c_fp),
                           _p(o["score"], c_fp), _p(o["is_corner"], c_bp), _p(o["angle"], c_fp), _p(o["descriptor"], c_bp), C.byref(n))
    assert nc >= 0, "the reference returned more features than the capacity"
    return {k: a[:n.value] for k, a in o.items()}, nc


def cell_of(w, h, n_features, u, v):
    (gs, _, _, skip, _, ncy, _), _ = grid(w, h, n_features)
    return ((np.asarray(u).astype(np.int64) // gs - skip) * ncy + (np.asarray(v).astype(np.int64) // gs - skip)).astype(np.int32)


def compare(w, h, n_features, ref, ora):
    """The pin's comparison of the reference's features with the restatement's. Cells whose picks (position and score bits, in order)
    differ are the tie / NaN cells; features closer than 5 pixels to a feature of such a cell may be suppressed differently and are set
    aside with them. On the rest: is_corner, and for corners on both sides the angle and the descriptor."""
    rc, oc = cell_of(w, h, n_features, ref["u"], ref["v"]), ora["cell"]
    cells = np.union1d(rc, oc)
    excluded = []
    for c in cells:
        a = np.stack([ref["u"][rc == c], ref["v"][rc == c], ref["score"][rc == c]])
        b = np.stack([ora["u"][oc == c], ora["v"][oc == c], ora["score"][oc == c]])
        if a.shape != b.shape or a.view(np.uint32).tobytes() != b.view(np.uint32).tobytes():
            excluded.append(int(c))
    excluded = np.array(excluded, np.int32)
    keep_r, keep_o = ~np.isin(rc, excluded), ~np.isin(oc, excluded)
    if len(excluded):
        eu = np.concatenate([ref["u"][~keep_r], ora["u"][~keep_o]])
        ev = np.concatenate([ref["v"][~keep_r], ora["v"][~keep_o]])
        near = lambda U, V: ((U[:, None] - eu[None]) ** 2 + (V[:, None] - ev[None]) ** 2 < 25).any(1)
        keep_r &= ~near(ref["u"], ref["v"])
        keep_o &= ~near(ora["u"], ora["v"])
    R = {k: ref[k][keep_r] for k in FIELDS}
    O = {k: ora[k][keep_o] for k in FIELDS}
    same_list = len(R["u"]) == len(O["u"]) and all(np.array_equal(R[k], O[k]) for k in ("u", "v")) and \
        R["score"].view(np.uint32).tobytes() == O["score"].view(np.uint32).tobytes()
    rep = dict(n_ref=len(ref["u"]), n_ora=len(ora["u"]), excluded_cells=excluded, set_aside=int((~keep_r).sum()), same_list=same_list,
               corner_mismatch=-1, angle_mismatch=-1, angle_max_ulp=-1, descriptor_mismatch=-1, corners=int(R["is_corner"].sum()))
    if same_list:
        both = (R["is_corner"] != 0) & (O["is_corner"] != 0)
        ra, oa = R["angle"][both].view(np.int32).astype(np.int64), O["angle"][both].view(np.int32).astype(np.int64)
        rep.update(corner_mismatch=int((R["is_corner"] != O["is_corner"]).sum()), angle_mismatch=int((ra != oa).sum()),
                   angle_max_ulp=int(np.abs(ra - oa).max()) if len(ra) else 0,
                   descriptor_mismatch=int((R["descriptor"][both] != O["descriptor"][both]).any(1).sum()))
    return rep


# ---------------------------------------------------------------------------------------------------------------- fixture images
def _hash2(x, y, seed):
    h = (x.astype(np.uint64) * np.uint64(0x9E3779B1) + y.astype(np.uint64) * np.uint64(0x85EBCA77) + np.uint64(seed) * np.uint64(0xC2B2AE3D))
    h &= np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(15)
    h = (h * np.uint64(0x2C1B3C6D)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(12)
    h = (h * np.uint64(0x297A2D39)) & np.uint64(0xFFFFFFFF)
    h ^= h >> np.uint64(15)
    return (h & np.uint64(0xFF)).astype(np.int64)


def render(w, h, seed, quantise=0, dots=0):
    """An exact float32 texture: value noise over lattices of 64, 32, 16, 8 and 4 pixels with integer bilinear weights, weighted
    5:4:3:2:2 / 16, divided by 65536 (values in [0, 255], every one exact). quantise=1 rounds down to whole grey levels (flat plateaus);
    dots > 0 then adds that many bright single pixels and 3x3 squares on flat ground, whose symmetric neighbourhoods give equal scores."""
    y, x = np.mgrid[0:h, 0:w].astype(np.int64)
    total = np.zeros((h, w), np.int64)
    for s, amp, o in ((64, 5, 1), (32, 4, 2), (16, 3, 3), (8, 2, 4), (4, 2, 5)):
        gx, gy, fx, fy = x // s, y // s, x % s, y % s
        r00, r10 = _hash2(gx, gy, seed * 8 + o), _hash2(gx + 1, gy, seed * 8 + o)
        r01, r11 = _hash2(gx, gy + 1, seed * 8 + o), _hash2(gx + 1, gy + 1, seed * 8 + o)
        N = r00 * (s - fx) * (s - fy) + r10 * fx * (s - fy) + r01 * (s - fx) * fy + r11 * fx * fy
        total += amp * N * (4096 // (s * s))
    img = (total.astype(np.float64) / 65536.0).astype(np.float32)
    if quantise:
        img = np.floor(img / 16).astype(np.float32) * 16        # coarse plateaus
        rng = np.random.default_rng(seed)
        for _ in range(dots):
            cx, cy, r = int(rng.integers(20, w - 20)), int(rng.integers(20, h - 20)), int(rng.integers(0, 2))
            img[cy - r:cy + r + 1, cx - r:cx + r + 1] += 48
    return np.ascontiguousarray(img, np.float32)


def image_sha(img):
    return hashlib.sha256(np.ascontiguousarray(img, np.float32).tobytes()).hexdigest()


def gamma_B(kind):
    """CalibHessian::B for a fixture: None (identity) or a strictly increasing non-identity response, exact in float."""
    if kind == "identity":
        return None
    i = np.arange(256, dtype=np.float64)
    return (np.round((255.0 * (i / 255.0) ** 0.7) * 64) / 64).astype(np.float32)


def fixtures():
    return sorted(glob.glob(os.path.join(GOLDEN, "corners_*.npz")))


def load(path):
    """One fixture: its arrays, and its image re-rendered and checked against the stored SHA-256."""
    z = dict(np.load(path))
    img = render(int(z["w"]), int(z["h"]), int(z["seed"]), int(z["quantise"]), int(z["dots"]))
    assert image_sha(img) == str(z["image_sha256"]), f"{path}: the rendered image is not the one the fixture was made from"
    z["image"] = img
    z["B"] = None if int(z["has_B"]) == 0 else z["B"]
    return z

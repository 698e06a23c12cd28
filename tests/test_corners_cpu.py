"""The corner-detection restatement (oracle/corners.cc) against the reference's own FeatureDetector (where the pin was built) and the
fixtures, its order rule on a constructed image, its suppression rule against the reference's pairwise loop, the grid checks, and the
C struct of the device entry point. No GPU needed."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from ldso_b200 import capi
from tests import corners_oracle as co
from tests.golden.make_corners_golden import CASES, expand_reference, restatement

ROOT = co.ROOT
FIXTURES = co.fixtures()
needs_pin = pytest.mark.skipif(co.pin() is None, reason="no reference checkout: the pin library was not built")


def _bits_equal(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def test_every_case_has_a_fixture():
    assert sorted(os.path.basename(p) for p in FIXTURES) == sorted(f"corners_{n}.npz" for n in CASES)


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_restatement_matches_fixture(path):
    z = co.load(path)
    got, nc = co.detect(z["image"], z["B"], int(z["n_features"]), z["pattern"])
    want = restatement(z)
    for k in co.FIELDS:
        assert _bits_equal(got[k], want[k].astype(got[k].dtype)), k
    assert nc == int(z["ora_n_corners"])


@needs_pin
@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_restatement_matches_reference(path):
    """Outside the cells whose picks depend on std::sort's handling of equal / NaN scores: the same features in the same order with
    the same score bits, the same corners and descriptors, and angles at most 1 ulp apart (atan2f against atan2 rounded to float)."""
    z = co.load(path)
    w, h, nF = int(z["w"]), int(z["h"]), int(z["n_features"])
    assert _bits_equal(co.ref_pattern(), z["pattern"])
    ref, rnc = co.ref_detect(z["image"], z["B"], nF)
    ora, _ = co.detect(z["image"], z["B"], nF, z["pattern"])
    rep = co.compare(w, h, nF, ref, ora)
    assert rep["same_list"] and rep["corner_mismatch"] == 0 and rep["descriptor_mismatch"] == 0, rep
    assert rep["angle_max_ulp"] <= 1, rep
    assert np.array_equal(rep["excluded_cells"], z["excluded_cells"])
    assert rnc == int(z["ref_n_corners"])
    # the fixture's encoding of the reference's outputs is exact
    exp = expand_reference(z)
    for k in co.FIELDS:
        assert _bits_equal(exp[k], ref[k]), k


@needs_pin
def test_reference_level0_is_the_restatements():
    img = co.render(640, 480, 1)
    B = co.gamma_B("gamma")
    i3, ag = np.zeros((480, 640, 3), np.float32), np.zeros((480, 640), np.float32)
    co.pin().cref_level0(640, 480, img.ctypes.data_as(co.c_fp), B.ctypes.data_as(co.c_fp), i3.ctypes.data_as(co.c_fp), ag.ctypes.data_as(co.c_fp))
    mine = co.level0(img)
    assert _bits_equal(i3[1:-1], mine[1:-1])          # the reference leaves the first and last rows' gradients unset
    assert _bits_equal(i3[:, :, 0], mine[:, :, 0])


def constructed_image():
    """A 640 x 480 level 0 (I, dx, dy) that is zero but for two pairs of gradients in the first cell: A (44,44) = (p, 0) and B (45,44)
    = (0, q) with p, q one ulp apart, whose Shi-Tomasi discriminant rounds below zero (NaN scores), and C (52,52) = (12, 0), D (53,52)
    = (0, 12), whose scores are equal. Both pairs lie in cell (gx, gy) = (3, 3) at 1500 features and in (2, 2) at 800."""
    img3 = np.zeros((480, 640, 3), np.float32)
    img3[44, 44, 1] = np.float32(14.040312)
    img3[44, 45, 2] = np.float32(14.040316)
    img3[52, 52, 1] = 12
    img3[52, 53, 2] = 12
    return img3


@pytest.mark.parametrize("n_features,expect", [(1500, [(52, 52)]), (800, [(52, 52), (53, 52)])])
def test_order_rule_ties_and_nan(n_features, expect):
    img3 = constructed_image()
    color = img3[:, :, 0].copy()
    got, nc = co.detect(color, None, n_features, np.zeros(1024, np.int32), img3=img3)
    assert [(int(u), int(v)) for u, v in zip(got["u"], got["v"])] == expect
    s = got["score"]
    assert np.all(np.isfinite(s)) and np.all(s == s[0])
    # with two picks, the first of the equal pair is suppressed by the later one (p > k && s_p >= s_k), as the reference's loop does
    assert list(got["is_corner"]) == ([1] if n_features == 1500 else [0, 1]) and nc == 1


def nan_image():
    """The NaN pair of constructed_image() alone: the cell's only candidates have NaN scores, so its pick is a NaN."""
    img3 = constructed_image()
    img3[52, 52, 1] = 0
    img3[52, 53, 2] = 0
    return img3


def test_order_rule_nan_pick():
    img3 = nan_image()
    got, nc = co.detect(img3[:, :, 0].copy(), None, 1500, np.zeros(1024, np.int32), img3=img3)
    assert [(int(u), int(v)) for u, v in zip(got["u"], got["v"])] == [(44, 44)]        # the first in push order
    assert got["score"].view(np.uint32)[0] == 0xFFC00000                               # x86's quiet NaN, as the reference stores it
    assert got["is_corner"][0] == 0 and nc == 0


def _reference_loop(u, v, score, initial):
    """FeatureDetector.cc:107-118 as written: every pair of initial corners, the first one loses unless its score is larger."""
    is_c = initial.astype(bool).copy()
    idx = np.flatnonzero(initial)
    for a in range(len(idx)):
        for b in range(a + 1, len(idx)):
            i, j = idx[a], idx[b]
            if np.sqrt(np.float32((u[i] - u[j]) ** 2 + (v[i] - v[j]) ** 2)) < 5:
                if score[i] > score[j]:
                    is_c[j] = False
                else:
                    is_c[i] = False
    return is_c.astype(np.uint8)


@pytest.mark.parametrize("seed", range(6))
def test_suppression_rule_equals_pairwise_loop(seed):
    rng = np.random.default_rng(seed)
    n = 300
    u = rng.integers(0, 40, n).astype(np.float32)
    v = rng.integers(0, 40, n).astype(np.float32)
    score = rng.integers(0, 6, n).astype(np.float32) * np.float32(0.5)       # many equal scores
    initial = (rng.random(n) < 0.8).astype(np.uint8)
    assert np.array_equal(co.suppress(u, v, score, initial), _reference_loop(u, v, score, initial))


def test_grid_and_footprint_checks():
    # the default density at 640 x 480 and the documented cases pass
    for w, h, nF, *_ in CASES.values():
        assert co.capacity(w, h, nF) > 0
    assert co.grid(640, 480, 1500)[0] == (14, 46, 35, 3, 40, 29, 1)
    # 635 x 480 at 317 features: the last cells' patches end exactly on the right and bottom edge; one column less leaves the image
    assert co.capacity(635, 480, 317) > 0 and co.capacity(634, 480, 317) == -1 and co.capacity(635, 479, 317) == -1
    # below about 320 features at 640 x 480 the grid size exceeds 30 and the last cells' patches leave the image
    assert co.capacity(640, 480, 320) > 0 and co.capacity(640, 480, 300) == -1
    for nF in (0, -5, 640 * 480 * 5):
        assert co.capacity(640, 480, nF) == -1
    # the library's host check is the same function of (w, h, nFeatures)
    L = capi.load()
    rng = np.random.default_rng(1)
    cases = [(640, 480, n) for n in (1, 100, 300, 317, 320, 800, 1500, 2000, 4000, 20000, 100000, 307200, 307201, 0, -1)]
    cases += [(int(rng.integers(40, 1400)), int(rng.integers(40, 800)), int(rng.integers(1, 6000))) for _ in range(300)]
    for w, h, nF in cases:
        want = co.capacity(w, h, nF)
        got = L.ldso_b200_feature_capacity(w, h, nF)
        assert got == (want if want >= 0 else -1), (w, h, nF)


def test_umax_table():
    assert list(co.umax()) == [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3]


def test_features_struct_matches_header(tmp_path):
    cls, cname = capi.FeaturesC, "ldso_b200_features"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ldso_b200.h"', 'int main(void) {',
             f'  printf("{cname} %zu\\n", sizeof({cname}));']
    for fname, *_ in cls._fields_:
        lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got[cname]) == C.sizeof(cls)
    for fname, *_ in cls._fields_:
        assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, fname

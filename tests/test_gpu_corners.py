"""Keyframe corners on the device (ldso_b200_detect_corners) against the restatement's fixtures, bit for bit, and against the
reference's own outputs outside the cells whose picks depend on std::sort (angles there differ from glibc's atan2f by at most 1 ulp,
as the restatement's do)."""
from __future__ import annotations

import os

import numpy as np
import pytest

from ldso_b200 import capi
from tests import corners_oracle as co
from tests.golden.make_corners_golden import expand_reference, restatement
from tests import undistort_oracle as uo
from tests.test_corners_cpu import constructed_image, nan_image

pytestmark = pytest.mark.gpu
FIXTURES = co.fixtures()


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _ctx(w, h, pattern=None, levels=3):
    ctx = capi.Context(w, h, levels)
    if pattern is not None:
        ctx.set_orb_pattern(pattern)
    return ctx


def _assert_same(got, want):
    assert len(got["u"]) == len(want["u"])
    for k in co.FIELDS:
        assert _bits(got[k]) == _bits(want[k].astype(got[k].dtype)), k


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_device_matches_restatement_and_reference(path):
    z = co.load(path)
    w, h, nF = int(z["w"]), int(z["h"]), int(z["n_features"])
    ctx = _ctx(w, h, z["pattern"])
    ctx.make_images(2, z["image"])
    got = ctx.detect_corners(2, nF, z["B"])
    want = restatement(z)
    _assert_same(got, want)
    assert got["n_corners"] == int(z["ora_n_corners"])
    # the reference: the same outside the excluded cells (and the features set aside beside them), angles within 1 ulp
    ref = expand_reference(z)
    cells = co.cell_of(w, h, nF, got["u"], got["v"])
    keep = ~np.isin(cells, z["excluded_cells"])
    fix = np.zeros(len(keep), bool)
    fix[z["ref_fix_idx"]] = True
    rcells = co.cell_of(w, h, nF, ref["u"], ref["v"])
    rkeep = ~np.isin(rcells, z["excluded_cells"])
    for k in ("u", "v", "score", "is_corner", "descriptor"):
        assert _bits(got[k][keep & ~fix]) == _bits(ref[k][rkeep][~fix[keep]]), k
    d = got["angle"][keep & ~fix].view(np.int32).astype(np.int64) - ref["angle"][rkeep][~fix[keep]].view(np.int32).astype(np.int64)
    assert np.abs(d).max(initial=0) <= 1
    # repeated calls give the same bits
    again = ctx.detect_corners(2, nF, z["B"])
    for k in co.FIELDS:
        assert _bits(again[k]) == _bits(got[k]), k
    ctx.close()


def test_immature_init_on_detected_features():
    z = co.load(FIXTURES[0])
    w, h, nF = int(z["w"]), int(z["h"]), int(z["n_features"])
    ctx = _ctx(w, h, z["pattern"])
    ctx.make_images(0, z["image"])
    got = ctx.detect_corners(0, nF, z["B"])
    a = ctx.immature_init(0, got["u"], got["v"])
    b = ctx.immature_init(0, z["ora_u"].astype(np.float32), z["ora_v"].astype(np.float32))
    for k in a:
        assert _bits(a[k]) == _bits(b[k]), k
    ctx.close()


@pytest.mark.parametrize("w,h", [(641, 481), (642, 481), (643, 481)])
def test_image_sizes_not_a_multiple_of_four(w, h):
    """w*h odd, 2 mod 4 and 3 mod 4 (the fixtures' sizes are all multiples of 4): bit for bit against the restatement."""
    pat = np.load(FIXTURES[0])["pattern"]
    img = co.render(w, h, 11)
    ctx = _ctx(w, h, pat)
    ctx.make_images(0, img)
    got = ctx.detect_corners(0, 1500)
    want, nc = co.detect(img, None, 1500, pat)
    assert len(want["u"]) > 0
    _assert_same(got, want)
    assert got["n_corners"] == nc
    ctx.close()


def test_from_undistort_frame():
    """A raw 8-bit frame through undistort_frame with a remap table and the undistortion fixtures' 256-entry inverse response
    (photometric mode 1): the corners equal the restatement's on the image the undistortion restatement makes of the same frame."""
    wOrg, hOrg, w, h = 704, 528, 640, 480
    raw = np.clip(co.render(wOrg, hOrg, 3, 1, 300), 0, 255).astype(np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    r2 = ((x - w / 2) / w) ** 2 + ((y - h / 2) / h) ** 2
    remapX = (wOrg / 2 + (x - w / 2) * (1.0 + 0.08 * r2)).astype(np.float32)      # mild barrel distortion, inside the raw frame
    remapY = (hOrg / 2 + (y - h / 2) * (1.0 + 0.08 * r2)).astype(np.float32)
    G = uo.tables()["G256"]
    pat = np.load(FIXTURES[0])["pattern"]
    ctx = _ctx(w, h, pat)
    ctx.set_undistort(wOrg, hOrg, remapX, remapY, G=G, photometric_mode=1)
    ctx.undistort_frame(1, raw, exposure=1.5)
    img, _, _ = uo.undistort(raw, w, h, remapX, remapY, G, None, 1, 1, 1.5, 1.0)
    assert _bits(ctx.download_frame_level(1, 0)[:, :, 0]) == _bits(img)
    got = ctx.detect_corners(1, 1500)
    want, nc = co.detect(img, None, 1500, pat)
    assert len(want["u"]) > 0
    _assert_same(got, want)
    assert got["n_corners"] == nc
    ctx.close()


def test_nan_pick_on_device():
    """A cell whose only candidates have NaN scores: its pick is the first in push order, stored with the reference's NaN bits."""
    img3 = nan_image()
    pat = np.load(FIXTURES[0])["pattern"]
    ctx = _ctx(640, 480, pat, levels=1)
    ctx.upload_frame(0, [img3])
    got = ctx.detect_corners(0, 1500)
    want, nc = co.detect(img3[:, :, 0].copy(), None, 1500, pat, img3=img3)
    _assert_same(got, want)
    assert got["score"].view(np.uint32).tolist() == [0xFFC00000] and got["n_corners"] == nc == 0
    ctx.close()


@pytest.mark.parametrize("n_features", [1500, 800])
def test_order_rule_on_device(n_features):
    img3 = constructed_image()
    pat = np.load(FIXTURES[0])["pattern"]
    ctx = _ctx(640, 480, pat, levels=1)
    ctx.upload_frame(0, [img3])
    got = ctx.detect_corners(0, n_features)
    want, nc = co.detect(img3[:, :, 0].copy(), None, n_features, pat, img3=img3)
    _assert_same(got, want)
    assert got["n_corners"] == nc
    ctx.close()


def test_error_returns():
    pat = np.load(FIXTURES[0])["pattern"]
    ctx = _ctx(640, 480)
    ctx.make_images(0, co.render(640, 480, 1))
    with pytest.raises(capi.Error, match="error -3"):            # no ORB pattern yet
        ctx.detect_corners(0, 1500)
    ctx.set_orb_pattern(pat)
    for slot in (-1, 16, 5):                                      # out of range, and a slot that was never filled
        with pytest.raises(capi.Error, match="error -1"):
            ctx.detect_corners(slot, 1500)
    for nF in (0, -3, 640 * 480 * 5, 300):                        # nFeatures <= 0, gridsize 0, patches leaving the image
        with pytest.raises(capi.Error, match="error -1"):
            ctx.detect_corners(0, nF, capacity=10000)
    cap = capi.feature_capacity(640, 480, 1500)
    with pytest.raises(capi.Error, match="error -1"):
        ctx.detect_corners(0, 1500, capacity=cap - 1)
    with pytest.raises(capi.Error):
        capi.feature_capacity(640, 480, 300)
    with pytest.raises(ValueError):
        ctx.detect_corners(0, 1500, B=np.zeros(10, np.float32))
    with pytest.raises(ValueError):
        ctx.set_orb_pattern(np.zeros(10, np.int32))
    # a missing output array, or no output struct at all
    import ctypes as C
    arr = [np.zeros(cap, np.float32) for _ in range(4)] + [np.zeros(cap, np.uint8), np.zeros(32 * cap, np.uint8)]
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    f = capi.FeaturesC(cap, 0, p(arr[0], C.c_float), p(arr[1], C.c_float), p(arr[2], C.c_float), p(arr[4], C.c_uint8),
                       None, p(arr[5], C.c_uint8), 0)
    assert ctx.L.ldso_b200_detect_corners(ctx.ctx, 0, 1500, None, C.byref(f)) == -1
    assert ctx.L.ldso_b200_detect_corners(ctx.ctx, 0, 1500, None, None) == -1
    # the context still works after the refusals
    assert ctx.detect_corners(0, 1500)["n_corners"] > 0
    ctx.close()

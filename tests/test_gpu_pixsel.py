"""DSO's pixel selection on the device (ldso_b200_select_pixels / make_new_traces_pixels) against the restatement's fixtures, bit
for bit, and the selected pixels' ImmaturePoints against immature_seed. Reads the fixtures only, never the reference."""
from __future__ import annotations

import os

import numpy as np
import pytest

from ldso_b200 import capi
from tests import corners_oracle as co
from tests import pixsel_oracle as po

pytestmark = pytest.mark.gpu
FIXTURES = po.fixtures()
SEG_FIELDS = ("u", "v", "my_type", "color", "weights", "gradH", "energyTH", "idepth_min", "idepth_max", "quality", "status", "uv",
              "interval", "live")


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


def _params(p):
    return capi.pixsel_params(**p)


def _in_range(w, h, mp):
    """makeNewTraces' features of a map (FullSystem.cc:1290-1297): raster order inside [3, w-4) x [3, h-4)."""
    y, x = np.nonzero(mp)
    k = (x >= 3) & (x < w - 4) & (y >= 3) & (y < h - 4)
    return x[k].astype(np.float32), y[k].astype(np.float32), mp[y[k], x[k]].astype(np.float32)


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_select_pixels_matches_fixture(path):
    z = po.load(path)
    w, h = int(z["w"]), int(z["h"])
    ctx = capi.Context(w, h, 3)
    pot = int(z["pot_before"][0])
    for k, img in enumerate(z["images"]):
        ctx.make_images(1, img)
        got = ctx.select_pixels(1, _params(z["params"]), z["B"], current_potential=pot, want_map=True)
        want = z["maps"][k]
        assert np.array_equal(got["map"], want), (path, k, int((got["map"] != want).sum()))
        assert got["n"] == int(z["n"][k]) and (got["n2"], got["n3"], got["n4"]) == tuple(z["counts"][k].tolist())
        assert got["current_potential"] == int(z["pot_after"][k])
        y, x = np.nonzero(want)
        assert np.array_equal(got["x"], x) and np.array_equal(got["y"], y) and np.array_equal(got["type"], want[y, x])
        pot = got["current_potential"]
    # the same call again gives the same bits
    again = ctx.select_pixels(1, _params(z["params"]), z["B"], current_potential=int(z["pot_before"][-1]), want_map=True)
    assert np.array_equal(again["map"], z["maps"][-1])
    ctx.close()


@pytest.mark.parametrize("name", ["d1500_640x480", "d1500_1232x368", "gamma_640x480", "init_640x480", "flat_640x480"])
def test_make_new_traces_pixels_matches_immature_seed(name):
    z = po.load(os.path.join(po.GOLDEN, f"pixsel_{name}.npz"))
    w, h = int(z["w"]), int(z["h"])
    ctx = capi.Context(w, h, 3)
    ctx.make_images(2, z["images"][0])
    ctx.make_images(5, z["images"][0])
    got = ctx.make_new_traces_pixels(2, _params(z["params"]), z["B"], current_potential=int(z["pot_before"][0]))
    assert got["n_selected"] == int(z["n"][0]) and got["current_potential"] == int(z["pot_after"][0])
    u, v, t = _in_range(w, h, z["maps"][0])
    assert _bits(got["u"]) == _bits(u) and _bits(got["v"]) == _bits(v) and _bits(got["my_type"]) == _bits(t)
    ctx.immature_seed(5, u, v, t)
    a, b = ctx.immature_read(2), ctx.immature_read(5)
    for k in SEG_FIELDS:
        assert _bits(a[k]) == _bits(b[k]), k
    ctx.close()


def test_non_finite_energy_is_dropped():
    w, h = 640, 480
    img = co.render(w, h, 31)
    img[3::9, 5::13] = np.nan                          # colours that make some candidates' energyTH NaN
    ctx = capi.Context(w, h, 3)
    ctx.make_images(0, img)
    ctx.make_images(1, img)
    sel = ctx.select_pixels(0)
    mp = np.zeros((h, w), np.uint8)
    mp[sel["y"], sel["x"]] = sel["type"]
    u, v, t = _in_range(w, h, mp)
    ctx.immature_seed(1, u, v, t)
    all_ = ctx.immature_read(1)
    fin = np.isfinite(all_["energyTH"])
    assert (~fin).any() and fin.any()
    got = ctx.make_new_traces_pixels(0)
    assert got["n"] == int(fin.sum()) and got["n_selected"] == sel["n"]
    ctx.immature_seed(1, u[fin], v[fin], t[fin])
    a, b = ctx.immature_read(0), ctx.immature_read(1)
    for k in SEG_FIELDS:
        assert _bits(a[k]) == _bits(b[k]), k
    assert _bits(got["u"]) == _bits(u[fin]) and _bits(got["my_type"]) == _bits(t[fin])
    ctx.close()


def test_growth_keeps_live_segments_and_tracing_matches_trace_immature():
    z = po.load(os.path.join(po.GOLDEN, "pixsel_d12000_640x480.npz"))
    w, h = int(z["w"]), int(z["h"])
    ctx = capi.Context(w, h, 3)
    ctx.make_images(0, z["images"][0])
    ctx.make_images(1, co.render(w, h, 40))
    ctx.make_images(3, np.roll(z["images"][0], 2, axis=1))
    small = ctx.make_new_traces_pixels(1, capi.pixsel_params(density=300.0))
    seg1 = ctx.immature_read(1)
    assert 0 < small["n"] < 1000
    big = ctx.make_new_traces_pixels(0, _params(z["params"]), current_potential=int(z["pot_before"][0]))
    assert big["n"] > 5 * small["n"]                   # the store grew while slot 1's entries were live
    for k, val in ctx.immature_read(1).items():
        assert _bits(val) == _bits(seg1[k]), k
    # one traceNewCoarse pass over slot 0's segment on the frame in slot 3, against trace_immature on the same entries
    s0 = ctx.immature_read(0)
    K = np.array([[500, 0, 320], [0, 500, 240], [0, 0, 1]], np.float64)
    th = 0.004
    R = np.array([[np.cos(th), 0, np.sin(th)], [0, 1, 0], [-np.sin(th), 0, np.cos(th)]])
    KRKi = (K @ R @ np.linalg.inv(K)).astype(np.float32)[None]
    Kt = (K @ np.array([0.05, 0.0, 0.0])).astype(np.float32)[None]
    aff = np.array([[1.0, 0.0]], np.float32)
    pts = dict(u=s0["u"], v=s0["v"], host=np.zeros(len(s0["u"]), np.int32), color=s0["color"], weights=s0["weights"], gradH=s0["gradH"],
               energyTH=s0["energyTH"], idepth_min=s0["idepth_min"].copy(), idepth_max=s0["idepth_max"].copy(), quality=s0["quality"].copy(),
               status=s0["status"].copy(), uv=s0["uv"].copy(), interval=s0["interval"].copy())
    ctx.trace_immature(3, pts, KRKi, Kt, aff)
    c7 = ctx.trace_new_coarse(3, [0], KRKi, Kt, aff, counts=True)
    s = ctx.immature_read(0)
    for k in ("idepth_min", "idepth_max", "quality", "status", "uv", "interval"):
        assert _bits(s[k]) == _bits(pts[k]), k
    assert c7[0] == len(s0["u"])
    ctx.close()


def test_errors():
    w, h = 320, 240
    ctx = capi.Context(w, h, 3)
    ctx.make_images(0, co.render(w, h, 5))
    ctx.make_images(4, co.render(w, h, 6))
    ctx.immature_seed(4, [30.0, 40.0], [30.0, 40.0])
    seg4 = ctx.immature_read(4)
    n = ctx.select_pixels(0)["n"]
    assert n > 0
    for bad in (lambda: ctx.select_pixels(7),                                        # never filled (slots 0 and 4 are)
                lambda: ctx.select_pixels(16),
                lambda: ctx.select_pixels(0, capi.pixsel_params(density=0.0)),
                lambda: ctx.select_pixels(0, capi.pixsel_params(density=-5.0)),
                lambda: ctx.select_pixels(0, current_potential=0),
                lambda: ctx.select_pixels(0, capacity=n - 1),
                lambda: ctx.make_new_traces_pixels(7),
                lambda: ctx.make_new_traces_pixels(0, capi.pixsel_params(density=0.0)),
                lambda: ctx.make_new_traces_pixels(4, current_potential=0),
                lambda: ctx.make_new_traces_pixels(0, capacity=n - 1)):
        with pytest.raises(capi.Error) as e:
            bad()
        assert "error -1" in str(e.value), str(e.value)
    for k, val in ctx.immature_read(4).items():          # the refused calls left the segment alone
        assert _bits(val) == _bits(seg4[k]), k
    ctx.close()
    two = capi.Context(w, h, 2)
    two.make_images(0, co.render(w, h, 5))
    for bad in (lambda: two.select_pixels(0), lambda: two.make_new_traces_pixels(0)):
        with pytest.raises(capi.Error, match="error -1"):
            bad()
    two.close()
    sh = capi.Context(w, h, 3)
    sh.make_images(0, co.render(w, h, 5))
    sh.set_shard(0, 1)
    with pytest.raises(capi.Error, match="error -3"):
        sh.make_new_traces_pixels(0)
    sh.close()

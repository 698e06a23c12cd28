"""The immature-point store on the device (ldso_b200_make_new_traces / immature_seed / trace_new_coarse / activate_immature /
immature_release / immature_read) against the one-shot entry points it reuses, bit for bit, and against the oracle at their bars:
seeding equals detect_corners + immature_init, tracing equals trace_immature and OracleTrace.trace_on, activation equals
select_activation + optimize_immature with the bookkeeping restated in tests/test_immature_store_cpu.py."""
from __future__ import annotations

import os

import numpy as np
import pytest

from ldso_b200 import capi, synth
from tests import corners_oracle as co
from tests import oracle_py
from tests.test_immature_store_cpu import apply_release, bookkeeping, gather

pytestmark = pytest.mark.gpu
FIELDS = ("idepth_min", "idepth_max", "quality", "status", "uv", "interval")


def _bits(a):
    return np.ascontiguousarray(a).tobytes()


@pytest.mark.parametrize("path", co.fixtures(), ids=os.path.basename)
def test_make_new_traces_seeds_like_detect_corners_and_immature_init(path):
    z = co.load(path)
    w, h, nFeat = int(z["w"]), int(z["h"]), int(z["n_features"])
    ctx = capi.Context(w, h, 3)
    ctx.set_orb_pattern(z["pattern"])
    ctx.make_images(2, z["image"])
    want = ctx.detect_corners(2, nFeat, z["B"])
    got = ctx.make_new_traces(2, nFeat, z["B"])
    for k in ("u", "v", "score", "is_corner", "angle", "descriptor"):
        assert _bits(got[k]) == _bits(want[k]), k
    assert got["n_corners"] == want["n_corners"]
    init = ctx.immature_init(2, want["u"], want["v"])
    s = ctx.immature_read(2)
    n = len(want["u"])
    assert len(s["u"]) == n and s["live"].all()
    assert _bits(s["u"]) == _bits(want["u"]) and _bits(s["v"]) == _bits(want["v"])
    for k in ("color", "weights", "gradH", "energyTH"):
        assert _bits(s[k]) == _bits(init[k]), k
    assert np.all(s["my_type"] == 1) and np.all(s["idepth_min"] == 0) and np.all(np.isnan(s["idepth_max"]))
    assert np.all(s["quality"] == 10000) and np.all(s["status"] == oracle_py.IPS_UNINITIALIZED)
    ctx.close()


def _geom(geom):
    if geom == "small":
        return synth.make_window(nF=6, pts_per_frame=40, w=320, h=240, seed=3), 150
    if geom == "vga":
        return synth.make_window(nF=8, pts_per_frame=250, seed=42), 250
    return synth.make_window(nF=5, pts_per_frame=150, w=1232, h=368, seed=11, K=np.array([718.856, 718.856, 607.1928, 185.2157])), 300


def _seed(ctx, case, hosts, my_type):
    for f in hosts:
        m = case.host == f
        ctx.immature_seed(int(f), case.u[m], case.v[m], my_type[m])


def _read_all(ctx, hosts):
    segs = [ctx.immature_read(int(f)) for f in hosts]
    return {k: np.concatenate([s[k] for s in segs]) for k in segs[0]}


def _trace(ctx, case, hosts, new, counts=False):
    return ctx.trace_new_coarse(new, hosts, case.KRKi[new][hosts], case.Kt[new][hosts], case.aff[new][hosts], counts=counts)


@pytest.mark.parametrize("geom", ["small", "vga", "kitti"])
def test_trace_new_coarse_matches_trace_immature_and_oracle(geom):
    win, per_host = _geom(geom)
    case = synth.make_trace_case(win, per_host, seed=5)
    hosts = np.unique(case.host).astype(np.int32)
    my_type = np.random.default_rng(11).choice(np.array([1.0, 2.0, 4.0], np.float32), case.n)
    ctx = capi.Context(win.w, win.h, win.levels)
    for i in range(win.nF):
        ctx.upload_frame(i, win.pyramids[i])
    _seed(ctx, case, hosts, my_type)
    s0 = _read_all(ctx, hosts)
    assert np.array_equal(s0["my_type"], my_type)
    tr = oracle_py.OracleTrace(win, case)
    tr.color, tr.weights, tr.gradH, tr.energyTH = s0["color"].copy(), s0["weights"].copy(), s0["gradH"].copy(), s0["energyTH"].copy()
    pts = dict(u=case.u, v=case.v, host=case.host, color=s0["color"], weights=s0["weights"], gradH=s0["gradH"], energyTH=s0["energyTH"],
               idepth_min=s0["idepth_min"].copy(), idepth_max=s0["idepth_max"].copy(), quality=s0["quality"].copy(),
               status=s0["status"].copy(), uv=s0["uv"].copy(), interval=s0["interval"].copy())
    for new in (win.nF - 2, win.nF - 1):
        so = tr.trace_on(new)
        ctx.trace_immature(new, pts, case.KRKi[new], case.Kt[new], case.aff[new])
        c7 = _trace(ctx, case, hosts, new, counts=True)
        s = _read_all(ctx, hosts)
        ora = dict(idepth_min=tr.idepth_min, idepth_max=tr.idepth_max, quality=tr.quality, status=so, uv=tr.uv, interval=tr.interval)
        for k in FIELDS:
            assert _bits(s[k]) == _bits(pts[k]), (geom, new, k, "trace_immature")
            assert _bits(s[k]) == _bits(ora[k].astype(s[k].dtype)), (geom, new, k, "oracle")
        for k in ("u", "v", "color", "weights", "gradH", "energyTH", "my_type"):
            assert _bits(s[k]) == _bits(s0[k]), k
        want = [case.n] + [int((so == st).sum()) for st in range(6)]
        assert c7.tolist() == want, (c7.tolist(), want)
        assert (so == oracle_py.IPS_GOOD).sum() > 0.3 * case.n
    ctx.close()


def _expected_activation(ctx, cand, newest, dist, flagged, min_obs, nF, o=None):
    """select_activation + optimize_immature on the gathered candidates, then the bookkeeping restatement (and, given the oracle,
    its selection bit for bit and its activation decisions at >= 99 %)."""
    args = (cand["u"], cand["v"], cand["frame"], cand["idepth_min"], cand["idepth_max"], cand["status"], cand["interval"],
            cand["quality"], cand["my_type"])
    action = ctx.select_activation(newest, dist, *args, frame_flagged=flagged)
    s = action == 1
    sel = (cand["u"][s], cand["v"][s], cand["frame"][s], cand["idepth_min"][s], cand["idepth_max"][s], cand["color"][s],
           cand["weights"][s], cand["energyTH"][s])
    ok, idepth, res = ctx.optimize_immature(*sel, min_obs=min_obs)
    if o is not None:
        ao, _ = o.select_activation(newest, dist, *args, frame_flagged=flagged)
        assert np.array_equal(action, ao), (dist, int((action != ao).sum()))
        oko, _, _ = o.optimize_immature(*sel, min_obs=min_obs)
        assert (ok == oko).mean() >= 0.99
    return action, bookkeeping(cand, action, ok, idepth, res, nF), int(ok.sum())


def _assert_same_records(got, want, n_valid, what):
    for k in want:
        assert _bits(got[k]) == _bits(want[k].astype(got[k].dtype)), (what, k)
    assert got["n_valid"] == n_valid, what


@pytest.mark.parametrize("geom,permuted", [("small", False), ("small", True), ("vga", False), ("kitti", True)])
def test_activate_immature_matches_select_and_optimize(geom, permuted):
    """permuted: window frame f lives in image slot (3f + 5) mod 16, so a frame index used as a slot (or the reverse) shows."""
    win, per_host = _geom(geom)
    case = synth.make_trace_case(win, per_host, seed=5)
    hosts = np.unique(case.host).astype(np.int32)
    slot_of = np.array([(3 * f + 5) % 16 if permuted else f for f in range(win.nF)], np.int32)
    my_type = np.random.default_rng(11).choice(np.array([1.0, 2.0, 4.0], np.float32), case.n)
    ctx = capi.Context(win.w, win.h, win.levels)
    for f in range(win.nF):
        ctx.upload_frame(int(slot_of[f]), win.pyramids[f])
    ctx.set_frames(win.Rcw, win.tcw, win.state_zero, win.state, win.ab_exposure, win.frame_id, slot_of, win.K)
    ctx.set_window(win.pt_host, win.pt_u, win.pt_v, win.pt_idepth, win.pt_idepth_zero, win.pt_has_prior, win.pt_color, win.pt_weights,
                   win.res_begin, win.res_target)
    o = oracle_py.OracleBA(win, threads_mode=0)
    newest = win.nF - 1
    seen = set()
    for dist, flag0, min_obs in ((0.0, 0, 1), (2.0, 1, 1), (4.0, 1, 3)):
        flagged = np.zeros(win.nF, np.uint8); flagged[0] = flag0
        for f in hosts:
            m = case.host == f
            ctx.immature_seed(int(slot_of[f]), case.u[m], case.v[m], my_type[m])
        for new in (win.nF - 2, win.nF - 1):
            ctx.trace_new_coarse(int(slot_of[new]), slot_of[hosts], case.KRKi[new][hosts], case.Kt[new][hosts], case.aff[new][hosts])
        segs = [ctx.immature_read(int(slot_of[f])) if f in hosts else None for f in range(win.nF)]
        cand = gather(segs, win.nF)
        action, want, n_valid = _expected_activation(ctx, cand, newest, dist, flagged, min_obs, win.nF, o)
        got = ctx.activate_immature(dist, frame_flagged=flagged, min_obs=min_obs)
        _assert_same_records(got, want, n_valid, (geom, permuted, dist, "first"))
        after = apply_release(segs, want)
        for f in hosts:
            r = ctx.immature_read(int(slot_of[f]))
            assert np.array_equal(r["live"], after[f]["live"])
            for k in ("u", "v", "color", "weights", "gradH", "energyTH") + FIELDS:
                assert _bits(r[k]) == _bits(segs[f][k]), k
        seen |= set(np.unique(action).tolist())
        # a second activation, with released entries in the middle of the segments: only what stayed live, same bar
        cand2 = gather(after, win.nF)
        assert len(cand2["u"]) == int((action == 0).sum())
        _, want2, n_valid2 = _expected_activation(ctx, cand2, newest, dist, flagged, min_obs, win.nF)
        again = ctx.activate_immature(dist, frame_flagged=flagged, min_obs=min_obs)
        _assert_same_records(again, want2, n_valid2, (geom, permuted, dist, "second"))
        after2 = apply_release(after, want2)
        for f in hosts:
            assert np.array_equal(ctx.immature_read(int(slot_of[f]))["live"], after2[f]["live"])
    assert seen == {0, 1, 2}, seen
    ctx.close()


def test_seeding_unequal_counts_grows_the_store():
    """immature_seed with increasing, unequal counts on one context: the store grows, every segment keeps its bits, and a refused
    seed leaves its segment as it was."""
    win, _ = _geom("small")
    ctx = capi.Context(win.w, win.h, win.levels)
    for i in range(win.nF):
        ctx.upload_frame(i, win.pyramids[i])
    rng = np.random.default_rng(3)
    pts = {}
    for f, n in ((0, 100), (1, 101), (2, 37), (3, 400), (0, 650)):        # slot 0 again, larger, while the others are live
        u = rng.integers(20, win.w - 20, n).astype(np.float32) + 0.25
        v = rng.integers(20, win.h - 20, n).astype(np.float32)
        t = rng.choice(np.array([1.0, 2.0], np.float32), n)
        ctx.immature_seed(f, u, v, t)
        pts[f] = (u, v, t)
        for g, (ug, vg, tg) in pts.items():
            s = ctx.immature_read(g)
            init = ctx.immature_init(g, ug, vg)
            assert len(s["u"]) == len(ug) and s["live"].all(), (f, g)
            assert _bits(s["u"]) == _bits(ug) and _bits(s["v"]) == _bits(vg) and _bits(s["my_type"]) == _bits(tg)
            for k in ("color", "weights", "gradH", "energyTH"):
                assert _bits(s[k]) == _bits(init[k]), (f, g, k)
    # traced state survives a growth too
    case = synth.make_trace_case(win, 1, seed=5)
    hs = np.array([1, 2, 3], np.int32)
    ctx.trace_new_coarse(win.nF - 1, hs, case.KRKi[win.nF - 1][hs], case.Kt[win.nF - 1][hs], case.aff[win.nF - 1][hs])
    before = {int(g): ctx.immature_read(int(g)) for g in hs}
    u = rng.integers(20, win.w - 20, 900).astype(np.float32)
    ctx.immature_seed(4, u, u % (win.h - 40) + 20)
    for g in hs:
        r = ctx.immature_read(int(g))
        assert all(_bits(r[k]) == _bits(before[int(g)][k]) for k in r), g
    # a refused seed (a pattern leaving the image) keeps the slot's segment
    with pytest.raises(capi.Error, match="error -1"):
        ctx.immature_seed(1, [1.0], [30.0])
    r = ctx.immature_read(1)
    assert all(_bits(r[k]) == _bits(before[1][k]) for k in r)
    ctx.close()


def test_make_new_traces_without_cells_gives_no_features():
    z = co.load([p for p in co.fixtures() if "synth_640x480" in p][0])
    ctx = capi.Context(640, 480, 3)
    ctx.set_orb_pattern(z["pattern"])
    ctx.make_images(2, z["image"])
    assert capi.feature_capacity(640, 480, 1) == 0
    want = ctx.detect_corners(2, 1)
    got = ctx.make_new_traces(2, 1)
    assert len(want["u"]) == 0 and len(got["u"]) == 0 and got["n_corners"] == want["n_corners"] == 0
    assert len(ctx.immature_read(2)["u"]) == 0
    ctx.close()


def test_life_cycle_on_one_context():
    win, per_host = _geom("small")
    case = synth.make_trace_case(win, per_host, seed=5)
    hosts = np.unique(case.host).astype(np.int32)
    ones = np.ones(case.n, np.float32)
    ctx = capi.Context(win.w, win.h, win.levels)
    ctx.load_synth_window(win)
    _seed(ctx, case, hosts, ones)
    _trace(ctx, case, hosts, win.nF - 2)
    before = {int(f): ctx.immature_read(int(f)) for f in hosts}
    # uploading a different image into a host's slot leaves its segment alone (then the keyframe's own image goes back)
    ctx.upload_frame(int(hosts[0]), win.pyramids[win.nF - 1])
    assert all(_bits(v) == _bits(before[int(hosts[0])][k]) for k, v in ctx.immature_read(int(hosts[0])).items())
    ctx.upload_frame(int(hosts[0]), win.pyramids[int(hosts[0])])
    rel = ctx.activate_immature(2.0)
    assert len(rel["frame"]) > 0
    released = {(int(f), int(k)) for f, k in zip(rel["frame"], rel["index"])}
    snap = {int(f): ctx.immature_read(int(f)) for f in hosts}
    # release host 1, re-seed host 2 from other coordinates, trace again: untouched segments keep their bits
    ctx.immature_release(int(hosts[1]))
    m2 = case.host == hosts[2]
    ctx.immature_seed(int(hosts[2]), case.u[m2][:50] + 1, case.v[m2][:50])
    r1 = ctx.immature_read(int(hosts[1]))
    assert not r1["live"].any() and all(_bits(r1[k]) == _bits(snap[int(hosts[1])][k]) for k in r1 if k != "live")
    r2 = ctx.immature_read(int(hosts[2]))
    assert len(r2["u"]) == 50 and r2["live"].all() and np.all(r2["status"] == oracle_py.IPS_UNINITIALIZED)
    _trace(ctx, case, hosts, win.nF - 1)
    r1b = ctx.immature_read(int(hosts[1]))
    assert all(_bits(r1b[k]) == _bits(r1[k]) for k in r1)
    r0 = ctx.immature_read(int(hosts[0]))
    dead = np.array([(int(hosts[0]), k) in released for k in range(len(r0["u"]))])
    for k in FIELDS:      # released entries never change again; live ones were traced
        assert _bits(r0[k][dead]) == _bits(snap[int(hosts[0])][k][dead]), k
    assert not np.array_equal(r0["status"][~dead], snap[int(hosts[0])]["status"][~dead])
    # a second make_new_traces on a slot replaces its segment (the store grows to the density's capacity once nothing is live)
    for f in hosts:
        ctx.immature_release(int(f))
    ctx.set_orb_pattern(co.load(co.fixtures()[0])["pattern"])
    f1 = ctx.make_new_traces(int(hosts[3]), 300)
    a = ctx.immature_read(int(hosts[3]))
    assert len(a["u"]) == len(f1["u"]) and _bits(a["u"]) == _bits(f1["u"]) and a["live"].all()
    f2 = ctx.make_new_traces(int(hosts[3]), 300)
    b = ctx.immature_read(int(hosts[3]))
    assert _bits(b["u"]) == _bits(f2["u"]) and np.all(b["status"] == oracle_py.IPS_UNINITIALIZED)
    ctx.close()


def test_errors_and_empty_cases():
    win, per_host = _geom("small")
    case = synth.make_trace_case(win, 20, seed=5)
    hosts = np.unique(case.host).astype(np.int32)
    ctx = capi.Context(win.w, win.h, win.levels)
    for i in range(win.nF):
        ctx.upload_frame(i, win.pyramids[i])
    # empty store, empty lists
    assert ctx.trace_new_coarse(win.nF - 1, hosts, case.KRKi[win.nF - 1][hosts], case.Kt[win.nF - 1][hosts], case.aff[win.nF - 1][hosts],
                                counts=True).tolist() == [0] * 7
    ctx.trace_new_coarse(win.nF - 1, [], np.zeros((0, 3, 3)), np.zeros((0, 3)), np.zeros((0, 2)))
    ctx.immature_seed(0, [], [])
    assert len(ctx.immature_read(0)["u"]) == 0
    ctx.immature_release(5)
    # activation before set_frames / set_window
    with pytest.raises(capi.Error, match="set_frames"):
        ctx.activate_immature(2.0, capacity=10)
    ctx.load_synth_window(win)
    assert len(ctx.activate_immature(2.0, capacity=1)["frame"]) == 0
    _seed(ctx, case, hosts, np.ones(case.n, np.float32))
    ctx.set_orb_pattern(co.load(co.fixtures()[0])["pattern"])
    # slot out of range, a host listed twice, coordinates whose pattern leaves the image, small capacities
    for bad in (lambda: ctx.immature_seed(16, case.u[:3], case.v[:3]), lambda: ctx.immature_seed(-1, case.u[:3], case.v[:3]),
                lambda: ctx.immature_seed(0, [1.0], [30.0]), lambda: ctx.immature_seed(0, [30.0], [win.h - 3.0]),
                lambda: ctx.immature_read(16), lambda: ctx.immature_release(16),
                lambda: ctx.immature_read(int(hosts[0]), capacity=5),
                lambda: ctx.trace_new_coarse(16, hosts[:1], case.KRKi[0][:1], case.Kt[0][:1], case.aff[0][:1]),
                lambda: ctx.trace_new_coarse(win.nF - 1, [0, 16], case.KRKi[0][:2], case.Kt[0][:2], case.aff[0][:2]),
                lambda: ctx.trace_new_coarse(win.nF - 1, [0, 0], case.KRKi[0][:2], case.Kt[0][:2], case.aff[0][:2]),
                lambda: ctx.activate_immature(2.0, capacity=5),
                lambda: ctx.make_new_traces(0, 0), lambda: ctx.make_new_traces(0, 1500, capacity=10)):
        with pytest.raises(capi.Error) as e:
            bad()
        assert "error -1" in str(e.value), str(e.value)
    seg0 = ctx.immature_read(0)
    assert len(seg0["u"]) == 20 and seg0["live"].all()          # the refused calls left slot 0's segment alone
    # a density that needs a larger store while entries are live, then again once every segment is empty
    with pytest.raises(capi.Error, match="error -3"):
        ctx.make_new_traces(0, 1500)
    assert all(_bits(v) == _bits(seg0[k]) for k, v in ctx.immature_read(0).items())
    for f in hosts:
        ctx.immature_release(int(f))
    ctx.make_new_traces(0, 1500)
    assert ctx.immature_read(0)["live"].all()
    ctx.close()
    # sharded contexts
    sh = capi.Context(win.w, win.h, win.levels)
    sh.upload_frame(0, win.pyramids[0])
    sh.set_shard(0, 1)
    for call in (lambda: sh.immature_seed(0, case.u[:3], case.v[:3]), lambda: sh.immature_read(0), lambda: sh.immature_release(0),
                 lambda: sh.trace_new_coarse(0, [], np.zeros((0, 9)), np.zeros((0, 3)), np.zeros((0, 2))),
                 lambda: sh.activate_immature(2.0, capacity=1), lambda: sh.make_new_traces(0, 1500)):
        with pytest.raises(capi.Error, match="error -3"):
            call()
    sh.close()

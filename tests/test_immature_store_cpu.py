"""The immature-point store without a GPU: the numpy restatement of activatePointsMT's bookkeeping (FullSystem.cc:1096-1188) that
the GPU tests hold the device store to, checked against the oracle's selection and activation LM, and the ABI drift guard of the
store's structs."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from ldso_b200 import capi, synth
from tests import oracle_py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FEATURE_VALID, FEATURE_OUTLIER = 1, 2


def gather(segs, nF):
    """activatePointsMT's candidates: the live entries of window frames 0..nF-2 in window order, then feature-index order.
    segs[f] is a segment as immature_read returns it (None = empty). Returns the candidate arrays and (frame, index) per candidate."""
    keys = ("u", "v", "idepth_min", "idepth_max", "status", "interval", "quality", "my_type", "color", "weights", "energyTH")
    parts = {k: [] for k in keys}
    frame, index = [], []
    for f in range(nF - 1):
        s = segs[f]
        if s is None:
            continue
        idx = np.nonzero(s["live"])[0]
        for k in keys:
            parts[k].append(s[k][idx])
        frame.append(np.full(len(idx), f, np.int32)); index.append(idx.astype(np.int32))
    out = {k: (np.concatenate(v) if v else np.zeros(0, np.float32)) for k, v in parts.items()}
    out["frame"] = np.concatenate(frame) if frame else np.zeros(0, np.int32)
    out["index"] = np.concatenate(index) if index else np.zeros(0, np.int32)
    return out


def bookkeeping(cand, action, ok, idepth, res_state, nF):
    """FullSystem.cc:1104-1109, 1119-1126, 1145-1149 (action 2: released as OUTLIER) and :1167-1186 (a selected candidate is
    released as VALID when optimizeImmaturePoint returned a point, as OUTLIER otherwise); action 0 stays live. ok / idepth /
    res_state are per selected candidate, in visiting order. Returns the released records in visiting order."""
    sel_pos = np.cumsum(action == 1) - 1
    rel = np.nonzero(action != 0)[0]
    sel = action[rel] == 1
    ok_rel = np.zeros(len(rel), bool)
    idp = np.full(len(rel), np.nan, np.float32)
    rs = np.full((len(rel), nF), 255, np.uint8)
    if sel.any():
        p = sel_pos[rel][sel]
        ok_rel[sel] = ok[p] != 0
        idp[sel] = idepth[p]
        rs[sel] = res_state[p]
    status = np.where(ok_rel, FEATURE_VALID, FEATURE_OUTLIER).astype(np.int32)
    return dict(frame=cand["frame"][rel], index=cand["index"][rel], status=status, idepth=idp, res_state=rs,
                idepth_min=cand["idepth_min"][rel], idepth_max=cand["idepth_max"][rel], color=cand["color"][rel],
                weights=cand["weights"][rel], energyTH=cand["energyTH"][rel], my_type=cand["my_type"][rel])


def apply_release(segs, released):
    """The store after activation: released entries are no longer live, everything else is unchanged."""
    out = [None if s is None else dict(s, live=s["live"].copy()) for s in segs]
    for f, k in zip(released["frame"], released["index"]):
        out[f]["live"][k] = False
    return out


def segments_from_oracle(tr, case, nF, my_type):
    """The oracle's traced candidates as store segments of window frames (the case's host = window frame = segment)."""
    segs = [None] * nF
    for f in np.unique(case.host):
        m = case.host == f
        segs[f] = dict(u=case.u[m], v=case.v[m], idepth_min=tr.idepth_min[m], idepth_max=tr.idepth_max[m], status=tr.status[m],
                       interval=tr.interval[m], quality=tr.quality[m], my_type=my_type[m], color=tr.color[m], weights=tr.weights[m],
                       energyTH=tr.energyTH[m], live=np.ones(int(m.sum()), bool))
    return segs


def test_bookkeeping_against_oracle_activation():
    win = synth.make_window(nF=6, pts_per_frame=40, w=320, h=240, seed=3)
    case = synth.make_trace_case(win, 150, seed=5)
    tr = oracle_py.OracleTrace(win, case)
    tr.trace_on(win.nF - 2); tr.trace_on(win.nF - 1)
    my_type = np.random.default_rng(11).choice(np.array([1.0, 2.0, 4.0], np.float32), case.n)
    segs = segments_from_oracle(tr, case, win.nF, my_type)
    segs[1]["live"][::7] = False                    # entries an earlier activation released are not candidates
    o = oracle_py.OracleBA(win, threads_mode=0)
    flagged = np.zeros(win.nF, np.uint8); flagged[0] = 1
    for dist in (0.0, 2.0):
        cand = gather(segs, win.nF)
        assert len(cand["u"]) == sum(int(s["live"].sum()) for s in segs if s is not None)
        assert np.all(np.diff(cand["frame"]) >= 0)
        args = (cand["u"], cand["v"], cand["frame"], cand["idepth_min"], cand["idepth_max"], cand["status"], cand["interval"],
                cand["quality"], cand["my_type"])
        action, _ = o.select_activation(win.nF - 1, dist, *args, frame_flagged=flagged)
        s = action == 1
        ok, idepth, res = o.optimize_immature(cand["u"][s], cand["v"][s], cand["frame"][s], cand["idepth_min"][s], cand["idepth_max"][s],
                                              cand["color"][s], cand["weights"][s], cand["energyTH"][s])
        rel = bookkeeping(cand, action, ok, idepth, res, win.nF)
        # the reference's rules, candidate by candidate
        never = ~np.isfinite(cand["idepth_max"]) | (cand["status"] == oracle_py.IPS_OUTLIER)
        assert np.all(action[never] == 2)
        assert len(rel["frame"]) == int((action != 0).sum())
        assert int((rel["status"] == FEATURE_VALID).sum()) == int(ok.sum())
        assert np.all(rel["status"][action[action != 0] == 2] == FEATURE_OUTLIER)
        assert np.all(np.isnan(rel["idepth"][action[action != 0] == 2]))
        assert np.array_equal(rel["idepth"][rel["status"] == FEATURE_VALID], idepth[ok != 0])
        after = apply_release(segs, rel)
        assert sum(int(a["live"].sum()) for a in after if a is not None) == sum(int(b["live"].sum()) for b in segs if b is not None) - len(rel["frame"])
        # a second activation sees only what stayed live
        again = gather(after, win.nF)
        assert len(again["u"]) == int((action == 0).sum())
        assert set(np.unique(action).tolist()) <= {0, 1, 2} and (action == 1).any() and (action == 2).any()


def test_store_structs_match_the_header(tmp_path):
    pairs = [("ldso_b200_activation_out", capi.ActivationOutC), ("ldso_b200_immature_segment", capi.ImmatureSegmentC)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ldso_b200.h"', 'int main(void) {',
             '  printf("VALID %d\\n", LDSO_B200_FEATURE_VALID);', '  printf("OUTLIER %d\\n", LDSO_B200_FEATURE_OUTLIER);']
    for cname, cls in pairs:
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, *_ in cls._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src = tmp_path / "abi.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "abi"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert (int(got["VALID"]), int(got["OUTLIER"])) == (capi.FEATURE_VALID, capi.FEATURE_OUTLIER) == (FEATURE_VALID, FEATURE_OUTLIER)
    for cname, cls in pairs:
        assert int(got[cname]) == C.sizeof(cls), (cname, got[cname], C.sizeof(cls))
        for fname, *_ in cls._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)

"""Write tests/golden/pixsel_*.npz: PixelSelector::makeMaps fixtures, so that the GPU tests need neither the reference nor the pin.

Needs the pin library (oracle/_ref/libref_pixsel_pin.so, built by `make -C oracle -f pixsel.mk ref_pin REF=<reference checkout>`).
Each case is a sequence of makeMaps calls on one selector (currentPotential carried from call to call). For each call it renders the
image (tests/pixsel_oracle.py image(): exact floats from a few integers; the fixture keeps those and the image's SHA-256), runs the
restatement and the reference's own makeImages + makeMaps, checks that maps, counts and potentials agree, and stores the restatement's
map, n, (n2, n3, n4), the pass's mixed direction masks and the potentials before and after.

    python tests/golden/make_pixsel_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import corners_oracle as co  # noqa: E402
from tests import pixsel_oracle as po  # noqa: E402

# name: (w, h, [(kind, seed), ...], B, pot_in, params)
CASES = {
    "d1500_640x480": (640, 480, [("noise", 11)], "identity", 3, {}),
    "d6000_640x480": (640, 480, [("noise", 23)], "identity", 3, dict(density=6000.0)),          # no recursion, no subsampling
    "d4000_640x480": (640, 480, [("noise", 12)], "identity", 3, dict(density=4000.0)),          # no recursion, subsampled
    "d12000_640x480": (640, 480, [("noise", 22)], "identity", 3, dict(density=12000.0)),        # quotia > 1.25: a smaller potential
    "d150_640x480": (640, 480, [("noise", 13)], "identity", 3, dict(density=150.0)),            # quotia < 0.25: a larger potential
    "d1500_1232x368": (1232, 368, [("noise", 14)], "identity", 3, {}),                          # thsSmoothed wrap, level-2 row h2-1
    "gamma_640x480": (640, 480, [("noise", 15)], "gamma", 3, {}),
    "nodir_640x480": (640, 480, [("noise", 16)], "identity", 3, dict(selectDirectionDistribution=0)),
    "init_640x480": (640, 480, [("noise", 17)], "identity", 3, dict(density=0.03 * 640 * 480, th_factor=2.0)),
    "flat_640x480": (640, 480, [("flat", 0)], "identity", 3, {}),
    "steps_640x480": (640, 480, [("steps", 18)], "identity", 3, {}),
    "seq3_640x480": (640, 480, [("noise", 19), ("noise", 20), ("steps", 21)], "identity", 3, {}),
}


def run(w, h, calls, B, pot_in, params, sel_cls):
    sel = sel_cls(w, h)
    sel.potential = pot_in
    out = []
    for kind, seed in calls:
        before = sel.potential
        r = sel.make_maps(po.image(kind, w, h, seed), B, **params)
        out.append((before, sel.potential) + tuple(r))
    return out


def pack(name, w, h, calls, Bk, pot_in, params):
    B = co.gamma_B(Bk)
    ora = run(w, h, calls, B, pot_in, params, po.Selector)
    ref = run(w, h, calls, B, pot_in, params, po.RefSelector)
    for (pb, pa, mp, n, cnt, mixed), (rpb, rpa, rmp, rn) in zip(ora, ref):
        assert (pb, pa, n) == (rpb, rpa, rn), (name, (pb, pa, n), (rpb, rpa, rn))
        assert np.array_equal(mp.astype(np.float32), rmp), name
        assert n == int((mp != 0).sum())
    p = dict(po.DEFAULT, **params)
    z = dict(w=w, h=h, kind=np.array([k for k, _ in calls]), seed=np.array([s for _, s in calls], np.int64),
             image_sha256=np.array([co.image_sha(po.image(k, w, h, s)) for k, s in calls]), has_B=int(B is not None),
             B=B if B is not None else np.zeros(256, np.float32), pot_before=np.array([o[0] for o in ora], np.int32),
             pot_after=np.array([o[1] for o in ora], np.int32), maps=np.stack([o[2] for o in ora]),
             n=np.array([o[3] for o in ora], np.int32), counts=np.array([o[4] for o in ora], np.int32),
             mixed=np.array([o[5] for o in ora], np.int32))
    for k, v in p.items():
        z["p_" + k] = v
    path = os.path.join(HERE, f"pixsel_{name}.npz")
    np.savez_compressed(path, **z)
    print(f"pixsel_{name}: n={z['n'].tolist()} counts={z['counts'].tolist()} pot {z['pot_before'].tolist()} -> {z['pot_after'].tolist()} "
          f"mixed={z['mixed'].tolist()} {os.path.getsize(path) / 1024:.0f} KB")


if __name__ == "__main__":
    assert po.pin() is not None, "build the pin first: make -C oracle -f pixsel.mk ref_pin REF=<reference checkout>"
    for name, args in CASES.items():
        pack(name, *args)

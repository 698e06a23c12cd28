"""Write tests/golden/corners_*.npz: FeatureDetector::DetectCorners fixtures, so that the GPU tests need neither the reference nor the pin.

Needs the pin library (oracle/_ref/libref_corners_pin.so, built by `make -C oracle -f corners.mk ref_pin REF=<reference checkout>`).
For each case it renders the image (tests/corners_oracle.py render(): exact floats from a few integers; the fixture keeps those integers
and the image's SHA-256), runs the reference's own makeImages + DetectCorners and the restatement, and stores:
  - the restatement's features (u, v as uint16, score, is_corner; angle and descriptor of the corners only) and n_corners;
  - the reference's features as their difference from the restatement: every feature of the excluded cells (the cells whose picks
    depend on how std::sort orders equal or NaN scores), the features beside them that the reference suppresses differently, and, per
    corner elsewhere, the angle's distance in ulps (atan2f against atan2 rounded to float). The script checks that this reproduces the
    reference's outputs exactly before it writes anything;
  - B, n_features, the ORB pattern (ldso::bit_pattern_31_ read from the compiled reference), the excluded cells.

    python tests/golden/make_corners_golden.py
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import corners_oracle as co  # noqa: E402

# name: (w, h, n_features, seed, quantise, dots, B)
CASES = {
    "synth_640x480": (640, 480, 1500, 1, 0, 0, "identity"),
    "synth_1232x368": (1232, 368, 1500, 2, 0, 0, "identity"),
    "render8_640x480": (640, 480, 1500, 3, 1, 300, "identity"),
    "gamma_640x480": (640, 480, 1500, 4, 0, 0, "gamma"),
    "d800_640x480": (640, 480, 800, 5, 0, 0, "identity"),
    "d2000_640x480": (640, 480, 2000, 6, 0, 0, "identity"),
    "d4000_640x480": (640, 480, 4000, 7, 0, 0, "identity"),
    "limit_635x480": (635, 480, 317, 8, 0, 0, "identity"),     # the last cells' patches end exactly on the right and bottom edge
}


def pack(name, w, h, nF, seed, quantise, dots, Bk):
    img = co.render(w, h, seed, quantise, dots)
    B = co.gamma_B(Bk)
    pat = co.ref_pattern()
    ref, rnc = co.ref_detect(img, B, nF)
    ora, onc = co.detect(img, B, nF, pat)
    rep = co.compare(w, h, nF, ref, ora)
    assert rep["same_list"] and rep["corner_mismatch"] == 0 and rep["descriptor_mismatch"] == 0 and rep["angle_max_ulp"] <= 1, rep
    ex = rep["excluded_cells"]
    rc, oc = co.cell_of(w, h, nF, ref["u"], ref["v"]), ora["cell"]
    corner = ora["is_corner"] != 0
    z = dict(w=w, h=h, seed=seed, quantise=quantise, dots=dots, image_sha256=co.image_sha(img), has_B=int(B is not None),
             B=B if B is not None else np.zeros(256, np.float32), n_features=nF, pattern=pat, excluded_cells=ex,
             ora_u=ora["u"].astype(np.uint16), ora_v=ora["v"].astype(np.uint16), ora_score=ora["score"], ora_is_corner=ora["is_corner"],
             ora_angle=ora["angle"][corner], ora_descriptor=ora["descriptor"][corner], ora_n_corners=onc, ref_n_corners=rnc)
    # the reference's features in the excluded cells, and the angle ulps of the rest
    inr, ino = np.isin(rc, ex), np.isin(oc, ex)
    for k in co.FIELDS:
        z["ref_ex_" + k] = ref[k][inr]
    z["ref_ex_u"], z["ref_ex_v"] = z["ref_ex_u"].astype(np.uint16), z["ref_ex_v"].astype(np.uint16)
    ulp = np.zeros(len(ora["u"]), np.int8)
    keep = ~ino
    # outside the excluded cells the two lists hold the same features in the same order
    rk = {k: ref[k][~inr] for k in co.FIELDS}
    assert np.array_equal(rk["u"], ora["u"][keep]) and np.array_equal(rk["v"], ora["v"][keep])
    d = rk["angle"].view(np.int32).astype(np.int64) - ora["angle"][keep].view(np.int32).astype(np.int64)
    # features set aside beside the excluded cells may be suppressed differently: those whose is_corner or descriptor differ are
    # stored whole
    fix = (rk["is_corner"] != ora["is_corner"][keep]) | (rk["descriptor"] != ora["descriptor"][keep]).any(1) | (np.abs(d) > 1)
    d[fix] = 0
    ulp[keep] = d
    z["ref_angle_ulp"] = ulp
    kidx = np.flatnonzero(keep)
    z["ref_fix_idx"] = kidx[fix].astype(np.int32)
    for k in ("is_corner", "angle", "descriptor"):
        z["ref_fix_" + k] = rk[k][fix]
    got = expand_reference(z)
    for k in co.FIELDS:
        assert got[k].tobytes() == ref[k].tobytes(), (name, k)
    np.savez_compressed(os.path.join(HERE, f"corners_{name}.npz"), **z)
    kb = os.path.getsize(os.path.join(HERE, f"corners_{name}.npz")) / 1024
    print(f"corners_{name}: n={len(ora['u'])} corners={onc} (reference {rnc}) excluded_cells={len(ex)} set_aside={rep['set_aside']} "
          f"angle_1ulp={rep['angle_mismatch']}/{rep['corners']} descriptor_mismatch={rep['descriptor_mismatch']} {kb:.0f} KB")


def restatement(z):
    """The restatement's features as the fixture stores them, expanded to full arrays."""
    n = len(z["ora_u"])
    corner = z["ora_is_corner"] != 0
    angle = np.zeros(n, np.float32)
    desc = np.zeros((n, 32), np.uint8)
    angle[corner] = z["ora_angle"]
    desc[corner] = z["ora_descriptor"]
    return dict(u=z["ora_u"].astype(np.float32), v=z["ora_v"].astype(np.float32), score=z["ora_score"].copy(), is_corner=z["ora_is_corner"].copy(),
                angle=angle, descriptor=desc)


def expand_reference(z):
    """The reference's features: the restatement's outside the excluded cells with the recorded angle ulps applied, the stored
    reference features inside them, in the reference's order (cells gx outer, gy inner)."""
    o = restatement(z)
    w, h, nF = int(z["w"]), int(z["h"]), int(z["n_features"])
    oc = co.cell_of(w, h, nF, o["u"], o["v"])
    ex = np.asarray(z["excluded_cells"])
    keep = ~np.isin(oc, ex)
    ang = o["angle"].copy()
    ang[keep] = (ang[keep].view(np.int32) + z["ref_angle_ulp"][keep].astype(np.int32)).view(np.float32)
    o["angle"] = ang
    for k in ("is_corner", "angle", "descriptor"):
        o[k][z["ref_fix_idx"]] = z["ref_fix_" + k]
    ex_f = {k: z["ref_ex_" + k] for k in co.FIELDS}
    ex_f["u"], ex_f["v"] = ex_f["u"].astype(np.float32), ex_f["v"].astype(np.float32)
    rc_ex = co.cell_of(w, h, nF, ex_f["u"], ex_f["v"])
    parts = {k: [] for k in co.FIELDS}
    cells = np.union1d(oc[keep], rc_ex)
    for c in cells:
        src, m = (ex_f, rc_ex == c) if c in set(ex.tolist()) else (o, (oc == c) & keep)
        for k in co.FIELDS:
            parts[k].append(src[k][m])
    out = {k: np.concatenate(parts[k]) if parts[k] else o[k][:0] for k in co.FIELDS}
    return out


if __name__ == "__main__":
    assert co.pin() is not None, "build the pin first: make -C oracle -f corners.mk ref_pin REF=<reference checkout>"
    for name, args in CASES.items():
        pack(name, *args)

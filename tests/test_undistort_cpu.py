"""No-GPU checks of the per-frame undistortion: the restatement (oracle/undistort.cc) against the reference's own
Undistort::undistort<T> (the pin, oracle/_ref/pin_undistort, where a reference checkout was found at build time) and against the
fixtures the pin wrote (tests/golden/undistort_*.npz); the edge rule; the C ABI's argument checks that need no device."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from ldso_b200 import capi
from tests import undistort_oracle as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_pin_against_the_reference():
    """Five camera models in crop mode, two with an explicit output calibration, one without rectification; 8- and 16-bit frames;
    photometric modes 0, 1, 2; the factor path through exposure <= 0 and through a missing gamma file: bit for bit."""
    if not os.path.exists(U.PIN):
        pytest.skip("the undistortion pin is built only where a reference checkout exists")
    r = subprocess.run([U.PIN], capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith("PIN ")]
    assert r.returncode == 0, "\n".join(l for l in lines if "mismatches=0" not in l)
    cases = [l for l in lines if "pixels=" in l]
    assert len(cases) == 8 * 11
    for l in cases:
        assert "mismatches=0" in l, l
    models = {l.split()[1].split("_")[0] for l in cases}
    assert models == {"fov", "radtan", "equidistant", "kb", "pinhole"}
    excluded = sum(int(re.search(r"excluded=(\d+)", l).group(1)) for l in cases)
    print(f"pin: {len(cases)} cases, {excluded} pixels excluded (taps past the end of the raw frame)")


@pytest.mark.parametrize("cam", U.CAMERAS)
def test_restatement_matches_fixtures(cam):
    t = U.tables()
    (rx, ry), cases = U.camera(cam)
    seen = set()
    for c, expected, past in cases:
        raw, G, vinv = U.case_inputs(t, c)
        out, e, p = U.undistort(raw, int(c["w"]), int(c["h"]), rx, ry, G, vinv, c["mode"], c["use_exposure"], c["exposure"], c["factor"])
        assert np.array_equal(out.view(np.uint32), expected.view(np.uint32)), (cam, c["name"])
        assert np.array_equal(p, past) and np.float32(e) == c["exposure_out"], (cam, c["name"])
        seen.add((int(c["bpp"]), int(c["mode"])))
    assert seen == {(b, m) for b in (1, 2) for m in (0, 1, 2)}


def test_edge_rule_reads_zero_past_the_end_and_wraps_rows():
    """The two offsets the reference's range check lets through with taps past the end read 0 there; a tap at xxi = wOrg-1 wraps to
    the next row; anything beyond the check is 0."""
    wOrg, hOrg = 5, 4
    raw = (np.arange(wOrg * hOrg, dtype=np.uint8) + 1).reshape(hOrg, wOrg)
    s = raw.reshape(-1).astype(np.float32)
    pts = [(0.5, 3.25),      # src_offset == (hOrg-1)*wOrg: taps +wOrg, +1+wOrg past the end
           (4.5, 2.25),      # src_offset == (hOrg-1)*wOrg - 1: tap +1+wOrg past the end, +1 wraps to the next row
           (4.5, 1.5),       # xxi = wOrg-1: +1 wraps
           (1.0, 3.5),       # src_offset > (hOrg-1)*wOrg: 0
           (-1.0, -1.0)]     # outside: 0
    rx = np.array([p[0] for p in pts], np.float32).reshape(1, -1)
    ry = np.array([p[1] for p in pts], np.float32).reshape(1, -1)
    out, _, past = U.undistort(raw, len(pts), 1, rx, ry, None, None, 0, 1, 1.0, 1.0)
    out, past = out.reshape(-1), past.reshape(-1)
    x, y = np.float32(0.5), np.float32(0.25)
    sp = np.concatenate([s, np.zeros(wOrg + 1, np.float32)])

    def bil(o, xx, yy):
        xxyy = xx * yy
        return xxyy * sp[o + 1 + wOrg] + (yy - xxyy) * sp[o + wOrg] + (xx - xxyy) * sp[o + 1] + (np.float32(1) - xx - yy + xxyy) * sp[o]
    assert out[0] == bil(15, x, y) and past[0] == 1
    assert out[1] == bil(14, x, y) and past[1] == 1
    assert out[2] == bil(9, x, np.float32(0.5)) and past[2] == 0
    assert out[3] == 0 and out[4] == 0


def test_calib_struct_matches_the_header(tmp_path):
    fields = [f for f, *_ in capi.UndistortCalibC._fields_]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ldso_b200.h"', 'int main(void) {',
             '  printf("size %zu\\n", sizeof(ldso_b200_undistort_calib));']
    lines += [f'  printf("{f} %zu\\n", offsetof(ldso_b200_undistort_calib, {f}));' for f in fields]
    lines += ['  return 0;', '}']
    (tmp_path / "abi.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(tmp_path / "abi.c"), "-o", str(tmp_path / "abi")])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / "abi")], text=True).splitlines())
    assert int(got["size"]) == C.sizeof(capi.UndistortCalibC)
    for f in fields:
        assert int(got[f]) == getattr(capi.UndistortCalibC, f).offset, f


def test_null_context_is_an_argument_error():
    L = capi.load()
    c = capi.UndistortCalibC(64, 48, 64, 48, None, None, None, 0, None, 2, 1)
    assert L.ldso_b200_set_undistort(None, C.byref(c)) == -1
    raw = np.zeros(64 * 48, np.uint8)
    assert L.ldso_b200_undistort_frame(None, 0, raw.ctypes.data_as(C.c_void_p), 1, 1.0, 1.0, None) == -1

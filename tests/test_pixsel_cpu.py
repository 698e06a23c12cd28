"""DSO's pixel selection (PixelSelector::makeMaps) without a GPU: the restatement (oracle/pixsel.cc) against the fixtures and, where
a reference checkout was built, against the reference's own PixelSelector2.cc (the pin); the library's randomPattern generator; the
two rules for memory the reference never writes; and the new C structs against the header."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from ldso_b200 import capi
from tests import corners_oracle as co
from tests import pixsel_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = po.fixtures()


def _calls(z):
    """(image, params) of each call of a fixture's sequence, on one selector starting from pot_before[0]."""
    for k, img in enumerate(z["images"]):
        yield k, img, z["params"]


def test_fixture_cases_cover_the_issue():
    # no recursion (d6000, subsampled: d4000), a smaller potential (d12000, init), a larger one (d150)
    names = {os.path.basename(p)[7:-4] for p in FIXTURES}
    assert {"d1500_640x480", "d4000_640x480", "d6000_640x480", "d12000_640x480", "d150_640x480", "d1500_1232x368", "gamma_640x480",
            "nodir_640x480", "init_640x480", "flat_640x480", "steps_640x480", "seq3_640x480"} <= names
    for p in FIXTURES:
        z = po.load(p)
        if os.path.basename(p).startswith("pixsel_steps"):
            assert z["mixed"][0] > 0                    # cells whose level-0 pick depends on the direction occur
        if os.path.basename(p).startswith("pixsel_flat"):
            assert z["n"][0] == 0 and z["counts"][0].sum() == 0


@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_restatement_matches_fixture(path):
    z = po.load(path)
    sel = po.Selector(int(z["w"]), int(z["h"]))
    sel.potential = int(z["pot_before"][0])
    for k, img, p in _calls(z):
        assert sel.potential == int(z["pot_before"][k])
        mp, n, cnt, mixed = sel.make_maps(img, z["B"], **p)
        assert np.array_equal(mp, z["maps"][k]), (path, k)
        assert (n, cnt, mixed) == (int(z["n"][k]), tuple(z["counts"][k].tolist()), int(z["mixed"][k]))
        assert sel.potential == int(z["pot_after"][k])
        assert n == int((mp != 0).sum())


@pytest.mark.skipif(po.pin() is None, reason="no reference checkout was built (oracle/_ref/libref_pixsel_pin.so)")
@pytest.mark.parametrize("path", FIXTURES, ids=os.path.basename)
def test_reference_matches_fixture(path):
    z = po.load(path)
    ref = po.RefSelector(int(z["w"]), int(z["h"]))
    ref.potential = int(z["pot_before"][0])
    for k, img, p in _calls(z):
        mp, n = ref.make_maps(img, z["B"], **p)
        assert np.array_equal(mp, z["maps"][k].astype(np.float32)) and n == int(z["n"][k]) and ref.potential == int(z["pot_after"][k])


@pytest.mark.parametrize("w,h", [(640, 480), (1232, 368), (33, 20)])
def test_random_pattern_is_the_references(w, h):
    got = capi.pixsel_pattern(w * h)
    assert np.array_equal(got, po.Selector(w, h).pattern())
    if po.pin() is not None:
        assert np.array_equal(got, po.RefSelector(w, h).pattern())
    # generating it leaves the process's rand() sequence alone
    libc = C.CDLL(None)
    libc.srand(7)
    a = [libc.rand() for _ in range(4)]
    libc.srand(7)
    libc.rand()
    capi.pixsel_pattern(1000)
    assert [libc.rand() for _ in range(3)] == a[1:]


def test_unwritten_thresholds_read_zero():
    # 1232 x 368: 38 x 11 written cells; a pixel in columns 1216.. reads the next row's first cell, one in rows 352.. reads past the end
    w, h = 1232, 368
    sel = po.Selector(w, h)
    _, ths = sel.set_frame(co.render(w, h, 3))
    w32, h32 = w // 32, h // 32
    assert ths.size == w32 * h32 and np.all(ths > 0)
    assert sel.th(1220, 40) == ths[38 + 1 * w32] == ths[0 + 2 * w32]        # (1220>>5) + (40>>5)*38 = 76
    assert sel.th(100, 300) == ths[3 + 9 * w32]
    assert sel.th(1226, 364) == 0.0                                          # index 38 + 11*38 = 456 >= 418


def test_unwritten_gradient_rows_are_zero():
    w, h = 640, 480
    img = po.image("steps", w, h, 4) + co.render(w, h, 4)
    sel = po.Selector(w, h)
    ag, _ = sel.set_frame(img)
    for a in ag:
        assert np.all(a[0] == 0) and np.all(a[-1] == 0) and (a[1:-1] != 0).any()
    # select() reads level 2 at row (int)(yf*0.25f + 0.125) = 119 = h2-1 for yf = h-4
    assert int(np.float32(h - 4) * np.float32(0.25) + 0.125) == (h >> 2) - 1
    if po.pin() is not None:          # the pin zeroes those rows in the reference's own arrays: both sides agree on such an image
        r = po.RefSelector(w, h)
        mp, n = r.make_maps(img)
        mo, no, _, _ = sel.make_maps(img)
        assert n == no and np.array_equal(mp, mo.astype(np.float32))


def test_pixsel_structs_match_the_header(tmp_path):
    pairs = [("ldso_b200_pixsel_params", capi.PixselParamsC), ("ldso_b200_pixels", capi.PixelsC),
             ("ldso_b200_pixel_traces", capi.PixelTracesC)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "ldso_b200.h"', 'int main(void) {']
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
    for cname, cls in pairs:
        assert int(got[cname]) == C.sizeof(cls), (cname, got[cname], C.sizeof(cls))
        for fname, *_ in cls._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(cls, fname).offset, (cname, fname)

"""Regenerate tests/golden/undistort_*.npz from the undistortion pin (oracle/_ref/pin_undistort, built by __graft_entry__.build()
where a reference checkout exists). The pin compares the restatement (oracle/undistort.cc) with the reference's own
Undistort::undistort<T> bit for bit and fails on any difference; the fixtures hold what it ran:

  undistort_tables.npz     the raw 8- and 16-bit frames, and the tables the reference built from the pin's files: G of the 256- and the
                           65536-entry gamma file (G256, G65536), vignetteMapInv of the 8- and the 16-bit vignette image
  undistort_<camera>.npz   remapX / remapY of one camera (none without rectification), and per case its settings and the restatement's
                           image (equal to the reference's at every pixel that does not read past the end of the raw frame; `past`
                           marks those pixels)

    python tests/golden/make_undistort_golden.py
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PIN = os.path.join(ROOT, "oracle", "_ref", "pin_undistort")

CASE_DTYPE = np.dtype([("name", "U16"), ("w", "<i4"), ("h", "<i4"), ("wOrg", "<i4"), ("hOrg", "<i4"), ("passthrough", "<i4"),
                       ("g_entries", "<i4"), ("mode", "<i4"), ("use_exposure", "<i4"), ("bpp", "<i4"), ("exposure", "<f4"),
                       ("factor", "<f4"), ("exposure_out", "<f4"), ("excluded", "<i4")])


def main():
    if not os.path.exists(PIN):
        sys.exit(f"{PIN} is missing: build it with a reference checkout present (__graft_entry__.build())")
    with tempfile.TemporaryDirectory() as d:
        subprocess.run([PIN, d], check=True, stdout=subprocess.DEVNULL)
        rd = lambda name, dt: np.fromfile(os.path.join(d, name), dt)  # noqa: E731
        rows = [l.split() for l in open(os.path.join(d, "manifest.txt"))]
        tables = {"raw8": rd("raw8.bin", np.uint8), "raw16": rd("raw16.bin", np.uint16)}
        cams = {}
        for r in rows:
            cam, case = r[0], r[1]
            w, h, wOrg, hOrg, pt, g, mode, use_exp, bpp = map(int, r[2:11])
            exposure, factor, e_out = map(np.float32, r[11:14])
            stem = f"{cam}.{case}"
            if g:       # one G per gamma file and one vignetteMapInv per vignette image, whatever the camera
                # mode 0: the constructor replaces G by a linear ramp, which processFrame never reads (the factor path)
                found = [(f"vinv{8 if g == 256 else 16}", rd(stem + ".vinv.bin", np.float32))]
                if mode:
                    found.append((f"G{g}", rd(stem + ".G.bin", np.float32)))
                for key, arr in found:
                    if key in tables:
                        assert np.array_equal(tables[key].view(np.uint32), arr.view(np.uint32)), (key, stem)
                    tables[key] = arr
            c = cams.setdefault(cam, {"cases": [], "arrays": {}})
            if not pt and "remapX" not in c["arrays"]:
                c["arrays"]["remapX"] = rd(stem + ".remapX.bin", np.float32).reshape(h, w)
                c["arrays"]["remapY"] = rd(stem + ".remapY.bin", np.float32).reshape(h, w)
            c["arrays"]["out_" + case] = rd(stem + ".out.bin", np.float32).reshape(h, w)
            c["arrays"]["past_" + case] = rd(stem + ".past.bin", np.uint8).reshape(h, w)
            c["cases"].append((case, w, h, wOrg, hOrg, pt, g, mode, use_exp, bpp, exposure, factor, e_out, int(r[14])))
    tables["raw8"] = tables["raw8"].reshape(hOrg, wOrg)
    tables["raw16"] = tables["raw16"].reshape(hOrg, wOrg)
    tables["vinv8"] = tables["vinv8"].reshape(hOrg, wOrg)
    tables["vinv16"] = tables["vinv16"].reshape(hOrg, wOrg)
    np.savez_compressed(os.path.join(HERE, "undistort_tables.npz"), **tables)
    for cam, c in cams.items():
        np.savez_compressed(os.path.join(HERE, f"undistort_{cam}.npz"), cases=np.array(c["cases"], CASE_DTYPE), **c["arrays"])
    print("wrote", len(cams) + 1, "fixtures")


if __name__ == "__main__":
    main()

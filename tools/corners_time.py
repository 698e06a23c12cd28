"""Time one keyframe's corner detection at 640x480 and 1500 features (setting_desiredImmatureDensity):

  device     ldso_b200_detect_corners on a resident slot: the four kernels, the one read-back copy and the synchronise
  reference  the reference's own FeatureDetector::DetectCorners on one CPU core (oracle/_ref/libref_corners.so, the reference's Release
             flags), on a frame whose pyramid is already built, as in FullSystem::makeNewTraces

Both are timed by the host clock; the two alternate in rounds, and the medians over --runs rounds are reported (the reference side
is the median of 5 calls per round). Needs a GPU and oracle/_ref/libref_corners.so (built by __graft_entry__.build() where a reference
checkout exists). Prints one JSON line.

    python tools/corners_time.py [--runs 30]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ldso_b200 import capi  # noqa: E402
from tests import corners_oracle as co  # noqa: E402

REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_corners.so")
W, H, NF = 640, 480, 1500


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("corners_time.py needs a GPU")
    if not os.path.exists(REF_LIB):
        sys.exit(f"{REF_LIB} is missing: run __graft_entry__.build() where a reference checkout exists")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)
    L = C.CDLL(REF_LIB)
    L.cref_time.restype = C.c_double
    L.cref_time.argtypes = [C.c_int, C.c_int, co.c_fp, co.c_fp, C.c_int, C.c_int, C.c_int]
    L.cref_pattern.argtypes = [co.c_ip]
    pat = np.zeros(1024, np.int32)
    L.cref_pattern(pat.ctypes.data_as(co.c_ip))
    img = co.render(W, H, 1)
    ctx = capi.Context(W, H, 4)
    ctx.set_orb_pattern(pat)
    ctx.make_images(0, img)
    for _ in range(5):
        ctx.detect_corners(0, NF)
    dev, ref = [], []
    for _ in range(args.runs):
        t0 = time.perf_counter()
        ctx.detect_corners(0, NF)
        dev.append(time.perf_counter() - t0)
        ref.append(L.cref_time(W, H, img.ctypes.data_as(co.c_fp), None, NF, 1, 5))
    ctx.close()
    md, mr = float(np.median(dev)) * 1e3, float(np.median(ref)) * 1e3
    print(json.dumps({"card": card, "geometry": f"{W}x{H}, {NF} features", "unit": "ms per keyframe (median)", "runs": args.runs,
                      "device": round(md, 4), "reference_1core": round(mr, 4), "speedup": round(mr / md, 2)}))


if __name__ == "__main__":
    main()

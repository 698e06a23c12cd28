"""Time one keyframe's DSO point selection (setting_pointSelection = 0) at 640x480 and density 1500 (setting_desiredImmatureDensity):

  device  ldso_b200_make_new_traces_pixels on a resident slot: makeMaps on the device, then the ImmaturePoint constructor of every
          feature into the slot's segment, ending with the read-back and the synchronise
  host    the path without it: download levels 0-2 of the pyramid (download_frame_level), the reference's own makeMaps on one CPU core
          (oracle/_ref/libref_pixsel.so, the reference's Release flags; the histogram is made in every call, as for each new keyframe),
          then immature_seed with the selected coordinates

All legs are timed by the host clock around calls that end in a synchronise; they alternate in rounds, and the medians over --runs
rounds are reported (the reference's makeMaps is the median of 5 calls per round). Prints the card's name and power limit in the same
run, as one JSON line. Needs a GPU and oracle/_ref/libref_pixsel.so (built by __graft_entry__.build() where a reference checkout exists).

    python tools/pixsel_time.py [--runs 30]
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
from tests import pixsel_oracle as po  # noqa: E402

W, H, DENSITY = 640, 480, 1500.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("pixsel_time.py needs a GPU")
    L = po.pin(po.FAST_LIB)
    if L is None:
        sys.exit(f"{po.FAST_LIB} is missing: run __graft_entry__.build() where a reference checkout exists")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)
    img = co.render(W, H, 1)
    ctx = capi.Context(W, H, 4)
    ctx.make_images(0, img)
    ctx.make_images(1, img)
    params = capi.pixsel_params(density=DENSITY)
    pot = 3
    for _ in range(5):
        pot = ctx.make_new_traces_pixels(0, params, current_potential=pot)["current_potential"]
    sel = ctx.select_pixels(0, params, current_potential=3)
    mp = np.zeros((H, W), np.uint8)
    mp[sel["y"], sel["x"]] = sel["type"]
    y, x = np.nonzero(mp)
    k = (x >= 3) & (x < W - 4) & (y >= 3) & (y < H - 4)
    u, v, t = x[k].astype(np.float32), y[k].astype(np.float32), mp[y[k], x[k]].astype(np.float32)
    n_ref = C.c_int(0)
    dev, down, ref, seed = [], [], [], []
    for _ in range(args.runs):
        t0 = time.perf_counter()
        out = ctx.make_new_traces_pixels(0, params, current_potential=pot)
        dev.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        for lvl in range(3):
            ctx.download_frame_level(0, lvl)
        down.append(time.perf_counter() - t0)
        ref.append(L.cref_pixsel_time(W, H, img.ctypes.data_as(po.c_fp), None, DENSITY, 1, 5, C.byref(n_ref)))
        t0 = time.perf_counter()
        ctx.immature_seed(1, u, v, t)
        seed.append(time.perf_counter() - t0)
    ctx.close()
    ms = lambda a: round(float(np.median(a)) * 1e3, 4)
    host = ms(down) + ms(ref) + ms(seed)
    print(json.dumps({"card": card, "geometry": f"{W}x{H}, density {DENSITY:g}", "unit": "ms per keyframe (median)", "runs": args.runs,
                      "features": int(out["n"]), "selected_device": int(out["n_selected"]), "selected_reference": int(n_ref.value),
                      "device": ms(dev), "host_download": ms(down), "host_reference_makeMaps_1core": ms(ref), "host_immature_seed": ms(seed),
                      "host_total": round(host, 4), "speedup": round(host / ms(dev), 2)}))


if __name__ == "__main__":
    main()

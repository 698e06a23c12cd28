"""Time one raw camera frame's way into a keyframe pyramid, TUM-mono geometry (1280x1024 raw -> 640x480 rectified, RadTan crop,
photometric mode 2), for 8- and 16-bit frames:

  device     ldso_b200_undistort_frame: raw upload, the fused photometric + geometric kernel, makeImages on the device
  host       the reference's own Undistort::undistort<T> on the CPU (oracle/_ref/libref_undistort.so, the reference's Release flags),
             then ldso_b200_make_images of its float image: the path a caller takes without this feature
  host_only  Undistort::undistort<T> alone

Each call is timed by the host clock around work that ends in a device synchronise. Cold: the L2 is flushed (a 256 MB write)
before every call; warm: back-to-back calls. The forms alternate; medians over --runs calls are reported. Needs a GPU and
oracle/_ref/libref_undistort.so (built by __graft_entry__.build() where a reference checkout exists).

    python tools/undistort_time.py [--runs 50]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ldso_b200 import capi  # noqa: E402

REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_undistort.so")
WORG, HORG, W, H, LEVELS = 1280, 1024, 640, 480, 4


def ref_lib():
    if not os.path.exists(REF_LIB):
        sys.exit(f"{REF_LIB} is missing: run __graft_entry__.build() where a reference checkout exists")
    L = C.CDLL(REF_LIB)
    L.uref_open.restype = C.c_void_p
    L.uref_open.argtypes = [C.c_char_p] + [C.c_int] * 9
    L.uref_tables.argtypes = [C.c_void_p] + [C.c_void_p] * 6
    L.uref_undistort.restype = C.c_float
    L.uref_undistort.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_void_p]
    L.uref_close.argtypes = [C.c_void_p]
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("undistort_time.py needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    L = ref_lib()
    rng = np.random.default_rng(1)
    out = {"card": card, "runs": args.runs, "geometry": f"{WORG}x{HORG} -> {W}x{H}, RadTan crop, mode 2, {LEVELS} levels",
           "unit": "ms per frame (median)"}
    with tempfile.TemporaryDirectory() as d:
        for bpp, gamma in ((1, 256), (2, 65536)):
            u = L.uref_open(d.encode(), 1, 0, WORG, HORG, W, H, gamma, 2, 1)
            wh = np.zeros(4, np.int32)
            rx, ry = np.zeros(W * H, np.float32), np.zeros(W * H, np.float32)
            G, vinv, ge = np.zeros(65536, np.float32), np.zeros(WORG * HORG, np.float32), C.c_int(0)
            L.uref_tables(u, wh.ctypes.data, rx.ctypes.data, ry.ctypes.data, G.ctypes.data, vinv.ctypes.data, C.addressof(ge))
            raw = rng.integers(0, 256 if bpp == 1 else 65536, (HORG, WORG)).astype(np.uint8 if bpp == 1 else np.uint16)
            img = np.zeros((H, W), np.float32)
            ctx = capi.Context(W, H, LEVELS)
            ctx.set_undistort(WORG, HORG, rx, ry, G[:ge.value], vinv, 2, True)

            def host_only():
                L.uref_undistort(u, raw.ctypes.data, bpp, 1.0, 1.0, img.ctypes.data)

            def host():
                host_only()
                ctx.make_images(1, img)
                ctx.synchronize()

            def device():
                ctx.undistort_frame(0, raw, 1.0, 1.0)
                ctx.synchronize()
            forms = {"device": device, "host": host, "host_only": host_only}
            for f in forms.values():
                f(), f()
            res = {}
            for cold in (True, False):
                times = {k: [] for k in forms}
                order = list(forms)
                for i in range(args.runs):
                    for k in order[i % 3:] + order[:i % 3]:
                        if cold:
                            flush.fill_(float(i))
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        forms[k]()
                        times[k].append(1e3 * (time.perf_counter() - t0))
                res["cold_l2" if cold else "warm_l2"] = {k: round(float(np.median(v)), 4) for k, v in times.items()}
            # the device's level 0 against the reference's image (Release build: contraction may move the last bit)
            ctx.undistort_frame(0, raw, 1.0, 1.0)
            host_only()
            got = ctx.download_frame_level(0, 0)[..., 0]
            res["max_abs_diff_vs_reference_release_build"] = float(np.abs(got - img).max())
            out[f"{8 * bpp}bit"] = res
            ctx.close()
            L.uref_close(u)
    C.CDLL(None).fflush(None)      # the reference's own progress messages go to C's stdout buffer: out of the way of the result line
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

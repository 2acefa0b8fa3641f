"""GPU timing of NL-means (b2f_nlmeans_dev) for every row of the reference's parameter table on 1920x1080 and 3840x2160
u8 frames (device-resident, CUDA events after warm-up), next to the serial reference (oracle/_ref, one host thread) on a
crop.  Prints the card and its power limit first, then one JSON line per (table row, size).

    python tools/nlmeans_timing.py [--reps 3] [--crop 96x64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from image_b200 import synth  # noqa: E402
from image_b200.nlmeans import nlmeans_dev, nlmeans_resolve  # noqa: E402
from oracle import ref_nlmeans as rn  # noqa: E402

ROWS = [(1, 10.0), (1, 20.0), (1, 40.0), (1, 60.0), (1, 90.0), (3, 10.0), (3, 40.0), (3, 80.0)]   # one sigma per table row
SIZES = [(1920, 1080), (3840, 2160)]


def flop_per_pixel(c, win, bloc):
    """Float operations per interior centre: per candidate the distance (sub, mul, add per patch value, one add per
    channel), offset, max, division and interpolation (~8), and the weighted sums (mul, add per patch value); then the
    centre's own patch, the division of the patch by the total and the per-pixel gather (one add per term)."""
    e = c * (2 * win + 1) ** 2
    k = (2 * bloc + 1) ** 2 - 1
    return k * (3 * e + c + 8 + 2 * e) + 2 * e + e + e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--crop", default="96x64")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": q}), flush=True)
    cw, ch = (int(v) for v in a.crop.split("x"))
    st = torch.cuda.Stream()                                                 # the events and the calls share this stream
    for w, h in SIZES:
        rgb = synth.frame_rgb(900, h, w)
        for c, sigma in ROWS:
            win, bloc, filt = nlmeans_resolve(c, sigma)
            planes = rgb.transpose(2, 0, 1)[:c].astype(np.float64)
            img = np.clip(np.rint(planes + np.random.default_rng(901).normal(0, sigma, planes.shape)), 0, 255).astype(np.uint8)
            d = torch.from_numpy(img).cuda()
            out = torch.empty((c, h, w), dtype=torch.float32, device="cuda")
            nlmeans_dev(d, 1, c, w, h, win, bloc, sigma, filt, out, stream=st.cuda_stream)   # warm-up (module load, arena, LUT)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(a.reps):
                nlmeans_dev(d, 1, c, w, h, win, bloc, sigma, filt, out, stream=st.cuda_stream)
            e1.record(st)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            fpp = flop_per_pixel(c, win, bloc)
            rec = {"channels": c, "sigma": sigma, "win": win, "bloc": bloc, "width": w, "height": h, "ms_per_frame": round(ms, 3),
                   "mpix_s": round(w * h / (ms * 1e-3) / 1e6, 2), "flop_per_pixel": fpp,
                   "tflop_s": round(fpp * w * h / (ms * 1e-3) / 1e12, 2)}
            if w == SIZES[0][0] and rn.have_ref():                 # the serial reference on a crop, once per row
                crop = img[:, :ch, :cw].astype(np.int32)
                t0 = time.perf_counter()
                rn.nlmeans(crop.ravel(), cw, ch, c, sigma)
                rec["reference_serial_crop"] = "%dx%d" % (cw, ch)
                rec["reference_serial_mpix_s"] = round(cw * ch / (time.perf_counter() - t0) / 1e6, 5)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()

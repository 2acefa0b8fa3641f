"""GPU timing of darknet (tiny-yolo-voc detection at 416, the tiny classifier at 224-min) at batch 1, 16 and 64: device-
resident (b2f_darknet_*_dev, frames already in HBM) and end to end (b2f_darknet_*_batch_rgb from host memory), wall
clock around calls that return only when their host outputs are written.  Multiply-adds are counted from the layer
shapes; GFLOP/s counts two flops per multiply-add.  The share of the SIMT bound uses half the H100 SXM data sheet's
67 TFLOP/s FP32 rate: the exact-order sum does a separate multiply and add, two instructions where an FMA would be one.
Per-layer kernel times (--profile) come from torch.profiler in a separate run, one row per launch in layer order, and the reference (oracle/_ref, network_predict) on
the host with one thread.  Prints the card, its power limit and SM clock first, then one JSON line per measurement.

    python tools/darknet_timing.py [--reps 10] [--out timing.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from image_b200 import darknet as dn  # noqa: E402
from oracle import ref_darknet as rd  # noqa: E402

SIMT_BOUND_TFLOPS = 67.0 / 2


def layer_macs(net, w, h):
    """Multiply-adds of each GPU layer of net at a w x h input (the geometry of darknet's parser; 0 for the pools)."""
    c, macs = 3, []
    for L in net["layers"]:
        if L["type"] == dn.B2F_DN_CONV:
            oh = (h + 2 * L["pad"] - L["size"]) // L["stride"] + 1
            ow = (w + 2 * L["pad"] - L["size"]) // L["stride"] + 1
            macs.append(ow * oh * L["filters"] * c * L["size"] * L["size"])
            c, h, w = L["filters"], oh, ow
        elif L["type"] == dn.B2F_DN_MAXPOOL:
            h, w = (h + 2 * L["pad"]) // L["stride"], (w + 2 * L["pad"]) // L["stride"]
            macs.append(0)
        elif L["type"] == dn.B2F_DN_AVGPOOL:
            h = w = 1
            macs.append(0)
    return macs


def conv_macs(net, w, h):
    """Multiply-adds of every convolution of net at a w x h input."""
    return sum(layer_macs(net, w, h))


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return float(np.median(ts))


def reference_ms(cfg, weights, name, mode):
    code = ("import sys,time; sys.path.insert(0, %r); from oracle import ref_darknet as rd; rd.load(%r, %r); "
            "im=rd.decode(%r); t=time.perf_counter(); rd.forward(im, %d); print((time.perf_counter()-t)*1e3)"
            % (ROOT, cfg, weights, name, mode))
    env = dict(os.environ, OMP_NUM_THREADS="1")
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True).stdout.split()
    return float(out[-1]) if out else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true", help="per-layer kernel times from torch.profiler instead")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    if not torch.cuda.is_available():
        raise SystemExit("no GPU: nothing measured")
    rows = []
    im = rd.decode("dog.jpg")
    models = [("detect", "tiny-yolo-voc.cfg", "tiny-yolo-voc.weights"), ("classify", "tiny.cfg", "tiny.weights")]
    for kind, cfg, wts in models:
        m = dn.load_network(rd.path(cfg), rd.path(wts))
        if kind == "detect":
            w, h = m.net["w"], m.net["h"]
        else:
            w, h = (im.shape[1] * m.net["w"] // im.shape[0], m.net["w"]) if im.shape[1] >= im.shape[0] else (m.net["w"], im.shape[0] * m.net["w"] // im.shape[1])
        macs = conv_macs(m.net, w, h)
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            frames = np.ascontiguousarray(np.broadcast_to(im, (16,) + im.shape))
            d = torch.from_numpy(frames).cuda()
            run = (lambda: dn.detect_dev(d, 16, im.shape[1], im.shape[0], m)) if kind == "detect" else \
                (lambda: dn.classify_dev(d, 16, im.shape[1], im.shape[0], m, True, 5))
            run()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
            # one launch per GPU layer after the ingest, in layer order: the kernels in launch order are the layers
            kern = sorted((e for e in prof.events() if "b2f::dn_" in e.name), key=lambda e: e.time_range.start)
            names = ["ingest"] + ["%d %s" % (i, L["name"]) for i, L in enumerate(m.net["layers"])
                                  if L["type"] in (dn.B2F_DN_CONV, dn.B2F_DN_MAXPOOL, dn.B2F_DN_AVGPOOL)]
            lmacs = [0] + layer_macs(m.net, w, h)
            for name, e, mac in zip(names, kern, lmacs):
                us = e.time_range.elapsed_us()
                r = dict(model=cfg, kind=kind, batch=16, layer=name, kernel=e.name.split("(")[0], us=round(us, 1),
                         gmacs=round(mac * 16 / 1e9, 3), gflops=round(2.0 * mac * 16 / us / 1e3, 1) if mac else None)
                rows.append(r)
                print(json.dumps(r))
            m.free()
            continue
        for n in (1, 16, 64):
            frames = np.ascontiguousarray(np.broadcast_to(im, (n,) + im.shape))
            d = torch.from_numpy(frames).cuda()
            if kind == "detect":
                t_dev = timed(lambda: dn.detect_dev(d, n, im.shape[1], im.shape[0], m), args.reps)
                t_e2e = timed(lambda: dn.detect_batch(frames, m), args.reps)
            else:
                t_dev = timed(lambda: dn.classify_dev(d, n, im.shape[1], im.shape[0], m, True, 5), args.reps)
                t_e2e = timed(lambda: dn.classify_batch(frames, m, True, 5), args.reps)
            for what, t in (("device", t_dev), ("end_to_end", t_e2e)):
                gflops = 2.0 * macs * n / t / 1e9
                r = dict(model=cfg, kind=kind, input="%dx%d" % (w, h), batch=n, form=what, ms_per_call=round(t * 1e3, 3),
                         ms_per_frame=round(t * 1e3 / n, 3), frames_per_s=round(n / t, 1), gmacs_per_frame=round(macs / 1e9, 3),
                         gflops=round(gflops, 1), simt_bound_share=round(gflops / (SIMT_BOUND_TFLOPS * 1e3), 3), card=card)
                rows.append(r)
                print(json.dumps(r))
        ref = reference_ms(rd.path(cfg), rd.path(wts), "dog.jpg", 0 if kind == "detect" else 1)
        r = dict(model=cfg, kind=kind, form="reference_1_thread", ms_per_frame=ref)
        rows.append(r)
        print(json.dumps(r))
        m.free()
    if args.out:
        mode = "a" if args.profile else "w"
        with open(args.out, mode) as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()

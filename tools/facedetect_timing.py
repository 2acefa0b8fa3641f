"""GPU timing of face detection (b2f_facedet_dev, b2f_facedet_batch_rgb) on 1024x683, 1920x1080 and 3840x2160 frames at
batch 1 and 16, CUDA events after warm-up; the per-layer kernel times of one 4K frame from torch.profiler; int8
multiply-adds counted from the layer shapes, achieved TOPS and the share of the H100 SXM data sheet's dense INT8 rate
(1,979 TOPS); and the reference (oracle/_ref, facedetect_cnn) on the host with one thread and with all cores.  Prints the
card, its power limit and SM clock first, then one JSON line per measurement.

    python tools/facedetect_timing.py [--reps 5] [--out timing.jsonl]
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
from image_b200.facedetect import facedetect_batch, facedetect_dev, load_model  # noqa: E402
from oracle import ref_facedetect as rf  # noqa: E402

SIZES = [(1024, 683), (1920, 1080), (3840, 2160)]
SHAPES = [(3, 3, 32), (1, 32, 16), (3, 16, 32), (1, 32, 32), (3, 32, 64), (1, 64, 32), (3, 32, 64), (3, 64, 128),
          (1, 128, 64), (3, 64, 128), (3, 128, 256), (1, 256, 128), (3, 128, 256), (3, 256, 256), (1, 256, 256),
          (3, 256, 256)]
POOL_AFTER = (1, 3, 6, 9, 12)
HEADS = [(6, 48), (9, 32), (12, 32), (15, 48)]       # source layer, loc + conf channels
PEAK_INT8_TOPS = 1979.0                              # H100 SXM data sheet, dense


def layer_macs(w, h):
    """int8 multiply-adds of each convolution (16 trunk layers, then the 4 fused heads) of one w x h frame."""
    lw, lh = (w + 1) // 2, (h + 1) // 2
    dims, macs = [], []
    for l, (k, c, n) in enumerate(SHAPES):
        dims.append((lw, lh))
        macs.append(lw * lh * n * k * k * c)
        if l in POOL_AFTER:
            lw, lh = lw // 2, lh // 2
    for s, n in HEADS:
        macs.append(dims[s][0] * dims[s][1] * n * 9 * SHAPES[s][2])
    return macs


def frame(w, h):
    base = np.load(os.path.join(ROOT, "tests", "golden", "facedetect_handshake.npz"))["rgb"]
    ry, rx = -(-h // base.shape[0]), -(-w // base.shape[1])
    return np.ascontiguousarray(np.tile(base, (ry, rx, 1))[:h, :w])


def reference_ms(fr, threads):
    code = ("import sys,time,numpy as np; sys.path.insert(0, %r); from oracle import ref_facedetect as rf; "
            "a=np.load(sys.argv[1]); rf.facedetect_cnn(a); t=time.perf_counter(); rf.facedetect_cnn(a); "
            "print((time.perf_counter()-t)*1e3)" % ROOT)
    path = os.path.join("/tmp", "fd_timing_frame_%d.npy" % os.getpid())
    np.save(path, fr)
    env = dict(os.environ)
    if threads:
        env["OMP_NUM_THREADS"] = str(threads)
    try:
        return float(subprocess.run([sys.executable, "-c", code, path], env=env, capture_output=True, text=True, check=True).stdout)
    finally:
        os.remove(path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    lines = []

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    emit({"device": torch.cuda.get_device_name(0), "nvidia_smi": q, "host_cpus": os.cpu_count()})
    model = load_model(rf.SO_PATH)
    st = torch.cuda.Stream()
    for w, h in SIZES:
        fr = frame(w, h)
        macs = sum(layer_macs(w, h))
        for n in (1, 16):
            host = np.ascontiguousarray(np.broadcast_to(fr, (n, h, w, 3)))
            d = torch.from_numpy(host).cuda()
            facedetect_dev(d, n, w, h, model, stream=st.cuda_stream)           # warm-up: modules, arena
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            for _ in range(a.reps):
                facedetect_dev(d, n, w, h, model, stream=st.cuda_stream)
            e1.record(st)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / a.reps
            facedetect_batch(host, model)
            t0 = time.perf_counter()
            for _ in range(a.reps):
                facedetect_batch(host, model)
            e2e = (time.perf_counter() - t0) * 1e3 / a.reps
            tops = 2.0 * macs * n / (ms * 1e-3) / 1e12
            emit({"width": w, "height": h, "batch": n, "gmacs_per_frame": round(macs / 1e9, 3),
                  "device_resident_ms_per_frame": round(ms / n, 3), "frames_s_device": round(n / (ms * 1e-3), 1),
                  "end_to_end_ms_per_frame": round(e2e / n, 3), "frames_s_end_to_end": round(n / (e2e * 1e-3), 1),
                  "achieved_int8_tops_whole_call": round(tops, 1), "share_of_dense_int8_peak": round(tops / PEAK_INT8_TOPS, 4)})
    # per-layer kernel times of one 4K frame (profiled in a run of its own)
    w, h = SIZES[-1]
    d = torch.from_numpy(frame(w, h)[None].copy()).cuda()
    facedetect_dev(d, 1, w, h, model)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        facedetect_dev(d, 1, w, h, model)
        torch.cuda.synchronize()
    kern = sorted([e for e in prof.events() if e.device_type.name == "CUDA" and "fd_" in e.name], key=lambda e: e.time_range.start)
    macs = layer_macs(w, h)
    layers, cur = [], None
    for e in kern:
        if "fd_conv" in e.name:
            cur = {"conv_us": e.time_range.elapsed_us(), "other_us": 0.0}
            layers.append(cur)
        elif cur is not None:
            cur["other_us"] += e.time_range.elapsed_us()
    names = ["L%d" % l for l in range(16)] + ["heads@L6", "heads@L9", "heads@L12", "heads@L15"]
    for name, lay, m in zip(names, layers, macs):
        t = lay["conv_us"] * 1e-6
        tops = 2.0 * m / t / 1e12 if t > 0 else 0.0
        emit({"layer": name, "width": w, "height": h, "conv_us": round(lay["conv_us"], 1),
              "requant_scalars_cand_us": round(lay["other_us"], 1), "gmacs": round(m / 1e9, 3), "int8_tops": round(tops, 1),
              "share_of_dense_int8_peak": round(tops / PEAK_INT8_TOPS, 4)})
    emit({"profiled_kernels_total_us": round(sum(e.time_range.elapsed_us() for e in kern), 1)})
    model.free()
    for w, h in (SIZES[0], SIZES[-1]):
        fr = frame(w, h)
        for threads in (1, 0):
            emit({"reference_facedetect_cnn": "%dx%d" % (w, h), "threads": threads or os.cpu_count(),
                  "ms": round(reference_ms(fr, threads), 1)})
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()

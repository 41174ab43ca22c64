#!/usr/bin/env python
"""bench_mono.py -- RGB24 vs mono8 input on the default bench configuration (752x480 EuRoC parameters, UseUndistort=1 with
the EuRoC rad-tan coefficients, 64-frame batches, the seed-7 stream of bench.py).

A mono frame m stands for the RGB24 frame (m, m, m), so both formats must produce the same nav records; the synthetic
stream is gray replicated into three channels, and its mono frames are the first channel.  In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - RGB and mono runs in alternating pairs (the order flips from pair to pair), each with frames resident in device memory
    (rb_pipeline_push_dev / _mono_dev) and with pinned host buffers (rb_pipeline_push / _mono), allocated as bench.py
    allocates them; median, min and max of frames/s per arm and the per-pair mono / RGB ratio;
  - per-pass CUDA-event time and effective bandwidth (algorithmic bytes / time) of the gray passes: 4 / 5 (RGB, RGB with
    undistortion) against 6 / 7 (mono, mono with undistortion);
  - whether the nav records of the two formats are byte-identical in every pair (exit status 1 if not).

Prints one JSON line (and writes it to --out if given).  Needs a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info(dev):
    import torch
    info = {"name": torch.cuda.get_device_name(dev), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=60).stdout.strip().split(", ")
        if len(out) == 2:
            info = {"name": out[0], "power_limit_w": float(out[1])}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        pass
    return info


def stats(v):
    v = np.asarray(v, np.float64)
    med = float(np.median(v))
    return {"median": med, "min": float(v.min()), "max": float(v.max()), "spread": float((v.max() - v.min()) / med),
            "runs": [float(x) for x in v]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=7, help="alternating RGB / mono pairs per input location (at least 5)")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--pass-iters", type=int, default=50)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.pairs < 5:
        ap.error("--pairs must be at least 5")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_mono.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    B, K, W = args.batch, args.steps, args.warmup
    total = B * (K + W)
    cam, params, _, _, seed0 = bench.stream_setup(2)
    kc = bench.undistort_of(2)
    ts, base, idx = bench.make_stream(seed0, total, cam=cam)
    h, w = cam["h"], cam["w"]
    N = h * w
    frames = base[idx]
    assert np.array_equal(frames[..., 0], frames[..., 1]) and np.array_equal(frames[..., 0], frames[..., 2])
    host = {"rgb": torch.empty((total, h, w, 3), dtype=torch.uint8, pin_memory=True),
            "mono": torch.empty((total, h, w), dtype=torch.uint8, pin_memory=True)}
    host["rgb"].numpy()[:] = frames
    host["mono"].numpy()[:] = frames[..., 0]
    devbuf = {k: v.to("cuda:%d" % dev) for k, v in host.items()}
    torch.cuda.synchronize()

    def run(fmt, where):
        pl = capi.Pipeline(params, max_batch=B, device=dev)
        pl.set_undistort(kc)
        buf = devbuf[fmt] if where == "resident" else host[fmt]
        push = {("rgb", "resident"): pl.push_dev, ("rgb", "host"): pl.push,
                ("mono", "resident"): pl.push_mono_dev, ("mono", "host"): pl.push_mono}[(fmt, where)]
        navs = [push(buf[s * B].data_ptr(), ts[s * B:(s + 1) * B]) for s in range(W)]
        torch.cuda.synchronize()
        pl.event_record(0)
        for s in range(W, W + K):
            navs.append(push(buf[s * B].data_ptr(), ts[s * B:(s + 1) * B]))
        pl.event_record(1)
        ms = pl.event_elapsed(0, 1)
        pl.close()
        return K * B / (ms * 1e-3), np.concatenate(navs)

    fps = {(f, wh): [] for f in ("rgb", "mono") for wh in ("resident", "host")}
    ratio = {"resident": [], "host": []}
    identical = True
    first_diff = None
    for p in range(args.pairs):
        for where in ("resident", "host"):
            order = ("rgb", "mono") if p % 2 == 0 else ("mono", "rgb")
            got = {}
            for fmt in order:
                got[fmt] = run(fmt, where)
                fps[(fmt, where)].append(got[fmt][0])
            ratio[where].append(got["mono"][0] / got["rgb"][0])
            a, b = got["rgb"][1], got["mono"][1]
            same = a.tobytes() == b.tobytes()
            if not same and first_diff is None:
                d = np.nonzero((a.view(np.uint8) != b.view(np.uint8)).reshape(len(a), -1).any(1))[0]
                first_diff = {"pair": p, "input": where, "frame": int(d[0]) if len(d) else None}
            identical = identical and same

    # gray passes over the batched workspace of a pipeline that has run (same batch, same undistortion map)
    pl = capi.Pipeline(params, max_batch=B, device=dev)
    pl.set_undistort(kc)
    pl.push_mono(host["mono"][0].data_ptr(), ts[:B])
    pl.push(host["rgb"][B].data_ptr(), ts[B:2 * B])
    passes = {}
    names = {4: "k_gray<rgb>", 5: "k_undistort_gray<rgb>", 6: "k_gray<mono>", 7: "k_undistort_gray<mono>"}
    for rep in range(3):   # (interleaved, best of three per pass)
        for pid in (4, 6, 5, 7):
            ms, by = pl.bench_pass(pid, B, args.pass_iters)
            q = passes.setdefault(names[pid], {"pass": pid, "bytes_per_launch": by, "ms_per_launch": ms})
            q["ms_per_launch"] = min(q["ms_per_launch"], ms)
    pl.close()
    peak, peak_src = bench.peaks()
    for q in passes.values():
        q["gbs"] = q["bytes_per_launch"] / (q["ms_per_launch"] * 1e-3) / 1e9
        q["frac_of_peak"] = q["gbs"] / peak
        q["us_per_frame"] = 1e3 * q["ms_per_launch"] / B

    out = {"what": "RGB24 vs mono8 input, frames/s (CUDA events over %d steps of %d frames after %d warm-up steps), "
                   "752x480 EuRoC parameters, UseUndistort=1, seed-7 stream" % (K, B, W),
           "gpu": gpu_info(dev), "pairs": args.pairs,
           "resident": {"rgb": stats(fps[("rgb", "resident")]), "mono": stats(fps[("mono", "resident")]),
                        "mono_over_rgb": stats(ratio["resident"])},
           "host": {"rgb": stats(fps[("rgb", "host")]), "mono": stats(fps[("mono", "host")]),
                    "mono_over_rgb": stats(ratio["host"])},
           "h2d_bytes_per_frame": {"rgb": 3 * N, "mono": N},
           "passes": passes, "peak_gbs": peak, "peak_source": peak_src,
           "nav_identical": identical, "first_difference": first_diff}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()

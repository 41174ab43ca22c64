#!/usr/bin/env python
"""bench_width.py -- frames of widths that are not a multiple of 4 (row-pitched scale space, odd-width input pass) against
the 4-aligned neighbour width, at KITTI odometry sizes: 1224x370 (4-aligned), 1226x370 (w = 2 mod 4) and 1241x376
(w = 1 mod 4), default parameters (752x480 EuRoC configuration file values), a seed-7 synthetic stream per width, 64-frame
batches.  In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - frames/s of every (width, input location, format, undistortion) cell: frames resident in device memory
    (rb_pipeline_push_dev / _mono_dev) or in pinned host buffers (rb_pipeline_push / _mono), RGB24 or mono8,
    UseUndistort 0 or 1; the widths alternate within each round and their order rotates from round to round; median, min,
    max and spread per cell, and keylines per frame;
  - per-pass CUDA-event time of rb_pipeline_bench_pass 0..7 at each width (best of three, interleaved), per frame and per
    pixel: the odd widths' gray passes 4 / 6 are the odd-width input kernel, 5 / 7 its undistorting twins.

Prints one JSON line (and writes it to --out if given).  Needs a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

WIDTHS = [(1224, 370), (1226, 370), (1241, 376)]
KC = (-0.12, 0.03, 0.0, 1e-4, 2e-5)   # a mild rad-tan model for the UseUndistort=1 cells
PASSES = {0: "row scan", 1: "row scan + box average", 2: "column scan", 3: "last box + DoG", 4: "rgb -> gray",
          5: "undistort + rgb -> gray", 6: "mono -> gray", 7: "undistort + mono -> gray"}


def cam_of(w, h):
    return dict(w=w, h=h, zfx=718.856, zfy=718.856, ppx=w / 2.0 - 13.3, ppy=h / 2.0 - 2.8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="runs per cell (the widths alternate within a round)")
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--pass-iters", type=int, default=50)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_width.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    B, K, W = args.batch, args.steps, args.warmup
    total = B * (K + W)
    data = {}
    for (w, h) in WIDTHS:
        cam = cam_of(w, h)
        ts, base, idx = bench.make_stream(7, total, base_n=64, cam=cam)
        frames = base[idx]
        host = {"rgb": torch.empty((total, h, w, 3), dtype=torch.uint8, pin_memory=True),
                "mono": torch.empty((total, h, w), dtype=torch.uint8, pin_memory=True)}
        host["rgb"].numpy()[:] = frames
        host["mono"].numpy()[:] = frames[..., 0]
        data[w] = (cam, ts, host, {k: v.to("cuda:%d" % dev) for k, v in host.items()})
    torch.cuda.synchronize()

    def run(w, fmt, where, kc):
        cam, ts, host, devbuf = data[w]
        pl = capi.Pipeline(capi.default_params(cam), max_batch=B, device=dev)
        pl.set_undistort(kc)
        buf = devbuf[fmt] if where == "resident" else host[fmt]
        push = {("rgb", "resident"): pl.push_dev, ("rgb", "host"): pl.push,
                ("mono", "resident"): pl.push_mono_dev, ("mono", "host"): pl.push_mono}[(fmt, where)]
        for s in range(W):
            push(buf[s * B].data_ptr(), ts[s * B:(s + 1) * B])
        torch.cuda.synchronize()
        pl.event_record(0)
        navs = [push(buf[s * B].data_ptr(), ts[s * B:(s + 1) * B]) for s in range(W, W + K)]
        pl.event_record(1)
        ms = pl.event_elapsed(0, 1)
        pl.close()
        nav = np.concatenate(navs)
        return K * B / (ms * 1e-3), float(nav["kn"].mean())

    cells = [(where, fmt, und) for where in ("resident", "host") for fmt in ("rgb", "mono") for und in (0, 1)]
    fps, kn = {}, {}
    for r in range(args.rounds):
        for where, fmt, und in cells:
            order = WIDTHS[r % 3:] + WIDTHS[:r % 3]
            for (w, _) in order:
                f, k = run(w, fmt, where, KC if und else None)
                fps.setdefault((w, where, fmt, und), []).append(f)
                kn[(w, where, fmt, und)] = k

    passes = {}
    for (w, h) in WIDTHS:
        cam, ts, host, _ = data[w]
        pl = capi.Pipeline(capi.default_params(cam), max_batch=B, device=dev)
        pl.set_undistort(KC)
        pl.push(host["rgb"][0].data_ptr(), ts[:B])
        best = {}
        for rep in range(3):
            for pid in PASSES:
                ms, by = pl.bench_pass(pid, B, args.pass_iters)
                best[pid] = min(best.get(pid, ms), ms)
        pl.close()
        passes["%dx%d" % (w, h)] = {str(pid): {"what": PASSES[pid], "ms_per_launch": best[pid],
                                               "us_per_frame": 1e3 * best[pid] / B,
                                               "ps_per_pixel": 1e9 * best[pid] / (B * w * h)} for pid in PASSES}

    res = {}
    for (w, where, fmt, und), v in fps.items():
        res.setdefault("%dx%d" % (w, dict(WIDTHS)[w]), {})["%s %s undistort=%d" % (where, fmt, und)] = dict(
            stats(v), keylines_per_frame=kn[(w, where, fmt, und)])
    out = {"what": "frames/s (CUDA events over %d steps of %d frames after %d warm-up steps) at 1224x370 (4-aligned), "
                   "1226x370 and 1241x376; per-pass times of rb_pipeline_bench_pass 0..7" % (K, B, W),
           "gpu": gpu_info(dev), "rounds": args.rounds, "fps": res, "passes": passes}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

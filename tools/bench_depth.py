#!/usr/bin/env python
"""bench_depth.py -- cost of the per-frame depth grid (rb_pipeline_set_depth, the viewer's depth_filler with its shipped
parameters: 10x10 blocks, ThreshRelRho 1, ThreshMatchNum 5, IterNum 10) at 752x480 with bench.py's configuration-2 parameters
(EuRoC, UseUndistort=1) and at 1280x960 (synthetic camera, no undistortion), frames resident in device memory
(rb_pipeline_push_dev), 64-frame batches.  In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - per size, runs with depth off and on in alternating pairs (the order flips from pair to pair): median, min and max of
    frames/s per arm and the per-pair on / off ratio; a third arm runs the fill's side stream at the tracker's priority
    (REBVO_B200_DEPTH_PRIO=1) instead of the lowest;
  - whether the nav records of the arms are byte-identical in every pair (exit status 1 if not);
  - the time of one rb_depth_fill_net stage call (CUDA events around many calls on one frame's records; each call copies
    the records in and the grid out and synchronises), the device time of its fill kernel alone (torch.profiler), and the
    reference depth_filler's CPU time on the same records (oracle/_ref/libref_depth.so, when it was built);
  - the share of a step with depth on that the batch-end join on the last frame's fill accounts for (one fill kernel time
    per batch, derived from the two measured numbers).

Prints one JSON line (and writes it to --out if given).  Needs a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CAM_1280 = dict(w=1280, h=960, zfx=900.0, zfy=900.0, ppx=640.5, ppy=479.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=7, help="alternating off / on pairs per size (at least 5)")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--calls", type=int, default=200, help="timed rb_depth_fill_net calls per size")
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.pairs < 5:
        ap.error("--pairs must be at least 5")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_depth.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    B, K, W = args.batch, args.steps, args.warmup
    dp = capi.depth_params()
    out = {"what": "depth grid off vs on, frames/s (CUDA events over %d timed steps of %d frames after %d warm-up steps), "
                   "frames resident in device memory; viewer parameters 10x10 / 1 / 5 / 10" % (K, B, W),
           "gpu": gpu_info(dev), "pairs": args.pairs}
    identical = True
    sizes = (("752x480", 2, None), ("1280x960", None, CAM_1280))
    for name, config, cam_over in sizes:
        total = B * (K + W)
        if config is not None:
            cam, params, _, _, seed0 = bench.stream_setup(config)
            kc = bench.undistort_of(config)
            ts, base, idx = bench.make_stream(seed0, total, cam=cam)
        else:
            cam, kc, seed0 = cam_over, None, 7
            params = capi.default_params(cam)
            ts, base, idx = bench.make_stream(seed0, total, base_n=40, cam=cam)
        devbuf = torch.from_numpy(np.ascontiguousarray(base[idx])).to("cuda:%d" % dev)
        torch.cuda.synchronize()

        def run(arm):
            os.environ["REBVO_B200_DEPTH_PRIO"] = "1" if arm == "on_hi" else "0"
            pl = capi.Pipeline(params, max_batch=B, device=dev)
            if kc is not None:
                pl.set_undistort(kc)
            if arm != "off":
                pl.set_depth(dp)
            navs = [pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]) for s in range(W)]
            torch.cuda.synchronize()
            pl.event_record(0)
            for s in range(W, W + K):
                navs.append(pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]))
            pl.event_record(1)
            ms = pl.event_elapsed(0, 1)
            rec = None
            if arm == "on":   # the last frame's records, for the stage-call timing below
                pl.set_mirror(2)
                pl.push_dev(devbuf[0].data_ptr(), ts[(W + K) * B - 1:(W + K) * B] + 1.0)
                rec = pl.mirror(0).copy()
            pl.close()
            return K * B / (ms * 1e-3), np.concatenate(navs), rec

        fps = {"off": [], "on": [], "on_hi": []}
        ratio, ratio_hi = [], []
        same_all = True
        rec = None
        for p in range(args.pairs):
            got = {}
            for arm in (("off", "on", "on_hi") if p % 2 == 0 else ("on_hi", "on", "off")):
                got[arm] = run(arm)
                fps[arm].append(got[arm][0])
            rec = got["on"][2]
            ratio.append(got["on"][0] / got["off"][0])
            ratio_hi.append(got["on_hi"][0] / got["off"][0])
            same_all = same_all and got["on"][1].tobytes() == got["off"][1].tobytes() == got["on_hi"][1].tobytes()
        os.environ.pop("REBVO_B200_DEPTH_PRIO", None)
        identical = identical and same_all
        res = {"off": stats(fps["off"]), "on": stats(fps["on"]), "on_tracker_priority": stats(fps["on_hi"]),
               "on_over_off": stats(ratio), "on_tracker_priority_over_off": stats(ratio_hi), "nav_identical": same_all,
               "grid": [cam["h"] // 10, cam["w"] // 10], "cells_bytes_per_frame": (cam["h"] // 10) * (cam["w"] // 10) * 32}
        # one stage call on that frame's records
        ctx = capi.Ctx(cam, params.Sigma0, params.KSigma, kl_capacity=params.kl_capacity)
        for _ in range(10):
            ctx.depth_fill_net(rec, dp)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.calls):
            ctx.depth_fill_net(rec, dp)
        e1.record()
        e1.synchronize()
        res["records"] = int(len(rec))
        res["stage_call_us"] = 1e3 * e0.elapsed_time(e1) / args.calls
        # the fill kernel alone (device time of k_depth_fill from a torch.profiler trace of a few more calls)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                ctx.depth_fill_net(rec, dp)
        ev = [e for e in prof.events() if "k_depth_fill" in e.name]
        t = [getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) for e in ev]
        if t:
            res["fill_kernel_us"] = float(np.median(t))
            # the batch waits for its last frame's fill: one fill per batch of B frames, against the step time with depth on
            res["tail_join_share_of_on_step"] = res["fill_kernel_us"] * 1e-6 / (B / res["on"]["median"])
        ctx.close()
        try:
            from oracle import ref_depth
            if ref_depth.available():
                ref_depth.depth_fill_net(cam, rec, 10, 10, 1.0, 5, 10)
                n = 20
                t0 = time.perf_counter()
                for _ in range(n):
                    ref_depth.depth_fill_net(cam, rec, 10, 10, 1.0, 5, 10)
                res["reference_cpu_us"] = 1e6 * (time.perf_counter() - t0) / n
        except OSError:
            pass
        out[name] = res
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()

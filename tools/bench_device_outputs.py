#!/usr/bin/env python
"""bench_device_outputs.py -- what moving the per-frame outputs from mapped pinned host memory to device memory
(rb_pipeline_set_output_memory) is worth, at 752x480 with bench.py's configuration-2 parameters (EuRoC, UseUndistort=1) and
at 1280x960 (synthetic camera, no undistortion), frames resident in device memory (rb_pipeline_push_dev), 64-frame batches.
In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - per size, five arms: mirror mode 1, mirror mode 2, depth grid only, grid + image mode 1, grid + image mode 2 (viewer
    parameters 10x10 / 1 / 5 / 10).  Each arm has a host-mode and a device-mode pipeline, timed in alternating pairs of
    windows (host first in even pairs, device first in odd ones): per window the pipeline is reset, runs the warm-up steps,
    then the timed steps between CUDA events.  Median, min, max of frames/s per mode and the per-pair device/host ratios
    with their spread;
  - whether the nav records of the two modes are byte-identical in every window (exit status 1 if not);
  - the host time of one push (1 frame and 64 frames) of a device-mode pipeline whose consumer stream is idle: with the
    fence (torch's current stream) and without it (the pipeline's own stream), in alternating pairs.

Prints one JSON line (and writes it to --out if given).  Needs a CUDA device: there is no CPU path.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CAM_1280 = dict(w=1280, h=960, zfx=900.0, zfy=900.0, ppx=640.5, ppy=479.5)
ARMS = ("mirror1", "mirror2", "grid", "grid_image1", "grid_image2")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=7, help="alternating host / device pairs per arm and size (at least 5)")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--fence-pairs", type=int, default=15)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.pairs < 5:
        ap.error("--pairs must be at least 5")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_device_outputs.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    B, K, W = args.batch, args.steps, args.warmup
    out = {"what": "host vs device output memory, frames/s (CUDA events over %d timed steps of %d frames after %d warm-up "
                   "steps, pipeline reset before each window), frames resident in device memory" % (K, B, W),
           "gpu": gpu_info(dev), "pairs": args.pairs}
    identical = True
    for name, config, cam_over in (("752x480", 2, None), ("1280x960", None, CAM_1280)):
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

        def pipeline(arm, where):
            pl = capi.Pipeline(params, max_batch=B, device=dev)
            if kc is not None:
                pl.set_undistort(kc)
            if arm.startswith("mirror"):
                pl.set_mirror(int(arm[-1]))
            else:
                pl.set_depth(capi.depth_params())
                if arm != "grid":
                    pl.set_depth_image(int(arm[-1]))
            pl.set_output_memory(where)
            return pl

        def window(pl):
            pl.reset()
            navs = [pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]) for s in range(W)]
            torch.cuda.synchronize()
            pl.event_record(0)
            for s in range(W, W + K):
                navs.append(pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]))
            pl.event_record(1)
            ms = pl.event_elapsed(0, 1)
            return K * B / (ms * 1e-3), np.concatenate(navs)

        res = {}
        for arm in ARMS:
            pls = {w: pipeline(arm, w) for w in ("host", "device")}
            fps = {"host": [], "device": []}
            ratio = []
            same = True
            try:
                for p in range(args.pairs):
                    got = {}
                    for w in (("host", "device") if p % 2 == 0 else ("device", "host")):
                        got[w] = window(pls[w])
                        fps[w].append(got[w][0])
                    ratio.append(got["device"][0] / got["host"][0])
                    same = same and got["host"][1].tobytes() == got["device"][1].tobytes()
            finally:
                for pl in pls.values():
                    pl.close()
            identical = identical and same
            res[arm] = {"host_fps": stats(fps["host"]), "device_fps": stats(fps["device"]),
                        "device_over_host": stats(ratio), "nav_identical": same}
        out[name] = res

    # one push with an idle consumer stream: the fence (a wait on torch's current stream) against none
    cam, params, _, _, seed0 = bench.stream_setup(2)
    ts, base, idx = bench.make_stream(seed0, B * 4, cam=cam)
    devbuf = torch.from_numpy(np.ascontiguousarray(base[idx])).to("cuda:%d" % dev)
    pl = capi.Pipeline(params, max_batch=B, device=dev)
    fence = {}
    try:
        pl.set_undistort(bench.undistort_of(2))
        pl.set_depth(capi.depth_params())
        pl.set_depth_image(2)
        pl.set_output_memory("device")
        consumer = torch.cuda.current_stream(dev).cuda_stream
        nav = np.zeros(B, capi.NAV)
        k = [0]

        def one(n, stream):
            pl.set_consumer_stream(stream)
            s = (k[0] * n) % (B * 3)
            k[0] += 1
            t0 = time.perf_counter()
            pl.check(pl.L.rb_pipeline_push_dev(pl.h_, C.c_void_p(devbuf[s].data_ptr()), capi._p(ts[s:s + n]), n,
                                               capi._p(nav)))
            return (time.perf_counter() - t0) * 1e3

        for n in (1, B):
            for _ in range(3):   # warm-up: capture this push size's batches
                one(n, consumer)
                one(n, pl.stream())
            t = {"fence": [], "no_fence": []}
            for p in range(args.fence_pairs):
                for arm in (("fence", "no_fence") if p % 2 == 0 else ("no_fence", "fence")):
                    t[arm].append(one(n, consumer if arm == "fence" else pl.stream()))
            fence["push_%d_frames_ms" % n] = {a: stats(v) for a, v in t.items()}
    finally:
        pl.close()
    out["one_push_idle_consumer"] = dict(fence, config="752x480 configuration 2, grid + image mode 2, device mode; host "
                                         "clock around rb_pipeline_push_dev, which synchronises before it returns")
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()

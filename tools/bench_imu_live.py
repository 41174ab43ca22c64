#!/usr/bin/env python
"""bench_imu_live.py -- live IMU input (rb_pipeline_set_imu_live + rb_pipeline_push_imu) against dataset mode
(rb_pipeline_set_imu) on bench.py's IMU configuration (752x480 EuRoC parameters, UseUndistort=1, the walked seed-7 stream and
its synthetic 200 Hz samples).

A live camera delivers one frame at a time, so both arms push 1-frame batches from host memory; in the live arm each push is
preceded by push_imu of that frame's samples (those up to its time and the first one past it).  The live ring's integration
step is dataset mode's (the samples' mean spacing), so both arms must give the same nav records.  In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - dataset and live runs in alternating pairs (the order flips from pair to pair): frames/s of each run (host clock around
    the timed pushes, which return after a device synchronise) and the per-push latency (push_imu + push in the live arm);
    median, min and max per arm and the per-pair live / dataset ratio;
  - whether the nav records of the two arms are byte-identical in every pair (exit status 1 if not).

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

from bench_mono import gpu_info, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=6, help="alternating dataset / live pairs (at least 5)")
    ap.add_argument("--steps", type=int, default=200, help="timed 1-frame pushes per run")
    ap.add_argument("--warmup", type=int, default=20, help="untimed 1-frame pushes per run")
    ap.add_argument("--buffer", type=int, default=1000, help="live ring size (CircBufferSize)")
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.pairs < 5:
        ap.error("--pairs must be at least 5")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_imu_live.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from rebvo_b200 import capi, synth
    dev = 0
    torch.cuda.set_device(dev)
    K, W = args.steps, args.warmup
    total = K + W
    cam, params, _, _, seed0 = bench.stream_setup(3)
    kc = bench.undistort_of(3)
    ts, base, idx = bench.make_stream(seed0, total, bench.IMU_BASE_N, cam=cam)
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=seed0, zf=cam["zfx"])
    imu = synth.imu_samples_walk(seq, total, min(bench.IMU_BASE_N, total))
    frames = np.ascontiguousarray(base[idx])
    ip = capi.default_imu_params(InitBias=1, InitBiasFrameNum=5)
    tsample = (imu[-1, 0] - imu[0, 0]) / (len(imu) - 1)
    # each frame's samples: those up to its time and the first one past it
    cut = np.minimum(np.searchsorted(imu[:, 0], ts, side="right") + 1, len(imu))

    def run(mode):
        pl = capi.Pipeline(params, max_batch=1, device=dev)
        pl.set_undistort(kc)
        if mode == "dataset":
            pl.set_imu(imu, ip)
        else:
            pl.set_imu_live(ip, tsample, args.buffer)
        navs, lat = [], []
        cur = 0
        t_start = 0.0
        for i in range(total):
            if i == W:
                torch.cuda.synchronize()
                t_start = time.perf_counter()
            t0 = time.perf_counter()
            if mode == "live":
                pl.push_imu(imu[cur:cut[i]])
                cur = int(cut[i])
                while True:   # (only the first frame's window (0, 0] needs one sample more than its chunk)
                    try:
                        nav = pl.push(frames[i:i + 1], ts[i:i + 1])
                        break
                    except capi.RbError:
                        if i >= W or cur >= len(imu):
                            raise
                        pl.push_imu(imu[cur:cur + 1])
                        cur += 1
            else:
                nav = pl.push(frames[i:i + 1], ts[i:i + 1])
            t1 = time.perf_counter()
            navs.append(nav)
            if i >= W:
                lat.append((t1 - t0) * 1e3)
        elapsed = time.perf_counter() - t_start
        pl.close()
        return K / elapsed, lat, np.concatenate(navs)

    fps = {"dataset": [], "live": []}
    lat_med = {"dataset": [], "live": []}
    lat_all = {"dataset": [], "live": []}
    ratio = []
    identical, first_diff = True, None
    for p in range(args.pairs):
        order = ("dataset", "live") if p % 2 == 0 else ("live", "dataset")
        got = {}
        for mode in order:
            got[mode] = run(mode)
            fps[mode].append(got[mode][0])
            lat_med[mode].append(float(np.median(got[mode][1])))
            lat_all[mode] += got[mode][1]
        ratio.append(got["live"][0] / got["dataset"][0])
        a, b = got["dataset"][2], got["live"][2]
        same = a.tobytes() == b.tobytes()
        if not same and first_diff is None:
            d = np.nonzero((a.view(np.uint8) != b.view(np.uint8)).reshape(len(a), -1).any(1))[0]
            first_diff = {"pair": p, "frame": int(d[0]) if len(d) else None}
        identical = identical and same

    res = {"gpu": gpu_info(dev), "frames_per_run": K, "warmup": W, "pairs": args.pairs, "push_frames": 1,
           "frame": "%dx%d" % (cam["w"], cam["h"]), "live_buffer": args.buffer, "sample_rate_hz": 200,
           "fps": {m: stats(v) for m, v in fps.items()},
           "push_latency_ms": {m: {"median": float(np.median(lat_all[m])), "p90": float(np.percentile(lat_all[m], 90)),
                                   "per_run_median": stats(lat_med[m])} for m in lat_all},
           "live_over_dataset_fps": stats(ratio), "nav_identical": identical, "first_diff": first_diff}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0 if identical else 1


if __name__ == "__main__":
    sys.exit(main())

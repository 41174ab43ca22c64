#!/usr/bin/env python
"""bench_odometry.py -- cost of the per-frame odometry records (rb_pipeline_set_odometry) on bench.py's configurations 2
(752x480 EuRoC parameters, UseUndistort=1, IMU off) and 3 (the same with IMU fusion), frames resident in device memory
(rb_pipeline_push_dev), 64-frame batches, the seed-7 stream of bench.py.  In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - per configuration, runs with the records off and on in alternating pairs (the order flips from pair to pair): median,
    min and max of frames/s per arm, and the per-pair on / off ratio with its spread;
  - whether the nav records of the two arms are byte-identical in every pair (exit status 1 if not).

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=7, help="alternating off / on pairs per configuration (at least 5)")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--imu-steps", type=int, default=3, help="timed steps in IMU mode (a host-driven flow, much slower)")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.pairs < 5:
        ap.error("--pairs must be at least 5")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_odometry.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi, synth
    dev = 0
    torch.cuda.set_device(dev)
    B = args.batch
    out = {"what": "odometry records off vs on, frames/s (CUDA events over the timed steps of %d frames after %d warm-up "
                   "steps), frames resident in device memory, seed-7 stream" % (B, args.warmup),
           "gpu": gpu_info(dev), "pairs": args.pairs, "d2h_bytes_per_frame": capi.ODOM.itemsize}
    identical = True
    for config in (2, 3):
        K, W = (args.steps if config == 2 else args.imu_steps), args.warmup
        total = B * (K + W)
        cam, params, _, _, seed0 = bench.stream_setup(config)
        kc = bench.undistort_of(config)
        ts, base, idx = bench.make_stream(seed0, total, cam=cam)
        imu = None
        if config == 3:   # as bench.py: IMU samples of the walked camera path
            seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=seed0, zf=cam["zfx"])
            imu = synth.imu_samples_walk(seq, total, min(bench.IMU_BASE_N, total))
        devbuf = torch.from_numpy(np.ascontiguousarray(base[idx])).to("cuda:%d" % dev)
        torch.cuda.synchronize()

        def run(on):
            pl = capi.Pipeline(params, max_batch=B, device=dev)
            if kc is not None:
                pl.set_undistort(kc)
            if imu is not None:
                pl.set_imu(imu, capi.default_imu_params(InitBias=1, InitBiasFrameNum=5))
            pl.set_odometry(on)
            navs = [pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]) for s in range(W)]
            torch.cuda.synchronize()
            pl.event_record(0)
            for s in range(W, W + K):
                navs.append(pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]))
                if on:
                    pl.odometry()
            pl.event_record(1)
            ms = pl.event_elapsed(0, 1)
            pl.close()
            return K * B / (ms * 1e-3), np.concatenate(navs)

        fps = {"off": [], "on": []}
        ratio = []
        same_all = True
        for p in range(args.pairs):
            got = {}
            for arm in (("off", "on") if p % 2 == 0 else ("on", "off")):
                got[arm] = run(arm == "on")
                fps[arm].append(got[arm][0])
            ratio.append(got["on"][0] / got["off"][0])
            same_all = same_all and got["on"][1].tobytes() == got["off"][1].tobytes()
        identical = identical and same_all
        r = stats(ratio)
        out["config%d" % config] = {"steps": K, "off": stats(fps["off"]), "on": stats(fps["on"]), "on_over_off": r,
                                    "nav_identical": same_all}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if identical else 1)


if __name__ == "__main__":
    main()

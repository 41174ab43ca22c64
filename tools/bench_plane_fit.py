#!/usr/bin/env python
"""bench_plane_fit.py -- DetectorPlaneFitSize 1..4 on the default bench configuration (752x480 EuRoC parameters,
UseUndistort=1 with the EuRoC rad-tan coefficients, 64-frame batches, the seed-7 stream of bench.py).

In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - R = 1..4 in rotating order (round k starts at R = 1 + k mod 4), frames resident in device memory
    (rb_pipeline_push_dev); per R the median, min and max of frames/s (CUDA events over the timed steps) and the mean
    keylines per frame;
  - per R the detector's time per frame from an eager run with the stage profile on (REBVO_B200_STAGE_PROF=1:
    k_update_thresh + k_detect_a<R> + k_seg_scan + k_detect_b + k_join between two events).  rb_pipeline_stage_ms[2] is
    not used for it: with the batch replayed as one CUDA graph it only covers the nav copy.

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

from bench_mono import gpu_info, stats  # noqa: E402

RADII = (1, 2, 3, 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="rotations over R = 1..4 (at least 5)")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.rounds < 5:
        ap.error("--rounds must be at least 5")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_plane_fit.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    B, K, W = args.batch, args.steps, args.warmup
    total = B * (K + W)
    cam, params, _, _, seed0 = bench.stream_setup(2)
    kc = bench.undistort_of(2)
    ts, base, idx = bench.make_stream(seed0, total, cam=cam)
    frames = torch.from_numpy(np.ascontiguousarray(base[idx])).to("cuda:%d" % dev)
    torch.cuda.synchronize()

    def with_r(R):
        p = capi.Params.from_buffer_copy(params)
        p.det.plane_fit_size = R
        return p

    def run(R):
        pl = capi.Pipeline(with_r(R), max_batch=B, device=dev)
        pl.set_undistort(kc)
        for s in range(W):
            pl.push_dev(frames[s * B].data_ptr(), ts[s * B:(s + 1) * B])
        torch.cuda.synchronize()
        pl.event_record(0)
        navs = [pl.push_dev(frames[s * B].data_ptr(), ts[s * B:(s + 1) * B]) for s in range(W, W + K)]
        pl.event_record(1)
        ms = pl.event_elapsed(0, 1)
        pl.close()
        nav = np.concatenate(navs)
        return K * B / (ms * 1e-3), float(nav["kn"].mean())

    fps = {R: [] for R in RADII}
    kn = {R: [] for R in RADII}
    for k in range(args.rounds):
        for j in range(len(RADII)):
            R = RADII[(k + j) % len(RADII)]
            f, n = run(R)
            fps[R].append(f)
            kn[R].append(n)

    detect_ms = {}
    os.environ["REBVO_B200_STAGE_PROF"] = "1"   # read at pipeline creation
    try:
        for R in RADII:   # (the kernels are warm from the timed runs; the profile covers every push of this pipeline)
            pl = capi.Pipeline(with_r(R), max_batch=B, device=dev)
            pl.set_undistort(kc)
            for s in range(W + K):
                pl.push_dev(frames[s * B].data_ptr(), ts[s * B:(s + 1) * B])
            prof, nfr = pl.stage_profile()
            pl.close()
            detect_ms[R] = {"detect_us_per_frame": prof["detect"], "reestimate_us_per_frame": prof["reestimate"],
                            "frames": int(nfr)}
    finally:
        del os.environ["REBVO_B200_STAGE_PROF"]

    out = {"what": "DetectorPlaneFitSize 1..4, frames/s (CUDA events over %d steps of %d frames after %d warm-up steps), "
                   "752x480 EuRoC parameters, UseUndistort=1, seed-7 stream, frames resident on the device" % (K, B, W),
           "gpu": gpu_info(dev), "rounds": args.rounds,
           "radii": {str(R): {"window": "%dx%d" % (2 * R + 1, 2 * R + 1), "fps": stats(fps[R]),
                              "keylines_per_frame": float(np.mean(kn[R])), **detect_ms[R]} for R in RADII}}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

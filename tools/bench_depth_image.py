#!/usr/bin/env python
"""bench_depth_image.py -- cost of the per-frame dense inverse-depth image (rb_pipeline_set_depth_image: depth_filler::getImgRho
at every pixel of each frame's depth grid) at 752x480 with bench.py's configuration-2 parameters (EuRoC, UseUndistort=1)
and at 1280x960 (synthetic camera, no undistortion), frames resident in device memory (rb_pipeline_push_dev), 64-frame
batches, the depth grid on in every arm with the viewer's parameters (10x10 blocks, ThreshRelRho 1, ThreshMatchNum 5,
IterNum 10).  In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - per size, three arms in rotations whose order alternates (grid only, grid + mode 1, grid + mode 2, then reversed):
    median, min and max of frames/s per arm and the per-rotation ratios of each image arm to the grid-only arm;
  - whether the nav records of the arms are byte-identical in every rotation (exit status 1 if not);
  - from a separate run under torch.profiler: the device time of the k_depth_image kernel in the pipeline (mode 1 and
    mode 2, writing into mapped pinned host memory), the bytes it moves per frame (w * h * 4 per plane written, plus the
    grid's gw * gh * 16 bytes read) and the effective rate (bytes / kernel time).

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

CAM_1280 = dict(w=1280, h=960, zfx=900.0, zfy=900.0, ppx=640.5, ppy=479.5)
ARMS = ("grid", "mode1", "mode2")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rotations", type=int, default=7, help="rotations of the three arms per size (at least 5)")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.rotations < 5:
        ap.error("--rotations must be at least 5")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_depth_image.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    B, K, W = args.batch, args.steps, args.warmup
    dp = capi.depth_params()
    out = {"what": "depth grid only vs grid + image mode 1 / 2, frames/s (CUDA events over %d timed steps of %d frames after "
                   "%d warm-up steps), frames resident in device memory; viewer parameters 10x10 / 1 / 5 / 10" % (K, B, W),
           "gpu": gpu_info(dev), "rotations": args.rotations}
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

        def pipeline(arm):
            pl = capi.Pipeline(params, max_batch=B, device=dev)
            if kc is not None:
                pl.set_undistort(kc)
            pl.set_depth(dp)
            if arm != "grid":
                pl.set_depth_image(int(arm[-1]))
            return pl

        def run(arm):
            pl = pipeline(arm)
            navs = [pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]) for s in range(W)]
            torch.cuda.synchronize()
            pl.event_record(0)
            for s in range(W, W + K):
                navs.append(pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B]))
            pl.event_record(1)
            ms = pl.event_elapsed(0, 1)
            pl.close()
            return K * B / (ms * 1e-3), np.concatenate(navs)

        fps = {a: [] for a in ARMS}
        ratio = {a: [] for a in ARMS[1:]}
        same_all = True
        for p in range(args.rotations):
            got = {}
            for arm in (ARMS if p % 2 == 0 else ARMS[::-1]):
                got[arm] = run(arm)
                fps[arm].append(got[arm][0])
            for a in ARMS[1:]:
                ratio[a].append(got[a][0] / got["grid"][0])
            same_all = same_all and got["grid"][1].tobytes() == got["mode1"][1].tobytes() == got["mode2"][1].tobytes()
        identical = identical and same_all
        gw, gh = cam["w"] // 10, cam["h"] // 10
        res = {a: stats(fps[a]) for a in ARMS}
        res.update({"%s_over_grid" % a: stats(ratio[a]) for a in ARMS[1:]})
        res["nav_identical"] = same_all
        res["grid_cells"] = [gh, gw]
        # the image kernel alone: device time of k_depth_image from a torch.profiler trace of a separate run per mode
        from torch.profiler import ProfilerActivity, profile
        for mode in (1, 2):
            pl = pipeline("mode%d" % mode)
            for s in range(W):
                pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B])
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for s in range(W, W + 2):
                    pl.push_dev(devbuf[s * B].data_ptr(), ts[s * B:(s + 1) * B])
                torch.cuda.synchronize()
            pl.close()
            ev = [e for e in prof.events() if "k_depth_image" in e.name]
            t = [getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) for e in ev]
            written = mode * cam["w"] * cam["h"] * 4
            m = {"bytes_written_per_frame": written, "grid_bytes_read_per_frame": gw * gh * 16,
                 "bytes_written_per_batch": written * B, "kernels_traced": len(t)}
            if t:
                us = float(np.median(t))
                m["kernel_us"] = {"median": us, "min": float(np.min(t)), "max": float(np.max(t))}
                m["effective_gb_per_s"] = (written + gw * gh * 16) / (us * 1e-6) / 1e9
            res["image_kernel_mode%d" % mode] = m
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

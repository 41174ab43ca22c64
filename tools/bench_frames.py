#!/usr/bin/env python
"""bench_frames.py -- what strided frame input (Pipeline.push_frames: rb_pipeline_push_frames / _dev) costs or saves against
packed input.  In one invocation:

  - the GPU's name and power limit (nvidia-smi);
  - host frames, 64-frame batches from a list of per-frame arrays (one allocation per frame, as ROS messages, cv2.imread or
    dataset loaders hand them over): np.stack + push against push_frames(list), at 752x480 with bench.py's configuration-2
    parameters (EuRoC, UseUndistort=1) and at 1280x960 (synthetic camera, no undistortion).  Alternating pairs of windows;
    per window the pipeline is reset, runs the warm-up steps, then the timed steps on the host clock (each push
    synchronises, and the np.stack is part of its arm).  frames/s;
  - live-style 1-frame pushes of host frames whose rows are padded to a 512-byte step, at 752x480 configuration 2:
    host-clock latency per push, push_frames([frame]) against np.ascontiguousarray (the repack) + push, in alternating pairs
    of blocks;
  - device frames: a packed tensor through push_dev / push_mono_dev against strided views through push_frames, frames/s
    with CUDA events, alternating pairs: 752x480 configuration 2 with a 512-byte-aligned step (RGB24 and mono8), and
    1226x900 crops (x 27.., y 30..) of 1280x960 frames (RGB24, no undistortion);
  - kernel times from a separate torch.profiler run with eager launches (REBVO_B200_NO_GRAPH=1): the gray and undistortion
    passes of packed and strided device pushes of 64 frames, in picoseconds per pixel, at 752x480 and at 1226x370 (the
    any-width path; there the strided pushes read packed frames, step w*bpp and frames frame_bytes apart, to compare
    the strided layout with the packed any-width one on the same bytes);
  - whether every arm's nav records equal its packed twin's (exit status 1 if not).

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
CROP = (27, 30, 1226, 900)   # x0, y0, w, h of the crop of a 1280x960 frame
CAM_CROP = dict(w=1226, h=900, zfx=900.0, zfy=900.0, ppx=640.5 - 27, ppy=479.5 - 30)
CAM_1226 = dict(w=1226, h=370, zfx=718.856, zfy=718.856, ppx=599.7, ppy=182.2)


def pitch512(row):
    return -(-row // 512) * 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=7, help="alternating pairs per arm (at least 7)")
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--live-pushes", type=int, default=20, help="1-frame pushes per block of the live-style comparison")
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.pairs < 7:
        ap.error("--pairs must be at least 7")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_frames.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    B, K, W = args.batch, args.steps, args.warmup
    total = B * (K + W)
    out = {"what": "strided (push_frames) against packed input; windows of %d timed steps of %d frames after %d warm-up "
                   "steps, pipeline reset before each window" % (K, B, W), "gpu": gpu_info(dev), "pairs": args.pairs}
    identical = True

    streams = {}

    def setup(name):
        if name not in streams:
            streams[name] = make(name)
        return streams[name]

    def make(name):
        if name == "752x480":
            cam, params, _, _, seed0 = bench.stream_setup(2)
            ts, base, idx = bench.make_stream(seed0, total, base_n=40, cam=cam)
            return cam, params, bench.undistort_of(2), ts, base, idx
        ts, base, idx = bench.make_stream(7, total, base_n=40, cam=CAM_1280)
        return CAM_1280, capi.default_params(CAM_1280), None, ts, base, idx

    def pipeline(params, kc):
        pl = capi.Pipeline(params, max_batch=B, device=dev)
        if kc is not None:
            pl.set_undistort(kc)
        return pl

    def pairs(arms, window):
        """alternating pairs of windows of the two arms: {arm: [rate]}, [rate ratio arm1 / arm0], nav records equal"""
        got = {a: [] for a in arms}
        ratio, same = [], True
        for p in range(args.pairs):
            res = {}
            for a in (arms if p % 2 == 0 else arms[::-1]):
                res[a] = window(a)
                got[a].append(res[a][0])
            ratio.append(res[arms[1]][0] / res[arms[0]][0])
            same = same and res[arms[0]][1].tobytes() == res[arms[1]][1].tobytes()
        return {a: stats(v) for a, v in got.items()}, stats(ratio), same

    # ---- host frames: a list of per-frame arrays, 64-frame batches --------------------------------------------------------
    host = {}
    for name in ("752x480", "1280x960"):
        cam, params, kc, ts, base, idx = setup(name)
        frames = [np.array(base[i]) for i in range(len(base))]   # one allocation per frame
        stream = [frames[i] for i in idx]
        pls = {a: pipeline(params, kc) for a in ("stack_push", "push_frames")}

        def window(arm):
            pl = pls[arm]
            pl.reset()
            navs = []
            for s in range(W + K):
                if s == W:
                    t0 = time.perf_counter()
                lst, t = stream[s * B:(s + 1) * B], ts[s * B:(s + 1) * B]
                navs.append(pl.push(np.stack(lst), t) if arm == "stack_push" else pl.push_frames(lst, t))
            return K * B / (time.perf_counter() - t0), np.concatenate(navs)
        try:
            fps, ratio, same = pairs(("stack_push", "push_frames"), window)
        finally:
            for pl in pls.values():
                pl.close()
        identical = identical and same
        host[name] = {"fps": fps, "push_frames_over_stack_push": ratio, "nav_identical": same,
                      "undistort": kc is not None}
    out["host_list_64"] = host

    # ---- live-style 1-frame pushes of padded host frames ----------------------------------------------------------------
    cam, params, kc, ts, base, idx = setup("752x480")
    h, w = cam["h"], cam["w"]
    step = pitch512(3 * w)
    padded = []
    for i in range(len(base)):
        buf = np.zeros(h * step, np.uint8)
        buf.reshape(h, step)[:, :3 * w] = base[i].reshape(h, 3 * w)
        padded.append(np.lib.stride_tricks.as_strided(buf, (h, w, 3), (step, 3, 1)))
    pls = {a: pipeline(params, kc) for a in ("repack_push", "push_frames")}
    lat = {a: [] for a in pls}
    k = {a: 0 for a in pls}
    try:
        def one(arm):
            i = k[arm]
            k[arm] += 1
            f, t = padded[idx[i % len(idx)]], ts[i:i + 1] if i < len(ts) else np.array([i / 20.0])
            t0 = time.perf_counter()
            if arm == "repack_push":
                pls[arm].push(np.ascontiguousarray(f)[None], t)
            else:
                pls[arm].push_frames([f], t)
            return (time.perf_counter() - t0) * 1e3
        for a in pls:   # warm-up: the first push, then the captured 1-frame batches of every ring phase
            for _ in range(5):
                one(a)
        for p in range(args.pairs):
            for a in (("repack_push", "push_frames") if p % 2 == 0 else ("push_frames", "repack_push")):
                lat[a].append(float(np.median([one(a) for _ in range(args.live_pushes)])))
    finally:
        for pl in pls.values():
            pl.close()
    out["live_1_frame"] = {"ms_per_push": {a: stats(v) for a, v in lat.items()}, "step": step,
                           "block_median_of": args.live_pushes, "config": "752x480 configuration 2, UseUndistort=1"}

    # ---- device frames ----------------------------------------------------------------------------------------------------
    devres = {}
    for name, fmt in (("752x480_step512_rgb", "rgb"), ("752x480_step512_mono", "mono"), ("1226x900_crop_of_1280x960", "rgb")):
        if name.startswith("752"):
            cam, params, kc, ts, base, idx = setup("752x480")
            h, w = cam["h"], cam["w"]
            frames = torch.from_numpy(np.ascontiguousarray(base)).cuda()[torch.from_numpy(idx).cuda()]
            src = frames if fmt == "rgb" else frames[..., 0]
            bpp = 3 if fmt == "rgb" else 1
            s = pitch512(w * bpp)
            big = torch.zeros((total, h, s), dtype=torch.uint8, device="cuda:%d" % dev)
            big[:, :, :w * bpp] = src.reshape(total, h, w * bpp)
            del frames, src
            view = big[:, :, :w * bpp]
            view = view.unflatten(2, (w, 3)) if fmt == "rgb" else view
        else:
            ts, base, idx = setup("1280x960")[3:]
            x0, y0, w, h = CROP
            cam, kc = CAM_CROP, None
            params = capi.default_params(cam)
            big = torch.from_numpy(np.ascontiguousarray(base)).cuda()[torch.from_numpy(idx).cuda()]
            view = big[:, y0:y0 + h, x0:x0 + w]
        packed = view.contiguous()
        torch.cuda.synchronize()
        pls = {a: pipeline(params, kc) for a in ("packed", "strided")}

        def window(arm):
            pl = pls[arm]
            pl.reset()
            navs = []
            for s_ in range(W + K):
                if s_ == W:
                    torch.cuda.synchronize()
                    pl.event_record(0)
                t = ts[s_ * B:(s_ + 1) * B]
                if arm == "packed":
                    ptr = packed[s_ * B].data_ptr()
                    navs.append(pl.push_dev(ptr, t) if fmt == "rgb" else pl.push_mono_dev(ptr, t))
                else:
                    navs.append(pl.push_frames(view[s_ * B:(s_ + 1) * B], t))
            pl.event_record(1)
            return K * B / (pl.event_elapsed(0, 1) * 1e-3), np.concatenate(navs)
        try:
            fps, ratio, same = pairs(("packed", "strided"), window)
        finally:
            for pl in pls.values():
                pl.close()
        identical = identical and same
        devres[name] = {"fps": fps, "strided_over_packed": ratio, "nav_identical": same, "undistort": kc is not None,
                        "step": int(view.stride(1))}
        del big, view, packed
    out["device"] = devres

    # ---- kernel times (torch.profiler, eager launches) --------------------------------------------------------------------
    out["kernels_ps_per_pixel"] = kernel_times(torch, capi, bench, B)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if identical else 1)


def kernel_times(torch, capi, bench, B, reps=4):
    """ps per pixel of each gray / undistortion kernel over `reps` 64-frame device pushes per arm, packed and strided."""
    from torch.profiler import ProfilerActivity, profile
    os.environ["REBVO_B200_NO_GRAPH"] = "1"
    res = {}
    try:
        for name, cam in (("752x480", None), ("1226x370", CAM_1226)):
            if cam is None:
                cam, params, _, _, seed0 = bench.stream_setup(2)
                kcs = (None, bench.undistort_of(2))
            else:
                params, seed0 = capi.default_params(cam), 7
                kcs = (None, (-0.12, 0.03, 0.0, 1e-4, 2e-5))
            h, w = cam["h"], cam["w"]
            ts, base, idx = bench.make_stream(seed0, B * (reps + 1), base_n=20, cam=cam)
            rgb = torch.from_numpy(np.ascontiguousarray(base[idx])).cuda()
            mono = rgb[..., 0].contiguous()
            for kc in kcs:
                for fmt, buf in (("rgb", rgb), ("mono", mono)):
                    pl = capi.Pipeline(params, max_batch=B)
                    if kc is not None:
                        pl.set_undistort(kc)
                    pl.push_frames(buf[:B], ts[:B])   # warm-up (first frame, module loads)
                    torch.cuda.synchronize()
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for r in range(1, reps + 1):
                            t = ts[r * B:(r + 1) * B]
                            p = buf[r * B].data_ptr()
                            pl.push_dev(p, t) if fmt == "rgb" else pl.push_mono_dev(p, t)
                            pl.push_frames(buf[r * B:(r + 1) * B], t)   # packed bytes, read through the frame table
                        torch.cuda.synchronize()
                    pl.close()
                    for e in prof.key_averages():
                        key = e.key
                        if "gray" not in key:
                            continue
                        short = key.replace("void ", "")   # the name with its template arguments, which may hold "("
                        short = short[:short.index(">") + 1] if "<" in short.split("(")[0] else short.split("(")[0]
                        tot = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)   # us
                        ent = res.setdefault(name, {}).setdefault("%s%s" % ("und_" if kc is not None else "", fmt), {})
                        ent[short] = {"ps_per_pixel": tot * 1e6 / (e.count * B * w * h), "launches": e.count}
    finally:
        os.environ.pop("REBVO_B200_NO_GRAPH", None)
    return res


if __name__ == "__main__":
    main()

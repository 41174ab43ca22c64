#!/usr/bin/env python
"""bench_async.py -- what asynchronous pushes (Pipeline.set_async / enqueue / wait: rb_pipeline_enqueue) recover for a live
caller that hands over one frame at a time.  In one invocation:

  - the GPU's name, power limit and SM clock (nvidia-smi, before and after the timed arms);
  - 1-frame pushes, synchronous against asynchronous at depth 2 and 4, from host memory (pinned, so that the enqueue's copy
    does not block) and from device memory, at 752x480 with bench.py's configuration-2 parameters (EuRoC, UseUndistort=1)
    and at 1280x960 (synthetic camera, no undistortion).  Per block the pipeline is reset, runs --warmup pushes, then
    --pushes timed ones on the host clock, the asynchronous arms keeping `depth` tickets in flight (enqueue, and wait for the
    oldest when the queue is full).  The three arms alternate, their order rotating from round to round.  frames/s,
    enqueue -> wait latency p50 / p90 (a push's own time for the synchronous arm), medians over the rounds with their
    ranges;
  - 64-frame batches from host memory at 752x480, synchronous against asynchronous depth 2, alternating pairs: frames/s;
  - overlap: one torch.profiler run (CUDA activities) of 1-frame device enqueues at depth 2 (752x480): the share of the
    front's kernel time (gray and scale space, on the front stream) during which a kernel of another stream (the back of the
    previous ticket) was running;
  - whether every arm's nav records equal the synchronous arm's (exit status 1 if not).

Prints one JSON line (and writes it to --out if given).  Needs a CUDA device: there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

CAM_1280 = dict(w=1280, h=960, zfx=900.0, zfy=900.0, ppx=640.5, ppy=479.5)


def sm_clock(dev):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=60).stdout.strip().split(", ")
        return {"sm_mhz": float(out[0]), "max_sm_mhz": float(out[1])}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="rounds of alternating arms (at least 3)")
    ap.add_argument("--pushes", type=int, default=100, help="timed 1-frame pushes per block")
    ap.add_argument("--warmup", type=int, default=12)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=4, help="timed 64-frame batches per window")
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    if args.rounds < 3:
        ap.error("--rounds must be at least 3")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_async.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    out = {"what": "asynchronous (enqueue / wait) against synchronous pushes", "gpu": gpu_info(dev),
           "sm_clock_before": sm_clock(dev), "rounds": args.rounds}
    identical = True
    n1 = args.warmup + args.pushes

    def setup(name, total):
        if name == "752x480":
            cam, params, _, _, seed0 = bench.stream_setup(2)
            ts, base, idx = bench.make_stream(seed0, total, base_n=40, cam=cam)
            return cam, params, bench.undistort_of(2), ts, base, idx
        ts, base, idx = bench.make_stream(7, total, base_n=20, cam=CAM_1280)
        return CAM_1280, capi.default_params(CAM_1280), None, ts, base, idx

    def pipeline(params, kc, batch, depth):
        pl = capi.Pipeline(params, max_batch=batch, device=dev)
        if kc is not None:
            pl.set_undistort(kc)
        if depth:
            pl.set_async(depth)
        return pl

    # ---- 1-frame pushes -----------------------------------------------------------------------------------------------------
    arms = ("sync", "async2", "async4")
    live = {}
    for name in ("752x480", "1280x960"):
        cam, params, kc, ts, base, idx = setup(name, n1)
        host = torch.from_numpy(np.ascontiguousarray(base[idx])).pin_memory()
        hostnp = host.numpy()
        devbuf = host.cuda()
        torch.cuda.synchronize()
        for where in ("host", "device"):
            frames = hostnp if where == "host" else devbuf
            pls = {a: pipeline(params, kc, 1, {"sync": 0, "async2": 2, "async4": 4}[a]) for a in arms}

            def block(arm):
                pl = pls[arm]
                pl.reset()
                navs, lat, pending = [], [], []
                for i in range(n1):
                    if i == args.warmup:
                        t0 = time.perf_counter()
                    f, t = frames[i:i + 1], ts[i:i + 1]
                    s = time.perf_counter()
                    if arm == "sync":
                        navs.append(pl.push(f, t) if where == "host" else pl.push_dev(f.data_ptr(), t))
                        lat.append(time.perf_counter() - s)
                        continue
                    pending.append((pl.enqueue(f, t), s))
                    if len(pending) == pl_depth[arm] or i == n1 - 1:
                        while pending and (i == n1 - 1 or len(pending) == pl_depth[arm]):
                            tk, s0 = pending.pop(0)
                            navs.append(pl.wait(tk))
                            lat.append(time.perf_counter() - s0)
                fps = args.pushes / (time.perf_counter() - t0)
                return fps, np.array(lat[args.warmup:]) * 1e3, np.concatenate(navs)
            pl_depth = {"async2": 2, "async4": 4}
            fps = {a: [] for a in arms}
            p50 = {a: [] for a in arms}
            p90 = {a: [] for a in arms}
            same = True
            try:
                for r in range(args.rounds):
                    res = {}
                    for a in arms[r % 3:] + arms[:r % 3]:
                        res[a] = block(a)
                        fps[a].append(res[a][0])
                        p50[a].append(float(np.percentile(res[a][1], 50)))
                        p90[a].append(float(np.percentile(res[a][1], 90)))
                    for a in arms[1:]:
                        same = same and res[a][2].tobytes() == res["sync"][2].tobytes()
            finally:
                for pl in pls.values():
                    pl.close()
            identical = identical and same
            live["%s_%s" % (name, where)] = {
                "fps": {a: stats(v) for a, v in fps.items()}, "latency_ms_p50": {a: stats(v) for a, v in p50.items()},
                "latency_ms_p90": {a: stats(v) for a, v in p90.items()},
                "fps_over_sync": {a: stats(np.array(fps[a]) / np.array(fps["sync"])) for a in arms[1:]},
                "nav_identical": same, "undistort": kc is not None}
        del host, hostnp, devbuf
    out["live_1_frame"] = live

    # ---- 64-frame batches -----------------------------------------------------------------------------------------------------
    B, K, W = args.batch, args.steps, 2
    cam, params, kc, ts, base, idx = setup("752x480", B * (K + W))
    frames = torch.from_numpy(np.ascontiguousarray(base[idx])).pin_memory().numpy()
    pls = {a: pipeline(params, kc, B, d) for a, d in (("sync", 0), ("async2", 2))}

    def window(arm):
        pl = pls[arm]
        pl.reset()
        navs, pending = [], []
        for s in range(W + K):
            if s == W:
                t0 = time.perf_counter()
            f, t = frames[s * B:(s + 1) * B], ts[s * B:(s + 1) * B]
            if arm == "sync":
                navs.append(pl.push(f, t))
                continue
            pending.append(pl.enqueue(f, t))
            if len(pending) == 2:
                navs.append(pl.wait(pending.pop(0)))
        navs += [pl.wait(tk) for tk in pending]
        return K * B / (time.perf_counter() - t0), np.concatenate(navs)
    fps = {a: [] for a in pls}
    ratio, same = [], True
    try:
        for r in range(args.rounds):
            res = {}
            for a in (("sync", "async2") if r % 2 == 0 else ("async2", "sync")):
                res[a] = window(a)
                fps[a].append(res[a][0])
            ratio.append(res["async2"][0] / res["sync"][0])
            same = same and res["async2"][1].tobytes() == res["sync"][1].tobytes()
    finally:
        for pl in pls.values():
            pl.close()
    identical = identical and same
    out["batch_64_host"] = {"fps": {a: stats(v) for a, v in fps.items()}, "async2_over_sync": stats(ratio),
                            "nav_identical": same, "config": "752x480 configuration 2, UseUndistort=1, pinned host frames"}
    out["sm_clock_after"] = sm_clock(dev)
    out["overlap"] = overlap(torch, capi, setup, pipeline, n1)
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    sys.exit(0 if identical else 1)


def overlap(torch, capi, setup, pipeline, n):
    """Share of the front's kernel time hidden behind kernels of other streams, 1-frame device enqueues at depth 2."""
    from torch.profiler import ProfilerActivity, profile
    cam, params, kc, ts, base, idx = setup("752x480", n)
    frames = torch.from_numpy(np.ascontiguousarray(base[idx])).cuda()
    pl = pipeline(params, kc, 1, 2)
    try:
        for i in range(8):   # warm-up: first frame, captures of every phase and workspace
            pl.wait(pl.enqueue(frames[i:i + 1], ts[i:i + 1]))
        torch.cuda.synchronize()
        pending = []
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(8, n):
                pending.append(pl.enqueue(frames[i:i + 1], ts[i:i + 1]))
                if len(pending) == 2:
                    pl.wait(pending.pop(0))
            for tk in pending:
                pl.wait(tk)
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                trace = json.load(f)
    finally:
        pl.close()
    kernels = [(e["ts"], e["ts"] + e["dur"], e["args"].get("stream"), e["name"]) for e in trace.get("traceEvents", [])
               if e.get("cat") == "kernel" and "dur" in e]
    front_streams = {s for _, _, s, name in kernels if "gray" in name}
    if len(front_streams) != 1:
        return {"error": "front stream not identified", "streams": sorted(map(str, front_streams))}
    fs = front_streams.pop()
    front = [(a, b) for a, b, s, _ in kernels if s == fs]
    others = sorted((a, b) for a, b, s, _ in kernels if s != fs)
    merged = []   # union of the other streams' busy intervals
    for a, b in others:
        if merged and a <= merged[-1][1]:
            merged[-1][1] = max(merged[-1][1], b)
        else:
            merged.append([a, b])
    starts = np.array([m[0] for m in merged])
    tot = hid = 0.0
    for a, b in front:
        tot += b - a
        k = max(int(np.searchsorted(starts, a, side="right")) - 1, 0)
        while k < len(merged) and merged[k][0] < b:
            hid += max(0.0, min(b, merged[k][1]) - max(a, merged[k][0]))
            k += 1
    return {"front_kernel_us_per_ticket": tot / max(n - 8, 1), "front_share_hidden": hid / tot if tot else None,
            "front_kernels": len(front), "tickets": n - 8, "config": "752x480 configuration 2, device frames, depth 2"}


if __name__ == "__main__":
    main()

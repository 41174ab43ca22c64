#!/usr/bin/env python
"""bench_mask.py -- what detection masks (Pipeline.set_detect_mask / push_masked) cost, and what they are for.  In one
invocation, at 752x480 with bench.py's configuration-2 parameters (EuRoC, UseUndistort=1), frames resident in device
memory and pushed as strided device frames by every arm:

  - the GPU's name and power limit (nvidia-smi);
  - four arms in alternating rounds, their order rotating from round to round: no mask; a fixed mask (the bottom 20 % of
    the rows and a 16-pixel frame); per-frame device masks (a disc that moves from frame to frame); the fixed mask set and
    cleared again.  64-frame batches and 1-frame pushes, --rounds rounds each: frames/s as a median with its range, the
    per-round ratio to no mask, and keylines per frame per arm;
  - k_detect_a against k_detect_a_masked kernel time from torch.profiler (CUDA activities), in a run of its own;
  - the use case as a number: a synthetic stream in which a textured patch moves against the scene, tracked unmasked and
    with the patch masked per frame; the RMS position error of each against the same stream without the patch.

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

ARMS = ("none", "fixed", "per_frame", "cleared")


def fixed_mask(h, w):
    m = np.full((h, w), 255, np.uint8)
    m[int(h * 0.8):] = 0
    m[:16] = m[:, :16] = m[:, -16:] = 0
    return m


def blob_masks(n, h, w, r, seed=0):
    """n masks, each zero on a disc of radius r whose centre walks across the frame."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    out = np.ones((n, h, w), np.uint8)
    cx, cy = w / 2, h / 2
    for i in range(n):
        cx = float(np.clip(cx + rng.uniform(-12, 12), r, w - r))
        cy = float(np.clip(cy + rng.uniform(-8, 8), r, h - r))
        out[i][(xx - cx) ** 2 + (yy - cy) ** 2 < r * r] = 0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=4, help="timed 64-frame batches per block")
    ap.add_argument("--pushes", type=int, default=64, help="timed 1-frame pushes per block")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_mask.py: no CUDA device (the measurement has no CPU path)")
    import bench
    from bench_mono import gpu_info, stats
    from rebvo_b200 import capi
    dev = 0
    torch.cuda.set_device(dev)
    out = {"what": "detection masks: no mask, fixed, per-frame device masks, fixed then cleared", "gpu": gpu_info(dev),
           "rounds": args.rounds}
    cam, params, _, _, seed0 = bench.stream_setup(2)
    kc = bench.undistort_of(2)
    h, w = cam["h"], cam["w"]
    B = 64
    total = (args.warmup + args.steps) * B
    ts, base, idx = bench.make_stream(seed0, total, base_n=40, cam=cam)
    frames = torch.from_numpy(np.ascontiguousarray(base[idx])).cuda()
    masks = torch.from_numpy(blob_masks(total, h, w, 0.15 * h)).cuda()
    F = fixed_mask(h, w)
    torch.cuda.synchronize()

    def pipeline(arm):
        pl = capi.Pipeline(params, max_batch=B, device=dev)
        pl.set_undistort(kc)
        if arm in ("fixed", "cleared"):
            pl.set_detect_mask(F)
        return pl

    pls = {a: pipeline(a) for a in ARMS}
    # the cleared arm: masked pushes first, then the mask cleared
    pls["cleared"].push_frames(frames[:B], ts[:B])
    pls["cleared"].set_detect_mask(None)

    def push(arm, s, n):
        pl = pls[arm]
        if arm == "per_frame":
            return pl.push_masked(frames[s:s + n], masks[s:s + n], ts[s:s + n])
        return pl.push_frames(frames[s:s + n], ts[s:s + n])

    def block(arm, n, count):
        pl = pls[arm]
        pl.reset()
        s = 0
        for _ in range(args.warmup):
            push(arm, s, n)
            s += n
        kn = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(count):
            nav = push(arm, s, n)
            kn += list(nav["kn"])
            s += n
        torch.cuda.synchronize()
        return count * n / (time.perf_counter() - t0), float(np.mean(kn))

    for name, n, count in (("batch64", B, args.steps), ("push1", 1, args.pushes)):
        fps = {a: [] for a in ARMS}
        kls = {a: [] for a in ARMS}
        for r in range(args.rounds):
            order = ARMS[r % len(ARMS):] + ARMS[:r % len(ARMS)]
            for a in order:
                f, k = block(a, n, count)
                fps[a].append(f)
                kls[a].append(k)
        out[name] = {a: {"fps": stats(fps[a]), "keylines_per_frame": float(np.mean(kls[a])),
                         "ratio_to_none": [x / y for x, y in zip(fps[a], fps["none"])]} for a in ARMS}

    # ---- kernel time, in a run of its own ----------------------------------------------------------------------------
    from torch.profiler import ProfilerActivity, profile
    for a in ("none", "fixed"):
        pls[a].reset()
        push(a, 0, B)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for a in ("none", "fixed"):
            for k in range(1, 3):
                push(a, k * B, B)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        nm = e.name
        if "k_detect_a" not in nm:
            continue
        key = "k_detect_a_masked" if "k_detect_a_masked" in nm else "k_detect_a"
        t = getattr(e, "device_time", None)
        if t is None:
            t = getattr(e, "cuda_time", 0.0)
        kern.setdefault(key, []).append(float(t))
    out["kernel_us"] = {k: {"calls": len(v), "mean_us": float(np.mean(v)), "median_us": float(np.median(v))}
                        for k, v in kern.items()}
    for pl in pls.values():
        pl.close()

    # ---- the use case: a textured patch that moves on its own -----------------------------------------------------------
    from rebvo_b200 import synth
    n_uc = 160
    seq = synth.Sequence(w=w, h=h, seed=11, zf=cam["zfx"])
    ts_uc, clean = seq.frames(n_uc)
    rng = np.random.default_rng(5)
    pw, ph = 200, 160
    patch = synth.to_rgb_u8(synth.rect_canvas(rng, pw, ph, 40), rng)
    dirty = clean.copy()
    pm = np.ones((n_uc, h, w), np.uint8)
    for i in range(n_uc):
        x0 = int(60 + 300 * (0.5 + 0.5 * np.sin(i / 9.0)))
        y0 = int(80 + 120 * (0.5 + 0.5 * np.cos(i / 13.0)))
        dirty[i, y0:y0 + ph, x0:x0 + pw] = patch
        pm[i, max(0, y0 - 4):y0 + ph + 4, max(0, x0 - 4):x0 + pw + 4] = 0
    pm_dev = torch.from_numpy(pm).cuda()
    pu = capi.default_params(cam)

    def track(fr, m=None):
        pl = capi.Pipeline(pu, max_batch=16, device=dev)
        navs = []
        for s in range(0, n_uc, 16):
            if m is None:
                navs.append(pl.push(fr[s:s + 16], ts_uc[s:s + 16]))
            else:
                navs.append(pl.push_masked(fr[s:s + 16], m[s:s + 16], ts_uc[s:s + 16]))
        pl.close()
        return np.concatenate(navs)

    ref = track(clean)
    unm = track(dirty)
    msk = track(dirty, pm_dev)

    def ate(a):
        d = np.asarray(a["Pos"], np.float64) - np.asarray(ref["Pos"], np.float64)
        return float(np.sqrt(np.mean(np.sum(d * d, axis=1))))

    out["moving_patch"] = {"frames": n_uc, "patch_px": [pw, ph], "ate_unmasked": ate(unm), "ate_masked": ate(msk),
                           "kn_clean": float(np.mean(ref["kn"])), "kn_unmasked": float(np.mean(unm["kn"])),
                           "kn_masked": float(np.mean(msk["kn"]))}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

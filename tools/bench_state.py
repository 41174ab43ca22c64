#!/usr/bin/env python
"""bench_state.py -- size and wall time of session checkpoints (rb_pipeline_save_state / rb_pipeline_load_state).

Two configurations: 752x480 with the EuRoC parameters and undistortion (the seed-7 stream of bench.py, ~15 k keylines per
map), and the 1280x960 synthetic stream of bench.py --config 4 with its parameters (~30 k keylines).  For each, a pipeline
tracks `--frames` frames so that the newest map is a converged one, then in `--rounds` rounds, alternating the order of
the two from round to round:
  - `--calls` saves into a preallocated host buffer (ctypes), each timed alone with a host clock (the call is synchronous);
  - `--calls` loads of that blob into a second pipeline of the same geometry, timed the same way.
Reported per configuration: blob bytes, keylines and bytes per keyline, and the median, min and max of the per-call
times over all rounds.  The GPU's name and power limit are read in the same invocation.  Prints one JSON line (and writes
it to --out if given).  Needs a CUDA device: there is no CPU path.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

EUROC_KC = (-0.28340811, 0.07395907, 0.0, 0.00019359, 1.76187114e-05)
BIG_CAM = dict(w=1280, h=960, zfx=780.0, zfy=778.0, ppx=640.5, ppy=479.25)   # bench.py --config 4


def gpu_info(dev=0):
    info = {"name": None, "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=60).stdout.strip().split(", ")
        if len(out) == 2:
            info = {"name": out[0], "power_limit_w": float(out[1])}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        pass
    return info


def config(name, n):
    from rebvo_b200 import capi, synth
    if name == "752x480":
        seq = synth.Sequence(w=synth.EUROC["w"], h=synth.EUROC["h"], seed=7, zf=synth.EUROC["zfx"])
        return capi.default_params(synth.EUROC), EUROC_KC, seq.frames(n)
    seq = synth.Sequence(w=BIG_CAM["w"], h=BIG_CAM["h"], seed=100, zf=BIG_CAM["zfx"], nrect_bg=1500, nrect_fg=200)
    p = capi.default_params(BIG_CAM, kl_ref=30000, kl_max=40000, TrackPoints=24000, kl_capacity=40000)
    return p, None, seq.frames(n)


def stats(v):
    v = np.asarray(v) * 1e3
    return {"median_ms": float(np.median(v)), "min_ms": float(v.min()), "max_ms": float(v.max()), "calls": int(len(v))}


def bench(name, args):
    from rebvo_b200 import capi
    params, kc, (ts, fr) = config(name, args.frames)
    src, dst = capi.Pipeline(params, max_batch=8), capi.Pipeline(params, max_batch=8)
    try:
        for pl in (src, dst):
            if kc is not None:
                pl.set_undistort(kc)
        for s in range(0, args.frames, 8):
            src.push(fr[s:s + 8], ts[s:s + 8])
        blob = src.save_state()
        info = capi.state_info(blob)
        L = src.L
        buf = C.create_string_buffer(len(blob))
        need = C.c_size_t(0)
        saves, loads = [], []

        def one_save():
            t0 = time.perf_counter()
            r = L.rb_pipeline_save_state(src.h_, buf, C.c_size_t(len(blob)), C.byref(need))
            saves.append(time.perf_counter() - t0)
            src.check(r)

        def one_load():
            t0 = time.perf_counter()
            r = L.rb_pipeline_load_state(dst.h_, blob, C.c_size_t(len(blob)))
            loads.append(time.perf_counter() - t0)
            dst.check(r)
        for _ in range(3):   # warm-up: staging buffers, first launches
            one_save()
            one_load()
        saves.clear()
        loads.clear()
        for k in range(args.rounds):
            arms = [one_save, one_load] if k % 2 == 0 else [one_load, one_save]
            for arm in arms:
                for _ in range(args.calls):
                    arm()
        assert buf.raw[:need.value] == blob, "a save of the unchanged session gave other bytes"
        assert dst.save_state() == blob, "the loaded session saves other bytes"
        return {"config": name, "blob_bytes": len(blob), "keylines": info["kn"],
                "bytes_per_keyline": len(blob) / max(1, info["kn"]), "save": stats(saves), "load": stats(loads),
                "rounds": args.rounds, "calls_per_round": args.calls}
    finally:
        src.close()
        dst.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--frames", type=int, default=24, help="frames tracked before the checkpoint")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--calls", type=int, default=20, help="calls per arm and round")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"gpu": gpu_info(), "results": [bench(n, args) for n in ("752x480", "1280x960")]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

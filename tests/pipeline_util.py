"""Helpers shared by the pipeline tests: the EuRoC-like stream, one push and one run of the fused pipeline, one run of
the reference executables on the same frames, and the comparisons and parity bars applied to what they return.  torch,
capi and refapi are imported inside the functions, so that tests without a GPU can use this module too."""
import collections
import os

import numpy as np
import pytest

# EuRoC cam0 radial-tangential coefficients (KcR2, KcR4, KcR6, KcP1, KcP2): GlobalConfig_EuRoC_2.txt:64-68
EUROC_KC = (-0.28340811, 0.07395907, 0.0, 0.00019359, 1.76187114e-05)


# ---- streams ----------------------------------------------------------------------------------------------------------
def euroc_sequence(seed=7, **seq_kw):
    """The seeded 752x480 stream with the EuRoC camera (synth.Sequence; imu_samples needs it)."""
    from rebvo_b200 import synth
    cam = synth.EUROC
    return synth.Sequence(w=cam["w"], h=cam["h"], seed=seed, zf=cam["zfx"], **seq_kw)


def euroc_stream(n, seed=7, **seq_kw):
    """(ts, frames): the first n frames of euroc_sequence(seed)."""
    return euroc_sequence(seed, **seq_kw).frames(n)


def walk(seq, n, base_n):
    """n frames of a continuous sequence built from base_n rendered frames walked back and forth (as bench.py)."""
    base_n = min(base_n, n)
    _, base = seq.frames(base_n)
    period = max(1, 2 * (base_n - 1))
    idx = np.arange(n) % period
    idx = np.where(idx < base_n, idx, period - idx)
    return np.arange(n) / 20.0, base[idx]


# ---- the fused pipeline -----------------------------------------------------------------------------------------------
def push(pl, frames, ts, how="host", offset=0):
    """One push of `frames` (RGB24 [n, h, w, 3] or mono [n, h, w]) from host memory, or from a device buffer in which
    they start `offset` bytes past an aligned allocation (freed after the push)."""
    mono = frames.ndim == 3
    if how == "host":
        return pl.push_mono(frames, ts) if mono else pl.push(frames, ts)
    import torch
    flat = torch.from_numpy(np.ascontiguousarray(frames).reshape(-1))
    buf = torch.zeros(flat.numel() + offset + 8, dtype=torch.uint8, device="cuda")
    buf[offset:offset + flat.numel()] = flat.cuda()
    # the pipeline's stream does not wait for torch's: the frames must be in the buffer before the push reads them
    torch.cuda.synchronize()
    try:
        return (pl.push_mono_dev if mono else pl.push_dev)(buf.data_ptr() + offset, ts)
    finally:
        del buf


Run = collections.namedtuple("Run", "nav maps mirrors counters odometry launches")


def run_pipeline(params, ts, frames, batch, how="host", fmt="rgb", offset=0, kc=None, mirror=0, imu=None,
                 odometry=False, collect=(), check_mirror=False):
    """The frames pushed through one Pipeline in `batch`-frame pushes.  fmt: "rgb", "mono" (the first channel of the RGB
    frames) or a list with one of the two per push, taken in turn.  imu: the samples of IMU mode.  `collect` names what
    the Run holds besides nav: "maps" (keylines and mask of the two newest maps after the last push), "mirrors" (every
    frame's mirror records), "counters" (the newest map's after every push), "odometry" (every frame's record),
    "launches" (per push).  check_mirror: after every push, its last frame's mirror records are those the newest map
    gives itself.  Environment switches are the caller's (monkeypatch) and stay set for the whole run."""
    from rebvo_b200 import capi
    pl = capi.Pipeline(params, max_batch=batch)
    out = {k: [] for k in collect}
    try:
        if kc is not None:
            pl.set_undistort(kc)
        if mirror:
            pl.set_mirror(mirror)
        if imu is not None:
            pl.set_imu(imu, capi.default_imu_params(InitBias=1, InitBiasFrameNum=5))
        if odometry:
            pl.set_odometry(True)
        navs = []
        for k, s in enumerate(range(0, len(ts), batch)):
            f = fmt if isinstance(fmt, str) else fmt[k % len(fmt)]
            src = frames[..., 0] if f == "mono" else frames
            l0 = pl.launches()
            nav = push(pl, src[s:s + batch], ts[s:s + batch], how, offset)
            navs.append(nav)
            if "launches" in out:
                out["launches"].append(pl.launches() - l0)
            if "mirrors" in out:
                out["mirrors"] += [pl.mirror(i).copy() for i in range(len(nav))]
            if "counters" in out:
                out["counters"].append(pl.map(0).counters())
            if "odometry" in out:
                out["odometry"].append(pl.odometry())
            if check_mirror:
                i, m = len(nav) - 1, pl.map(0)
                want = m.keylines() if mirror == 1 else m.pack_net(float(nav[i]["K"]))
                got = pl.mirror(i)
                assert len(got) == len(want) == nav[i]["kn"]
                assert got.tobytes() == np.ascontiguousarray(want).tobytes(), "mirror %d, frame %d" % (mirror, s + i)
        if "maps" in out:
            out["maps"] = [(m.keylines(), m.mask()) for m in (pl.map(0), pl.map(1))]
    finally:
        pl.close()
    if "odometry" in out:
        out["odometry"] = np.concatenate(out["odometry"])
    return Run(np.concatenate(navs), *(out.get(k) for k in Run._fields[1:]))


# ---- the reference ----------------------------------------------------------------------------------------------------
def shim_exe():
    """oracle/_ref/shim_rebvo: the reference's unmodified REBVO on include/rebvo_b200_shim.hpp."""
    from oracle import refapi
    return os.path.join(os.path.dirname(refapi.EXE), "shim_rebvo")


def frames_file(tmp_path, ts, frames):
    """The frames in the raw file the reference drivers read; returns its path."""
    from rebvo_b200 import synth
    path = str(tmp_path / "frames.bin")
    synth.write_frames_file(path, ts, frames)
    return path


def run_reference(tmp_path, ts, frames, params=None, exe=None, kc=None, imu=None, timeout=600, required=True, **kv):
    """(info, records) of the reference's three-thread REBVO on the frames: exe is refapi.EXE (the default), shim_exe()
    or build_pose_graph.EXE.  Its parameters are refapi.ref_params_from(params) when params are given, then kv; kc
    switches on the undistortion and imu (the samples) IMU mode.  When exe is missing the test is skipped, or None is
    returned if the run is not `required`."""
    from oracle import refapi
    from rebvo_b200 import synth
    exe = exe or refapi.EXE
    if not os.path.exists(exe):
        if not required:
            return None
        pytest.skip("oracle/_ref/%s not built" % os.path.basename(exe))
    if kc is not None:
        kv.update(UseUndistort=1, KcR2=kc[0], KcR4=kc[1], KcR6=kc[2], KcP1=kc[3], KcP2=kc[4])
    if imu is not None:
        csv = str(tmp_path / "imu.csv")
        synth.write_imu_csv(csv, imu)
        kv.update(ImuMode=2, ImuFile=csv, ImuTimeScale=1, InitBias=1, InitBiasFrameNum=5)
    if params is not None:
        kv = refapi.ref_params_from(params, **kv)
    path = frames_file(tmp_path, ts, frames)
    try:
        return refapi.run_full_rebvo(path, path + ".out", kv, timeout=timeout, exe=exe)
    finally:
        os.remove(path)


def trim(a, b):
    """a and b cut to their common length."""
    n = min(len(a), len(b))
    return a[:n], b[:n]


def run_both(tmp_path, ts, frames, params, batch=20):
    """(reference records, pipeline nav records) of the same frames and parameters, cut to their common length."""
    _, rec = run_reference(tmp_path, ts, frames, params, timeout=1500)
    return trim(rec, run_pipeline(params, ts, frames, batch).nav)


# ---- comparisons ------------------------------------------------------------------------------------------------------
def raw(nav):
    return np.ascontiguousarray(nav).view(np.uint8)


def keylines_equal(a, b):
    from rebvo_b200 import capi
    if len(a) != len(b):
        return False
    return all(np.array_equal(a[f], b[f], equal_nan=True) for f in capi.KEYLINE.names)


def assert_runs_identical(a, b, what):
    """Two Runs give the same bits: raw nav records, then the maps, mirrors, counters and odometry records both hold."""
    assert len(a.nav) == len(b.nav), "%s: %d vs %d nav records" % (what, len(a.nav), len(b.nav))
    diff = np.nonzero((raw(a.nav) != raw(b.nav)).reshape(len(a.nav), -1).any(1))[0]
    assert len(diff) == 0, "%s: nav records differ from frame %d" % (what, diff[0])
    if a.maps is not None and b.maps is not None:
        for age, ((kl_a, mask_a), (kl_b, mask_b)) in enumerate(zip(a.maps, b.maps)):
            assert keylines_equal(kl_a, kl_b), "%s: keylines of map %d" % (what, age)
            assert np.array_equal(mask_a, mask_b), "%s: mask of map %d" % (what, age)
    if a.mirrors is not None and b.mirrors is not None:
        assert len(a.mirrors) == len(b.mirrors)
        for i, (x, y) in enumerate(zip(a.mirrors, b.mirrors)):
            ok = np.array_equal(x, y) if x.dtype == np.uint8 else keylines_equal(x, y)
            assert ok, "%s: mirror records of frame %d" % (what, i)
    if a.counters is not None and b.counters is not None:
        for i, (x, y) in enumerate(zip(a.counters, b.counters)):
            assert x == y, "%s: push %d: (fwd_match, nmatch, reg_num) %r against %r" % (what, i, x, y)
    if a.odometry is not None and b.odometry is not None:
        assert np.array_equal(raw(a.odometry), raw(b.odometry)), "%s: odometry records" % what


def _est_ok(r):
    return r["est_ok"] if "est_ok" in r.dtype.names else r["estimation_ok"]


def assert_counts_equal(rec, nav):
    """Equal keyline counts, match counts and estimation_ok (the first frame's match count is not compared)."""
    assert np.array_equal(rec["kn"], nav["kn"]), np.nonzero(rec["kn"] != nav["kn"])[0][:10]
    bad = np.nonzero(rec["matches"][1:] != nav["matches"][1:])[0] + 1
    assert not len(bad), "match counts differ at frames %s: ref %s gpu %s" % (bad[:5], rec["matches"][bad[:5]],
                                                                             nav["matches"][bad[:5]])
    assert np.array_equal(_est_ok(rec)[1:] != 0, _est_ok(nav)[1:] != 0)


def assert_tight(rec, nav, min_frames):
    """The bar of a run that follows the reference's arithmetic: equal counts, ATE <= 1e-7 m, Kp within rtol 1e-8.
    Returns refapi.trajectory_parity."""
    from oracle import refapi
    rec, nav = trim(rec, nav)
    par = refapi.trajectory_parity(rec, nav)
    print(par)
    assert par["frames"] >= min_frames
    assert_counts_equal(rec, nav)
    assert par["ate_m"] <= 1e-7, par
    assert np.allclose(rec["Kp"][1:], nav["Kp"][1:], rtol=1e-8, atol=0)
    return par


def assert_knife_edge(ref, nav, min_frames, what=""):
    """The bar against the CPU reference, whose sums run in another order: a frame whose LM decision sits on a knife
    edge may take the other branch.  Equal kn and estimation_ok, matches within 0.5 % of the largest count, ATE and
    largest position error <= 1e-3 m."""
    ref, nav = trim(ref, nav)
    n = len(ref)
    assert n >= min_frames
    e = np.sqrt(((ref["Pos"] - nav["Pos"]) ** 2).sum(1))
    ate = float(np.sqrt((e ** 2).mean()))
    first = int(np.nonzero(e > 1e-9)[0][0]) if (e > 1e-9).any() else -1
    dm = np.abs(ref["matches"][1:].astype(int) - nav["matches"][1:].astype(int))
    print("%s: ATE %.3e m, max %.3e m over %d frames, first frame above 1e-9 m: %d, max |d matches| %d, kn %d..%d" % (
        what, ate, e.max(), n, first, dm.max(), nav["kn"].min(), nav["kn"].max()))
    assert np.array_equal(ref["kn"], nav["kn"])
    assert np.array_equal(_est_ok(ref)[1:] != 0, _est_ok(nav)[1:] != 0)
    assert dm.max() <= 0.005 * ref["matches"][1:].max(), dm.max()
    assert ate <= 1e-3 and e.max() <= 1e-3


def assert_shim_equals(nav, rec):
    """The reference's REBVO on the shim (rec) and the fused pipeline (nav) on the same frames: equal kn and matches,
    positions within 1e-9 m."""
    nav, rec = trim(nav, rec)
    assert np.array_equal(nav["kn"], rec["kn"])
    assert np.array_equal(nav["matches"][1:], rec["matches"][1:])
    d = np.abs(nav["Pos"] - rec["Pos"]).max()
    print("shim vs pipeline max |dPos| %.3e" % d)
    assert d <= 1e-9

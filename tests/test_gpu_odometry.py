"""Per-frame odometry records (rb_pipeline_set_odometry / rb_pipeline_odometry): the relative motion and information matrix
SecondThread appends to REBVO::poses (rebvo_second_t.cpp:323-334 IMU mode, :371-382 vision only), against the pose graph file
the reference's own 3-thread REBVO writes on the same frames (oracle/_ref/ref_rebvo_pg with PoseGraphFile=).  Also: the
match-count restart that sets QK, the empty old map, the records across schedules and resets, and that the records leave the
nav records and the launches of a push unchanged."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ZERO_FIELDS = ("AcelMeas", "VisualMeas", "GMeas", "Rs", "Rv", "Rg")


def _pushes(pl, fr, ts, batch, push="push"):
    navs, recs, launches = [], [], []
    for s in range(0, len(ts), batch):
        l0 = pl.launches()
        navs.append(getattr(pl, push)(fr[s:s + batch], ts[s:s + batch]))
        launches.append(pl.launches() - l0)
        recs.append(pl.odometry() if pl._odom else None)
    return np.concatenate(navs), (np.concatenate(recs) if pl._odom else None), launches


def _pipeline(params, batch, odom=True, env=None, monkeypatch=None):
    from rebvo_b200 import capi
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    pl = capi.Pipeline(params, max_batch=batch)
    for k in (env or {}):
        monkeypatch.delenv(k)
    pl._odom = odom
    if odom:
        pl.set_odometry(True)
    return pl


def _run(params, fr, ts, batch, odom=True, env=None, monkeypatch=None):
    pl = _pipeline(params, batch, odom, env, monkeypatch)
    try:
        return _pushes(pl, fr, ts, batch)
    finally:
        pl.close()


def _reference(tmp_path, params, fr, ts, **kv):
    from oracle import build_pose_graph, refapi
    from rebvo_b200 import capi, synth
    if not os.path.exists(build_pose_graph.EXE):
        pytest.skip("oracle/_ref/ref_rebvo_pg not built")
    path = str(tmp_path / "frames.bin")
    synth.write_frames_file(path, ts, fr)
    ps = str(tmp_path / "poses_list.ps")
    _, nav = refapi.run_full_rebvo(path, str(tmp_path / "out.bin"), refapi.ref_params_from(params, PoseGraphFile=ps, **kv),
                                   timeout=1500, exe=build_pose_graph.EXE)
    os.remove(path)
    return capi.read_pose_graph(ps), nav


def _euroc(n, seed=7):
    from rebvo_b200 import synth
    cam = synth.EUROC
    return synth.Sequence(w=cam["w"], h=cam["h"], seed=seed, zf=cam["zfx"]).frames(n)


def _w_err(ref, got):
    """per record: max |W_got - W_ref| / max |W_ref|"""
    scale = np.abs(ref["WrelPosPose"]).reshape(len(ref), -1).max(1)
    return np.abs(got["WrelPosPose"] - ref["WrelPosPose"]).reshape(len(ref), -1).max(1) / scale


def _raw(a):
    return np.ascontiguousarray(a).view(np.uint8)


def test_vision_records_match_reference(built, tmp_path):
    from rebvo_b200 import capi, synth
    ts, fr = _euroc(60)
    p = capi.default_params(synth.EUROC)
    ref, _ = _reference(tmp_path, p, fr, ts)
    _, odo, _ = _run(p, fr, ts, 7)
    assert len(odo) == 60 and odo["tracked"][0] == 0 and np.all(odo["tracked"][1:] == 1)
    got = odo[1:]
    assert len(ref) == len(got)
    dp = np.abs(got["relPosPose"] - ref["relPosPose"]).max()
    dw = _w_err(ref, got).max()
    dq = np.abs(got["QK"] / ref["QK"] - 1).max()
    print("vision: max |d relPosPose| %.3e, max per-record |d W| / max |W| %.3e, max rel |d QK| %.3e" % (dp, dw, dq))
    assert dp <= 1e-9
    assert dw <= 1e-8
    assert np.allclose(got["QK"], ref["QK"], rtol=1e-8, atol=0)
    for k in ("K", "WK", "KF_ID") + ZERO_FIELDS:
        assert np.array_equal(got[k], ref[k]), k
    # the pose graph file of the pipeline's records is the reference's layout: it parses back to the same values
    path = str(tmp_path / "gpu.ps")
    with open(path, "wb") as f:
        f.write(capi.format_pose_graph(odo))
    back = capi.read_pose_graph(path)
    assert np.array_equal(_raw(back), _raw(got))


def test_restart_branch_qk(built, tmp_path):
    """GlobalMatchThreshold above every frame's match count: every frame restarts, P_Kp = 10 from the second tracked frame on."""
    from rebvo_b200 import capi, synth
    ts, fr = _euroc(24)
    p = capi.default_params(synth.EUROC, MatchThreshold=10 ** 6)
    ref, _ = _reference(tmp_path, p, fr, ts)
    _, odo, _ = _run(p, fr, ts, 8)
    got = odo[1:]
    assert len(ref) == len(got)
    assert got["QK"][0] == 5e-6 and np.all(got["QK"][1:] == 10)
    assert np.array_equal(got["QK"], ref["QK"])
    assert np.abs(got["relPosPose"] - ref["relPosPose"]).max() <= 1e-9
    assert _w_err(ref, got).max() <= 1e-8


def test_black_frame_and_empty_old_map(built, tmp_path):
    """A black frame 6 (an empty edge map): no old keyline finds a match, the match-count gate restarts (frame 7 finds
    P_Kp = 10, in the reference as here), and frame 7 tracks against the empty old map, for which the pipeline writes a
    zero information matrix (the reference's W_X is uninitialised there) and V is the prior; frame 8 restarts again."""
    from rebvo_b200 import capi, synth
    ts, fr = _euroc(14)
    fr = fr.copy()
    fr[6] = 0
    p = capi.default_params(synth.EUROC)
    ref, _ = _reference(tmp_path, p, fr, ts)
    nav, odo, _ = _run(p, fr, ts, 7)
    got = odo[1:]
    assert len(ref) == len(got)
    assert nav["kn"][6] == 0 and nav["estimation_ok"][6] == 0 and nav["estimation_ok"][7] == 0
    assert odo["QK"][7] == 10 and odo["QK"][8] == 10
    assert np.allclose(got["QK"], ref["QK"], rtol=1e-8, atol=0)
    empty = 7 - 1                                     # record r = frame r + 1
    assert np.array_equal(got["WrelPosPose"][empty], np.zeros((6, 6)))
    keep = np.ones(len(got), bool)
    keep[empty] = False
    assert np.isfinite(got["relPosPose"]).all() and np.isfinite(ref["relPosPose"]).all()
    assert np.abs(got["relPosPose"] - ref["relPosPose"]).max() <= 1e-9
    zero = np.abs(ref["WrelPosPose"]).reshape(len(ref), -1).max(1) == 0   # frame 6: nothing matched, JtJ = 0
    assert zero[6 - 1] and np.array_equal(got["WrelPosPose"][zero], ref["WrelPosPose"][zero])
    assert _w_err(ref[keep & ~zero], got[keep & ~zero]).max() <= 1e-8


def test_imu_mode_records_match_reference(built, tmp_path):
    from rebvo_b200 import capi, synth
    nf = 50
    cam = synth.EUROC
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=7, zf=cam["zfx"])
    ts, fr = seq.frames(nf)
    smp = synth.imu_samples(seq, nf)
    csv = str(tmp_path / "imu.csv")
    synth.write_imu_csv(csv, smp)
    p = capi.default_params(cam)
    ref, _ = _reference(tmp_path, p, fr, ts, ImuMode=2, ImuFile=csv, ImuTimeScale=1, InitBias=1, InitBiasFrameNum=5)
    pl = capi.Pipeline(p, max_batch=10)
    pl.set_imu(smp, capi.default_imu_params(InitBias=1, InitBiasFrameNum=5))
    pl._odom = True
    pl.set_odometry(True)
    _, odo, _ = _pushes(pl, fr, ts, 10)
    pl.close()
    assert odo["tracked"][0] == 0 and np.all(odo["tracked"][1:] == 1)
    got = odo[1:]
    # the reference's last record is not comparable: its first thread waits for that frame's inertial samples in a loop that
    # ends when the driver stops the threads (rebvo_first_t.cpp:294-301), so what it integrates depends on the shutdown
    n = min(len(ref) - 1, len(got))
    assert n >= nf - 3
    ref, got = ref[:n], got[:n]
    dp = np.abs(got["relPosPose"] - ref["relPosPose"]).max()
    dw = _w_err(ref, got).max()
    # the scale / gravity filter runs from n_frame > 4 + InitBiasFrameNum on (record r: n_frame = r); before that the
    # reference's g_est is uninitialised, the pipeline's zero
    start = 4 + 5 + 1
    assert not got["GMeas"][:start].any()
    rel, bad = {}, {}
    for k in ("AcelMeas", "VisualMeas", "GMeas", "Rs", "Rv", "Rg", "K", "WK", "QK"):
        s0 = start if k == "GMeas" else 0
        a, b = got[k][s0:].reshape(n - s0, -1), ref[k][s0:].reshape(n - s0, -1)
        rel[k] = float((np.abs(a - b) / np.maximum(np.abs(b), 1e-300)).max())
        if not np.allclose(a, b, rtol=1e-6, atol=0):
            bad[k] = rel[k]
    print("IMU: max |d relPosPose| %.3e, max per-record |d W| / max |W| %.3e, max rel errors %s" % (dp, dw, rel))
    assert np.array_equal(got["KF_ID"], ref["KF_ID"])
    assert dp <= 1e-6
    assert dw <= 1e-5
    assert not bad, bad


def test_records_leave_nav_and_launches_unchanged(built, monkeypatch):
    """With the records on, the nav records are bit-identical and a push launches exactly the kernels it launches without
    them (the constant of rb_pipeline_set_odometry is 0), in both map schedules; switching them off restores the launches."""
    from rebvo_b200 import capi, synth
    ts, fr = _euroc(40)
    p = capi.default_params(synth.EUROC)
    for env in ({}, {"REBVO_B200_MAP_CHAIN": "0"}):
        nav0, _, l0 = _run(p, fr, ts, 7, odom=False, env=env, monkeypatch=monkeypatch)
        nav1, _, l1 = _run(p, fr, ts, 7, odom=True, env=env, monkeypatch=monkeypatch)
        assert np.array_equal(_raw(nav0), _raw(nav1)), env
        assert l1 == l0, (env, l0, l1)
        pl = _pipeline(p, 7, True, env, monkeypatch)   # on for the first pushes, then off
        navs, lc = [], []
        for k, s in enumerate(range(0, len(ts), 7)):
            if k == 3:
                pl.set_odometry(False)
                pl._odom = False
                with pytest.raises(capi.RbError):
                    pl.odometry()
            n0 = pl.launches()
            navs.append(pl.push(fr[s:s + 7], ts[s:s + 7]))
            lc.append(pl.launches() - n0)
        pl.close()
        assert lc == l0, (env, l0, lc)
        assert np.array_equal(_raw(np.concatenate(navs)), _raw(nav0))


def test_records_same_across_schedules_and_resets(built, monkeypatch):
    """Bit-identical records from the default schedule, the reference map schedule (REBVO_B200_MAP_CHAIN=0) and the
    one-cluster minimiser (REBVO_B200_MIN_G=1), with host and device input; after rb_pipeline_reset the records are those of
    a fresh pipeline (first frame untracked, QK from 5e-6 again)."""
    import torch
    from rebvo_b200 import capi, synth
    ts, fr = _euroc(30)
    p = capi.default_params(synth.EUROC)
    nav_b, base, _ = _run(p, fr, ts, 7)
    _, odo, _ = _run(p, fr, ts, 7, env={"REBVO_B200_MAP_CHAIN": "0"}, monkeypatch=monkeypatch)
    assert np.array_equal(_raw(odo), _raw(base))
    # the one-cluster minimiser sums its reductions over one cluster instead of four: its nav records already differ from
    # the default's in the last bits, and so do the records (measured on H100: 2e-17 in relPosPose, 4e-14 of max |W|)
    nav_g, odo, _ = _run(p, fr, ts, 7, env={"REBVO_B200_MIN_G": "1"}, monkeypatch=monkeypatch)
    print("MIN_G=1: nav identical %s, max |d relPosPose| %.3e, W rel %.3e" %
          (np.array_equal(_raw(nav_g), _raw(nav_b)), np.abs(odo["relPosPose"] - base["relPosPose"]).max(),
           _w_err(base[1:], odo[1:]).max()))
    for k in ("K", "WK", "KF_ID", "tracked") + ZERO_FIELDS:
        assert np.array_equal(odo[k], base[k]), k
    assert np.abs(odo["relPosPose"] - base["relPosPose"]).max() <= 1e-15
    assert np.allclose(odo["QK"], base["QK"], rtol=1e-12, atol=0)
    assert _w_err(base[1:], odo[1:]).max() <= 1e-12
    pl = _pipeline(p, 10)
    dev = torch.from_numpy(np.ascontiguousarray(fr)).cuda()
    for s in range(0, 30, 10):   # device input, other batch size
        pl.push_dev(dev[s:s + 10].data_ptr(), ts[s:s + 10])
        assert np.array_equal(_raw(pl.odometry()), _raw(base[s:s + 10]))
    pl.reset()
    again = []
    for s in range(0, 30, 10):
        pl.push(fr[s:s + 10], ts[s:s + 10])
        again.append(pl.odometry())
    pl.close()
    again = np.concatenate(again)
    assert again["tracked"][0] == 0 and again["QK"][1] == 5e-6
    assert np.array_equal(_raw(again), _raw(base))

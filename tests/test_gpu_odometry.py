"""Per-frame odometry records (rb_pipeline_set_odometry / rb_pipeline_odometry): the relative motion and information matrix
SecondThread appends to REBVO::poses (rebvo_second_t.cpp:323-334 IMU mode, :371-382 vision only), against the pose graph file
the reference's own 3-thread REBVO writes on the same frames (oracle/_ref/ref_rebvo_pg with PoseGraphFile=).  Also: the
match-count restart that sets QK, the empty old map, the records across schedules and resets, and that the records leave the
nav records and the launches of a push unchanged."""
import numpy as np
import pytest

from pipeline_util import euroc_sequence, euroc_stream, push, raw, run_pipeline, run_reference

pytestmark = pytest.mark.gpu

ZERO_FIELDS = ("AcelMeas", "VisualMeas", "GMeas", "Rs", "Rv", "Rg")


def _records(params, ts, fr, batch, **kw):
    """nav and odometry records of the frames pushed with the records on, in `batch`-frame pushes"""
    r = run_pipeline(params, ts, fr, batch, odometry=True, collect=("odometry",), **kw)
    return r.nav, r.odometry


def _pose_graph(tmp_path, params, fr, ts, **kw):
    """the records of the pose graph file the reference writes on the frames"""
    from oracle import build_pose_graph
    from rebvo_b200 import capi
    ps = str(tmp_path / "poses_list.ps")
    run_reference(tmp_path, ts, fr, params, exe=build_pose_graph.EXE, timeout=1500, PoseGraphFile=ps, **kw)
    return capi.read_pose_graph(ps)


def _w_err(ref, got):
    """per record: max |W_got - W_ref| / max |W_ref|"""
    scale = np.abs(ref["WrelPosPose"]).reshape(len(ref), -1).max(1)
    return np.abs(got["WrelPosPose"] - ref["WrelPosPose"]).reshape(len(ref), -1).max(1) / scale


def test_vision_records_match_reference(built, tmp_path):
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(60)
    p = capi.default_params(synth.EUROC)
    ref = _pose_graph(tmp_path, p, fr, ts)
    _, odo = _records(p, ts, fr, 7)
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
    assert np.array_equal(raw(back), raw(got))


def test_restart_branch_qk(built, tmp_path):
    """GlobalMatchThreshold above every frame's match count: every frame restarts, P_Kp = 10 from the second tracked frame on."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(24)
    p = capi.default_params(synth.EUROC, MatchThreshold=10 ** 6)
    ref = _pose_graph(tmp_path, p, fr, ts)
    _, odo = _records(p, ts, fr, 8)
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
    ts, fr = euroc_stream(14)
    fr[6] = 0
    p = capi.default_params(synth.EUROC)
    ref = _pose_graph(tmp_path, p, fr, ts)
    nav, odo = _records(p, ts, fr, 7)
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
    seq = euroc_sequence()
    ts, fr = seq.frames(nf)
    smp = synth.imu_samples(seq, nf)
    p = capi.default_params(synth.EUROC)
    ref = _pose_graph(tmp_path, p, fr, ts, imu=smp)
    _, odo = _records(p, ts, fr, 10, imu=smp)
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
    ts, fr = euroc_stream(40)
    p = capi.default_params(synth.EUROC)
    for env in ({}, {"REBVO_B200_MAP_CHAIN": "0"}):
        with monkeypatch.context() as m:   # the map schedule is chosen at creation
            for k, v in env.items():
                m.setenv(k, v)
            off = run_pipeline(p, ts, fr, 7, collect=("launches",))
            on = run_pipeline(p, ts, fr, 7, odometry=True, collect=("launches",))
            pl = capi.Pipeline(p, max_batch=7)   # on for the first pushes, then off
        assert np.array_equal(raw(off.nav), raw(on.nav)), env
        assert on.launches == off.launches, (env, off.launches, on.launches)
        pl.set_odometry(True)
        navs, lc = [], []
        for k, s in enumerate(range(0, len(ts), 7)):
            if k == 3:
                pl.set_odometry(False)
                with pytest.raises(capi.RbError):
                    pl.odometry()
            n0 = pl.launches()
            navs.append(push(pl, fr[s:s + 7], ts[s:s + 7]))
            lc.append(pl.launches() - n0)
        pl.close()
        assert lc == off.launches, (env, off.launches, lc)
        assert np.array_equal(raw(np.concatenate(navs)), raw(off.nav))


def test_records_same_across_schedules_and_resets(built, monkeypatch):
    """Bit-identical records from the default schedule, the reference map schedule (REBVO_B200_MAP_CHAIN=0) and the
    one-cluster minimiser (REBVO_B200_MIN_G=1), with host and device input; after rb_pipeline_reset the records are those of
    a fresh pipeline (first frame untracked, QK from 5e-6 again)."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(30)
    p = capi.default_params(synth.EUROC)
    nav_b, base = _records(p, ts, fr, 7)
    with monkeypatch.context() as m:
        m.setenv("REBVO_B200_MAP_CHAIN", "0")
        _, odo = _records(p, ts, fr, 7)
    assert np.array_equal(raw(odo), raw(base))
    # the one-cluster minimiser sums its reductions over one cluster instead of four: its nav records already differ from
    # the default's in the last bits, and so do the records (measured on H100: 2e-17 in relPosPose, 4e-14 of max |W|)
    with monkeypatch.context() as m:
        m.setenv("REBVO_B200_MIN_G", "1")
        nav_g, odo = _records(p, ts, fr, 7)
    print("MIN_G=1: nav identical %s, max |d relPosPose| %.3e, W rel %.3e" %
          (np.array_equal(raw(nav_g), raw(nav_b)), np.abs(odo["relPosPose"] - base["relPosPose"]).max(),
           _w_err(base[1:], odo[1:]).max()))
    for k in ("K", "WK", "KF_ID", "tracked") + ZERO_FIELDS:
        assert np.array_equal(odo[k], base[k]), k
    assert np.abs(odo["relPosPose"] - base["relPosPose"]).max() <= 1e-15
    assert np.allclose(odo["QK"], base["QK"], rtol=1e-12, atol=0)
    assert _w_err(base[1:], odo[1:]).max() <= 1e-12
    pl = capi.Pipeline(p, max_batch=10)
    pl.set_odometry(True)
    for s in range(0, 30, 10):   # device input, other batch size
        push(pl, fr[s:s + 10], ts[s:s + 10], "device")
        assert np.array_equal(raw(pl.odometry()), raw(base[s:s + 10]))
    pl.reset()
    again = []
    for s in range(0, 30, 10):
        push(pl, fr[s:s + 10], ts[s:s + 10])
        again.append(pl.odometry())
    pl.close()
    again = np.concatenate(again)
    assert again["tracked"][0] == 0 and again["QK"][1] == 5e-6
    assert np.array_equal(raw(again), raw(base))

"""Whole-pipeline parity: rb_pipeline_push (device-resident REBVO flow) against the reference's own 3-thread
REBVO class (oracle/_ref/ref_rebvo, built from the unmodified sources) on the same synthetic 752x480 stream.

Bars (north_star): identical keyline counts per frame (integer work is bit-exact), directed-matching counts equal,
pose ATE <= 1e-3 m (here the streams are deterministic, so the observed ATE is ~1e-9); batch size must not
change the result (frames are processed in order)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NF = 60


@pytest.fixture(scope="module")
def stream():
    from rebvo_b200 import synth
    cam = synth.EUROC
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=7, zf=cam["zfx"])
    return seq.frames(NF)


@pytest.fixture(scope="module")
def ref_run(stream, tmp_path_factory):
    from oracle import refapi
    from rebvo_b200 import synth
    if not os.path.exists(refapi.EXE):
        pytest.skip("oracle/_ref/ref_rebvo not built")
    d = tmp_path_factory.mktemp("ref")
    ts, fr = stream
    path = str(d / "frames.bin")
    synth.write_frames_file(path, ts, fr)
    info, rec = refapi.run_full_rebvo(path, str(d / "out.bin"))
    os.remove(path)
    return info, rec


def _gpu_run(stream, batch):
    from rebvo_b200 import capi, synth
    ts, fr = stream
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=batch)
    navs = []
    for s in range(0, NF, batch):
        navs.append(pl.push(fr[s:s + batch], ts[s:s + batch]))
    launches = pl.launches()
    pl.close()
    return np.concatenate(navs), launches


def test_trajectory_vs_reference(built, stream, ref_run):
    info, rec = ref_run
    nav, launches = _gpu_run(stream, 20)
    n = min(len(rec), NF - 1)
    assert n >= NF - 2
    print("ref fps %.1f, launches/frame %.1f" % (info["fps"], launches / NF))
    kn_ref, kn_gpu = rec["kn"][:n], nav["kn"][:n]
    assert np.array_equal(kn_ref, kn_gpu), "keyline counts differ at frames %s" % np.nonzero(kn_ref != kn_gpu)[0][:10]
    m_ref, m_gpu = rec["matches"][1:n], nav["matches"][1:n]
    assert np.array_equal(m_ref, m_gpu), "match counts differ: %s vs %s" % (m_ref[:10], m_gpu[:10])
    d = rec["Pos"][:n] - nav["Pos"][:n]
    ate = float(np.sqrt((d ** 2).sum(1).mean()))
    mx = float(np.sqrt((d ** 2).sum(1)).max())
    path_len = float(np.linalg.norm(np.diff(rec["Pos"][:n], axis=0), axis=1).sum())
    print("ATE rmse %.3e m, max %.3e m over %d frames (path length %.3f)" % (ate, mx, n, path_len))
    assert path_len > 1e-3, "degenerate trajectory"
    assert ate <= 1e-3
    assert ate <= 1e-7, "expected near bit-level agreement on a deterministic stream"
    dl = np.abs(rec["PoseLie"][:n] - nav["PoseLie"][:n]).max()
    print("max |PoseLie diff| %.3e rad" % dl)
    assert dl <= 1e-7
    assert np.allclose(rec["Kp"][1:n], nav["Kp"][1:n], rtol=1e-9, atol=0)
    assert np.array_equal(rec["est_ok"][1:n] != 0, nav["estimation_ok"][1:n] != 0)
    try:
        os.makedirs("gpurun_out", exist_ok=True)
        np.savez("gpurun_out/trajectory_parity.npz", ref_pos=rec["Pos"][:n], gpu_pos=nav["Pos"][:n], ate=ate)
    except OSError:
        pass


def test_batch_size_invariance(built, stream, monkeypatch):
    a, _ = _gpu_run(stream, 20)
    b, _ = _gpu_run(stream, 7)
    c, _ = _gpu_run(stream, 1)
    # host-input pushes of >= 3 x REBVO_B200_SUB frames are cut into a head and the rest (copy/compute overlap)
    monkeypatch.setenv("REBVO_B200_SUB", "5")
    d, _ = _gpu_run(stream, 20)
    for f in ("Pos", "Pose", "kn", "matches", "Kp"):
        assert np.array_equal(a[f], b[f]) and np.array_equal(a[f], c[f]) and np.array_equal(a[f], d[f]), f


def test_device_input_equals_host_input(built, stream):
    """rb_pipeline_push_dev reads the caller's device buffer in place; same bits as the host-input path."""
    import torch
    from rebvo_b200 import capi, synth
    ts, fr = stream
    a, _ = _gpu_run(stream, 20)
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=20)
    navs = []
    for s in range(0, NF, 20):
        dev = torch.from_numpy(np.ascontiguousarray(fr[s:s + 20])).cuda()
        navs.append(pl.push_dev(dev.data_ptr(), ts[s:s + 20]))
        del dev
    pl.close()
    b = np.concatenate(navs)
    for f in ("Pos", "Pose", "kn", "matches", "Kp"):
        assert np.array_equal(a[f], b[f]), f


def test_graph_replay_equals_eager_launches(built, stream, monkeypatch):
    """Batches after the first are replayed as a CUDA graph; the eager path must give the same bits."""
    a, la = _gpu_run(stream, 10)
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    b, lb = _gpu_run(stream, 10)
    assert la == lb, "launch accounting differs between graph replay and eager launches"
    for f in ("Pos", "Pose", "kn", "matches", "Kp", "score"):
        assert np.array_equal(a[f], b[f]), f


@pytest.mark.parametrize("env", [{"REBVO_B200_MIN_EARLY": "0"}, {"REBVO_B200_PRIO": "0"}])
def test_schedule_variants_do_not_change_the_result(built, stream, monkeypatch, env):
    """Switches that only change when or where work runs (operand staging after the PDL wait, stream priorities): same
    arithmetic in the same order, hence the same bits -- also across a batch boundary and a graph replay."""
    a, _ = _gpu_run(stream, 20)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    b, lb = _gpu_run(stream, 20)
    for f in ("Pos", "Pose", "kn", "matches", "Kp", "score", "s_rho_p"):
        assert np.array_equal(a[f], b[f]), (env, f)
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    c, lc = _gpu_run(stream, 7)   # other batch size, eager
    assert np.array_equal(a["Pos"], c["Pos"]) and np.array_equal(a["s_rho_p"], c["s_rho_p"])


def test_fallback_paths_agree(built, stream, monkeypatch):
    """The switches in DESIGN.md section 5 select the slower formulations of the same stages (one launch per TryVelRot
    evaluation, detector on the tracker stream, plain stream order): same keylines and matches, poses equal to the
    rounding of the differently ordered sums."""
    a, _ = _gpu_run(stream, 20)
    for k in ("REBVO_B200_MIN_PERSIST", "REBVO_B200_OVERLAP", "REBVO_B200_PDL"):
        monkeypatch.setenv(k, "0")
    b, _ = _gpu_run(stream, 20)
    assert np.array_equal(a["kn"], b["kn"])                       # the detector does not depend on the tracker
    assert np.abs(a["matches"].astype(int) - b["matches"].astype(int)).max() <= 3   # a threshold decision may flip
    assert np.abs(a["Pos"] - b["Pos"]).max() <= 1e-6
    assert np.abs(a["Kp"] - b["Kp"]).max() <= 1e-6


def test_keyline_mirror_matches_reference_layout(built, stream):
    """The 168-byte AoS mirror handed to host consumers (callback / net packer) is populated and consistent."""
    from rebvo_b200 import capi, synth
    ts, fr = stream
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=4)
    nav = pl.push(fr[:4], ts[:4])
    m = pl.map(0)
    kl = m.keylines()
    assert len(kl) == nav["kn"][3] and capi.KEYLINE.itemsize == 168
    mask = m.mask()
    assert (mask >= 0).sum() == len(kl)
    assert np.array_equal(mask.ravel()[kl["p_inx"]], np.arange(len(kl)))
    assert (kl["m_id"] >= 0).sum() == nav["matches"][3] or (kl["m_id"] >= 0).sum() >= nav["matches"][3]
    assert np.all(kl["rho"] > 0) and np.all(kl["s_rho"] > 0)
    pl.close()


def test_host_mirror(built, stream):
    """rb_pipeline_set_mirror: the per-frame records written to host memory during the push equal, for every frame, what the stage calls
    return when the same stream is pushed one frame at a time (so that every frame is once the newest map): mode 1 =
    KeyLine AoS vs rb_map_sync_host_keylines field by field, mode 2 = net_keyline records vs rb_map_pack_net_keylines with
    the frame's K (itself bit-exact against the reference's packer, test_gpu_netpack.py).  The poses do not change."""
    from rebvo_b200 import capi, synth
    ts, fr = stream
    got = {}
    for mode in (1, 2):
        pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=20)
        pl.set_mirror(mode)
        navs, mirrors = [], []
        for s in range(0, NF, 20):
            nav = pl.push(fr[s:s + 20], ts[s:s + 20])
            navs.append(nav)
            for i in range(len(nav)):
                m = pl.mirror(i)
                assert len(m) == nav["kn"][i]
                mirrors.append(m.copy())
        pl.close()
        got[mode] = (np.concatenate(navs), mirrors)
    nav, aos = got[1]
    assert np.array_equal(got[2][0]["Pos"], nav["Pos"])
    one = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=1)
    for f in range(NF):
        nav1 = one.push(fr[f:f + 1], ts[f:f + 1])
        assert np.array_equal(nav1["Pos"][0], nav["Pos"][f])
        kl = one.map(0).keylines()
        assert len(kl) == len(aos[f])
        for name in capi.KEYLINE.names:
            assert np.array_equal(kl[name], aos[f][name], equal_nan=True), "frame %d field %s" % (f, name)
        net = one.map(0).pack_net(k_prof=float(nav1["K"][0]))
        assert len(net) == len(kl) and np.array_equal(net, got[2][1][f]), "frame %d net records" % f
    one.close()
    assert int((aos[30]["m_id"] >= 0).sum()) > 1000 and float(np.abs(aos[30]["rho"] - aos[30]["rho0"]).max()) > 0


EUROC_KC = (-0.28340811, 0.07395907, 0.0, 0.00019359, 1.76187114e-05)   # GlobalConfig_EuRoC_2.txt:64-68, UseUndistort=1


def test_undistort_in_the_flow(built, stream, tmp_path):
    """UseUndistort=1 (every EuRoC configuration of the reference): rb_pipeline_set_undistort against the unmodified reference
    run with the same distortion coefficients.  The undistortion is integer arithmetic on a host-built map, so the keyline
    counts stay identical and the trajectory stays at round-off distance; and it does change the input (other counts than
    without it)."""
    from oracle import refapi
    from rebvo_b200 import capi, synth
    if not os.path.exists(refapi.EXE):
        pytest.skip("oracle/_ref/ref_rebvo not built")
    ts, fr = stream
    n = 40
    path = str(tmp_path / "frames.bin")
    synth.write_frames_file(path, ts[:n], fr[:n])
    kv = dict(UseUndistort=1, KcR2=EUROC_KC[0], KcR4=EUROC_KC[1], KcR6=EUROC_KC[2], KcP1=EUROC_KC[3], KcP2=EUROC_KC[4])
    info, rec = refapi.run_full_rebvo(path, str(tmp_path / "out.bin"), kv)
    os.remove(path)
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=20)
    pl.set_undistort(EUROC_KC)
    nav = np.concatenate([pl.push(fr[s:s + 20], ts[s:s + 20]) for s in range(0, n, 20)])
    pl.set_undistort(None)   # switching it off again drops the captured batches
    pl.close()
    plain, _ = _gpu_run(stream, 20)
    par = refapi.trajectory_parity(rec, nav)
    print(par)
    assert par["kn_equal"] and par["matches_equal"] and par["ate_m"] < 1e-9
    assert not np.array_equal(nav["kn"][:n], plain["kn"][:n])

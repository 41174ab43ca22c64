"""Whole-pipeline parity: rb_pipeline_push (device-resident REBVO flow) against the reference's own 3-thread
REBVO class (oracle/_ref/ref_rebvo, built from the unmodified sources) on the same synthetic 752x480 stream.

Bars (north_star): identical keyline counts per frame (integer work is bit-exact), directed-matching counts equal,
pose ATE <= 1e-3 m (here the streams are deterministic, so the observed ATE is ~1e-9); batch size must not
change the result (frames are processed in order)."""
import os

import numpy as np
import pytest

from pipeline_util import EUROC_KC, assert_runs_identical, euroc_stream, push, run_pipeline, run_reference

pytestmark = pytest.mark.gpu

NF = 60


@pytest.fixture(scope="module")
def stream():
    return euroc_stream(NF)


@pytest.fixture(scope="module")
def ref_run(stream, tmp_path_factory):
    return run_reference(tmp_path_factory.mktemp("ref"), *stream)


def _euroc_run(stream, batch, how="host", mirror=0, collect=("launches",)):
    from rebvo_b200 import capi, synth
    ts, fr = stream
    return run_pipeline(capi.default_params(synth.EUROC), ts, fr, batch, how, mirror=mirror, collect=collect)


def test_trajectory_vs_reference(built, stream, ref_run):
    info, rec = ref_run
    r = _euroc_run(stream, 20)
    nav = r.nav
    n = min(len(rec), NF - 1)
    assert n >= NF - 2
    print("ref fps %.1f, launches/frame %.1f" % (info["fps"], sum(r.launches) / NF))
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
    a = _euroc_run(stream, 20)
    for batch in (7, 1):
        assert_runs_identical(a, _euroc_run(stream, batch), "batch %d" % batch)
    # host-input pushes of >= 3 x REBVO_B200_SUB frames are cut into a head and the rest (copy/compute overlap)
    monkeypatch.setenv("REBVO_B200_SUB", "5")
    assert_runs_identical(a, _euroc_run(stream, 20), "SUB=5")


def test_device_input_equals_host_input(built, stream):
    """rb_pipeline_push_dev reads the caller's device buffer in place; same bits as the host-input path."""
    assert_runs_identical(_euroc_run(stream, 20), _euroc_run(stream, 20, how="device"), "device input")


def test_graph_replay_equals_eager_launches(built, stream, monkeypatch):
    """Batches after the first are replayed as a CUDA graph; the eager path must give the same bits."""
    a = _euroc_run(stream, 10)
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    b = _euroc_run(stream, 10)
    assert a.launches == b.launches, "launch accounting differs between graph replay and eager launches"
    assert_runs_identical(a, b, "eager")


@pytest.mark.parametrize("env", [{"REBVO_B200_MIN_EARLY": "0"}, {"REBVO_B200_PRIO": "0"}])
def test_schedule_variants_do_not_change_the_result(built, stream, monkeypatch, env):
    """Switches that only change when or where work runs (operand staging after the PDL wait, stream priorities): same
    arithmetic in the same order, hence the same bits -- also across a batch boundary and a graph replay."""
    a = _euroc_run(stream, 20)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    assert_runs_identical(a, _euroc_run(stream, 20), str(env))
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    assert_runs_identical(a, _euroc_run(stream, 7), "%s, batch 7, eager" % env)   # other batch size, eager


def test_fallback_paths_agree(built, stream, monkeypatch):
    """The switches in DESIGN.md section 5 select the slower formulations of the same stages (detector on the tracker
    stream, plain stream order): same keylines and matches, poses equal to the rounding of the differently ordered sums."""
    a = _euroc_run(stream, 20).nav
    for k in ("REBVO_B200_OVERLAP", "REBVO_B200_PDL"):
        monkeypatch.setenv(k, "0")
    b = _euroc_run(stream, 20).nav
    assert np.array_equal(a["kn"], b["kn"])                       # the detector does not depend on the tracker
    assert np.abs(a["matches"].astype(int) - b["matches"].astype(int)).max() <= 3   # a threshold decision may flip
    assert np.abs(a["Pos"] - b["Pos"]).max() <= 1e-6
    assert np.abs(a["Kp"] - b["Kp"]).max() <= 1e-6


def test_keyline_mirror_matches_reference_layout(built, stream):
    """The 168-byte AoS mirror handed to host consumers (callback / net packer) is populated and consistent."""
    from rebvo_b200 import capi, synth
    ts, fr = stream
    r = run_pipeline(capi.default_params(synth.EUROC), ts[:4], fr[:4], 4, collect=("maps",))
    nav, (kl, mask) = r.nav, r.maps[0]
    assert len(kl) == nav["kn"][3] and capi.KEYLINE.itemsize == 168
    assert (mask >= 0).sum() == len(kl)
    assert np.array_equal(mask.ravel()[kl["p_inx"]], np.arange(len(kl)))
    assert (kl["m_id"] >= 0).sum() == nav["matches"][3] or (kl["m_id"] >= 0).sum() >= nav["matches"][3]
    assert np.all(kl["rho"] > 0) and np.all(kl["s_rho"] > 0)


def test_host_mirror(built, stream):
    """rb_pipeline_set_mirror: the per-frame records written to host memory during the push equal, for every frame, what the stage calls
    return when the same stream is pushed one frame at a time (so that every frame is once the newest map): mode 1 =
    KeyLine AoS vs rb_map_sync_host_keylines field by field, mode 2 = net_keyline records vs rb_map_pack_net_keylines with
    the frame's K (itself bit-exact against the reference's packer, test_gpu_netpack.py).  The poses do not change."""
    from rebvo_b200 import capi, synth
    ts, fr = stream
    got = {mode: _euroc_run(stream, 20, mirror=mode, collect=("mirrors",)) for mode in (1, 2)}
    for r in got.values():
        assert [len(m) for m in r.mirrors] == list(r.nav["kn"])
    nav, aos = got[1].nav, got[1].mirrors
    assert np.array_equal(got[2].nav["Pos"], nav["Pos"])
    one = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=1)
    for f in range(NF):
        nav1 = push(one, fr[f:f + 1], ts[f:f + 1])
        assert np.array_equal(nav1["Pos"][0], nav["Pos"][f])
        kl = one.map(0).keylines()
        assert len(kl) == len(aos[f])
        for name in capi.KEYLINE.names:
            assert np.array_equal(kl[name], aos[f][name], equal_nan=True), "frame %d field %s" % (f, name)
        net = one.map(0).pack_net(k_prof=float(nav1["K"][0]))
        assert len(net) == len(kl) and np.array_equal(net, got[2].mirrors[f]), "frame %d net records" % f
    one.close()
    assert int((aos[30]["m_id"] >= 0).sum()) > 1000 and float(np.abs(aos[30]["rho"] - aos[30]["rho0"]).max()) > 0


def test_undistort_in_the_flow(built, stream, tmp_path):
    """UseUndistort=1 (every EuRoC configuration of the reference): rb_pipeline_set_undistort against the unmodified reference
    run with the same distortion coefficients.  The undistortion is integer arithmetic on a host-built map, so the keyline
    counts stay identical and the trajectory stays at round-off distance; and it does change the input (other counts than
    without it)."""
    from oracle import refapi
    from rebvo_b200 import capi, synth
    ts, fr = stream
    n = 40
    _, rec = run_reference(tmp_path, ts[:n], fr[:n], kc=EUROC_KC)
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=20)
    pl.set_undistort(EUROC_KC)
    nav = np.concatenate([push(pl, fr[s:s + 20], ts[s:s + 20]) for s in range(0, n, 20)])
    pl.set_undistort(None)   # switching it off again drops the captured batches
    pl.close()
    plain = _euroc_run(stream, 20).nav
    par = refapi.trajectory_parity(rec, nav)
    print(par)
    assert par["kn_equal"] and par["matches_equal"] and par["ate_m"] < 1e-9
    assert not np.array_equal(nav["kn"][:n], plain["kn"][:n])

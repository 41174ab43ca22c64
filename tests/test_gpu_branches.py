"""Branches of the per-frame flow that an ordinary stream never takes, each forced on BOTH sides (rb_pipeline and the
reference's own 3-thread REBVO, oracle/_ref/ref_rebvo) with the same frames and parameters:
  * match-count restart            rebvo_second_t.cpp:412-423   (GlobalMatchThreshold above every frame's match count)
  * NaN guard                      rebvo_second_t.cpp:387-398   (a black frame: empty new map -> JtJ = 0 -> NaN pose;
                                   this is also the rank-deficient input of the init iterations' SVD solve, :659-661)
  * empty old map                  global_tracker.cpp:601       (Minimizer_RV returns at once)
  * TrackerInitType 0 and 1        global_tracker.cpp:628-642
  * the minimiser's abort flag     (test hook REBVO_B200_MIN_FORCE_ABORT: error reported, flag cleared)
and the long-run agreement the speed claim rests on: >= 500 frames at 752x480 (EuRoC parameters) and a 640x480
stream with the TUM desk parameters (TrackerIterNum=10, MatchNumThresh=4, auto-gain 1e-6)."""
import numpy as np
import pytest

from pipeline_util import assert_counts_equal, assert_tight, euroc_sequence, euroc_stream, run_both, run_pipeline, walk

pytestmark = pytest.mark.gpu


def test_long_run_752x480(built, tmp_path):
    from rebvo_b200 import capi, synth
    ts, fr = walk(euroc_sequence(), 520, 130)
    par = assert_tight(*run_both(tmp_path, ts, fr, capi.default_params(synth.EUROC), batch=40), 515)
    assert par["path_length_m"] > 0.05
    assert par["max_pos_err_m"] <= 1e-6, par        # bar in north_star: 1e-3 m
    assert par["max_poselie_err_rad"] <= 1e-6


def test_long_run_640x480_desk_parameters(built, tmp_path):
    """app/rebvorun/GlobalConfig_desk.txt: 17 TryVelRot evaluations per frame, match-count gate 4, auto-gain 1e-6."""
    from rebvo_b200 import capi, synth
    cam = dict(w=640, h=480, zfx=525.0, zfy=525.0, ppx=320.0, ppy=240.0)
    ts, fr = walk(synth.Sequence(w=640, h=480, seed=21, zf=525.0), 300, 100)
    p = capi.default_params(cam, Sigma0=1.7818, kl_max=25000, kl_ref=15000, gain=1e-6, thresh_max=0.05, thresh_min=0.03,
                            SearchRange=20, TrackerIterNum=10, TrackerMatchThresh=1.0, MatchNumThresh=4,
                            ReshapeQRelative=1e-2, kl_capacity=25000)
    # the bar includes the depth-filter state (config 5's criterion): the rescaling estimate Kp integrates every keyline's
    # rho / s_rho
    par = assert_tight(*run_both(tmp_path, ts, fr, p, batch=30), 295)
    assert par["max_pos_err_m"] <= 1e-6, par


def test_restart_branch(built, tmp_path):
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(24)
    rec, nav = run_both(tmp_path, ts, fr, capi.default_params(synth.EUROC, MatchThreshold=10 ** 6), batch=8)
    assert_counts_equal(rec, nav)
    assert not nav["estimation_ok"][1:].any(), "every frame must take the restart branch"
    assert np.array_equal(rec["Kp"][1:], nav["Kp"][1:]) and np.all(nav["Kp"][1:] == 1.0)
    assert np.abs(rec["Pos"] - nav["Pos"]).max() <= 1e-9 and np.abs(rec["PoseLie"] - nav["PoseLie"]).max() <= 1e-9


def test_nan_guard_and_rank_deficient_solve(built, tmp_path):
    """A black frame gives an empty new edge map: no old keyline finds a match, JtJ = 0, the init iterations solve a
    zero matrix (pseudo-inverse -> h = 0), the main loop's Cholesky divides by zero, V / W come out NaN and the caller's
    guard fires.  The frame after it has an empty OLD map (Minimizer_RV returns at once)."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(14)
    fr[6] = 0
    rec, nav = run_both(tmp_path, ts, fr, capi.default_params(synth.EUROC), batch=7)
    assert_counts_equal(rec, nav)
    assert nav["kn"][6] == 0 and nav["estimation_ok"][6] == 0
    assert np.array_equal(np.isnan(rec["Pos"]), np.isnan(nav["Pos"])), "NaN poses must appear in the same frames"
    ok = ~np.isnan(rec["Pos"]).any(1)
    assert ok[:6].all()
    assert np.abs(rec["Pos"][ok] - nav["Pos"][ok]).max() <= 1e-9


def test_empty_first_frames(built, tmp_path):
    """Two black frames at the start: empty old maps (global_tracker.cpp:601), then the restart branch, then tracking."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(16)
    fr[:2] = 0
    rec, nav = run_both(tmp_path, ts, fr, capi.default_params(synth.EUROC), batch=8)
    assert_counts_equal(rec, nav)
    assert np.isfinite(nav["Pos"]).all() and np.isfinite(rec["Pos"]).all()
    assert np.abs(rec["Pos"] - nav["Pos"]).max() <= 1e-8
    assert nav["estimation_ok"][-1] == 1


@pytest.mark.parametrize("init_type", [0, 1])
def test_init_types(built, tmp_path, init_type):
    from oracle import refapi
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(30)
    rec, nav = run_both(tmp_path, ts, fr, capi.default_params(synth.EUROC, TrackerInitType=init_type), batch=10)
    assert_counts_equal(rec, nav)
    par = refapi.trajectory_parity(rec, nav)
    assert par["ate_m"] <= 1e-8, par


def test_minimiser_abort_is_reported_and_cleared(built, monkeypatch):
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = euroc_stream(6)
    monkeypatch.setenv("REBVO_B200_MIN_FORCE_ABORT", "1")
    pl = capi.Pipeline(capi.default_params(cam), max_batch=6)
    with pytest.raises(capi.RbError, match="timed out"):
        pl.push(fr, ts)
    pl.close()
    monkeypatch.delenv("REBVO_B200_MIN_FORCE_ABORT")
    assert np.isfinite(run_pipeline(capi.default_params(cam), ts, fr, 6).nav["Pos"]).all()

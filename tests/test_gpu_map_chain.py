"""The per-frame map chain after the minimiser: k_match (FordwardMatch's apply + directed_matching against the unrotated
old map) and k_reg_ekf (gate + Regularize_1_iter + EKF + rotate_keylines of the old map), against the reference schedule
(REBVO_B200_MAP_CHAIN=0): the stage kernels in the reference's order, k_fm_apply -> k_rotate -> k_directed_match -> gate ->
k_regularize_a / k_regularize_b -> k_ekf, the kernels that test_gpu_parity.py and test_gpu_mapper_states.py pin to the
reference bit for bit.  Both must give the same bits: raw nav records, the keylines and masks of the two newest maps, and
per frame the FordwardMatch winners, directed hits and regularised keylines.

This stream makes few decisions near a threshold.  The same kernels are pinned to the reference bit for bit on seeded
states that reach every branch by test_gpu_map_chain_states.py (k_match and k_reg_ekf, through rb_map_match_update) and
test_gpu_minimiser_forms.py (FordwardMatch's arg-max folded into the minimiser's last round, through
rb_minimizer_rv_forward)."""
import numpy as np
import pytest

from pipeline_util import EUROC_KC, assert_runs_identical, euroc_stream, raw, run_pipeline

pytestmark = pytest.mark.gpu

NF = 72


@pytest.fixture(scope="module")
def stream():
    return euroc_stream(NF)


@pytest.fixture(scope="module")
def special(stream):
    """the stream with a black first frame (frame 1 tracks against an empty old map), a black frame 30 (nothing to
    track: the NaN guard clears do_match) and frame 45 taken from another scene (few matches: the mapping gate closes)"""
    ts, rgb = stream
    rgb = rgb.copy()
    rgb[0] = 0
    rgb[30] = 0
    rgb[45] = euroc_stream(1, seed=99)[1][0]
    return ts, rgb


def _two_schedules(monkeypatch, frames, batch, how="host", kc=None, mirror=0):
    """the run with the two-kernel chain (the default) and with the reference schedule (REBVO_B200_MAP_CHAIN=0)"""
    from rebvo_b200 import capi, synth
    ts, rgb = frames
    p = capi.default_params(synth.EUROC)
    kw = dict(how=how, kc=kc, mirror=mirror, collect=("maps", "counters") + (("mirrors",) if mirror else ()))
    a = run_pipeline(p, ts, rgb, batch, **kw)
    with monkeypatch.context() as m:
        m.setenv("REBVO_B200_MAP_CHAIN", "0")
        return a, run_pipeline(p, ts, rgb, batch, **kw)


@pytest.mark.parametrize("kc", [None, EUROC_KC], ids=["plain", "undistort"])
@pytest.mark.parametrize("how", ["host", "device"])
def test_chain_equals_four_kernel_chain(built, stream, monkeypatch, kc, how):
    for batch in (64, 7, 1):
        ab = _two_schedules(monkeypatch, stream, batch, how, kc)
        assert_runs_identical(*ab, "batch %d" % batch)
    nav, cnt = ab[0].nav, ab[0].counters
    # both matchers and the regularisation did work on this stream
    assert (nav["fwd_matches"] > 0).sum() >= NF // 2 and (nav["matches"] > 0).sum() >= NF // 2
    assert sum(c[2] > 0 for c in cnt) >= NF // 2


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_chain_mirror(built, stream, monkeypatch, mode):
    """the host mirror of every frame's map (mode 1 keeps the rescaling inline on the tracker stream)"""
    assert_runs_identical(*_two_schedules(monkeypatch, stream, 20, kc=EUROC_KC, mirror=mode), "mirror %d" % mode)


@pytest.mark.parametrize("env", ["REBVO_B200_OVERLAP", "REBVO_B200_NO_GRAPH"])
def test_chain_schedules(built, stream, monkeypatch, env):
    """one stream without the side streams (OVERLAP=0), and eager launches (NO_GRAPH=1)"""
    monkeypatch.setenv(env, "1" if env == "REBVO_B200_NO_GRAPH" else "0")
    assert_runs_identical(*_two_schedules(monkeypatch, stream, 20), env)


def test_chain_special_frames(built, special, monkeypatch):
    """black frames, an empty old map and a frame whose match count closes the mapping gate"""
    from rebvo_b200 import capi, synth
    p = capi.default_params(synth.EUROC)
    for batch in (20, 1):
        ab = _two_schedules(monkeypatch, special, batch)
        assert_runs_identical(*ab, "batch %d" % batch)
    nav = ab[0].nav
    assert nav["kn"][0] == 0 and nav["kn"][30] == 0
    assert nav["kn"][1] > 0 and nav["matches"][1] < p.MatchThreshold   # tracked against the empty map of frame 0
    assert nav["estimation_ok"][30] == 0


def test_stage_profile_keys(built, stream, monkeypatch):
    """the eager stage profile runs both schedules and reports every stage key as a number"""
    monkeypatch.setenv("REBVO_B200_STAGE_PROF", "1")
    from rebvo_b200 import capi, synth
    ts, rgb = stream
    res = []
    for chain in ("1", "0"):
        monkeypatch.setenv("REBVO_B200_MAP_CHAIN", chain)
        pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=16)
        nav = pl.push(rgb[:16], ts[:16])
        st, frames = pl.stage_profile()
        pl.close()
        assert frames == 16
        for k in ("minimizer", "quantile+field", "fwdmatch+rotate", "directed_match", "regularize+ekf", "rescale"):
            assert np.isfinite(st[k]) and st[k] >= 0, k
        assert st["quantile+field"] > 0 and st["directed_match"] > 0 and st["regularize+ekf"] > 0
        res.append(nav)
    assert np.array_equal(raw(res[0]), raw(res[1]))

"""The seeded IMU-mode states of tests/imu_states.py are valid, on the CPU against the compiled reference: every case
reaches its target (a vacuous case fails), the TryVel set-up restatement agrees with what the reference wrote, the
Minimizer_V restatement agrees with the reference's Minimizer_V to 1e-12, no LM decision sits within 1e-9 (relative) of
flipping on a step that moves V, and every ExtRotVel system keeps its singular values at least a factor 10 away from
SVD<>'s smax / 1e9 cut."""
import numpy as np
import pytest

import imu_states as S


@pytest.fixture(scope="module")
def base(built):
    from oracle import refapi
    if not refapi.available():
        pytest.skip("compiled reference not available")
    return S.RefBase()


@pytest.mark.parametrize("state", list(S.TV))
def test_try_vel_state(base, state):
    st = base.tv_state(state)
    errs, hits = base.tv_check(st)
    print("%s: %s" % (state, hits))
    assert not errs, "restatement against the reference: %s" % errs
    vac = base.tv_vacuous(st, hits)
    assert not vac, "vacuous case: %s" % vac


def _close(ref, got, tol):
    ref, got = np.asarray(ref, np.float64), np.asarray(got, np.float64)
    same_nan = np.array_equal(np.isnan(ref), np.isnan(got)) and np.array_equal(np.isinf(ref), np.isinf(got))
    fin = np.isfinite(ref)
    return same_nan and bool(np.all(np.abs(ref[fin] - got[fin]) <= tol * np.maximum(np.abs(ref[fin]), 1e-300)))


@pytest.mark.parametrize("state", list(S.MV))
def test_minimizer_v_state(base, state):
    st = base.mv_state(state)
    ref, drv = st["ref"], st["drv"]
    assert _close(ref["V"], drv["V"], 1e-12), (ref["V"], drv["V"])
    assert _close(ref["F"], drv["F"], 1e-12), (ref["F"], drv["F"])
    assert _close(ref["RVel"], drv["RVel"], 1e-12), (ref["RVel"], drv["RVel"])
    assert np.array_equal(st["m_id_f"], st["m_id_f_drv"])
    ill, clear = S.knife(st["tr"])
    vac, info = S.mv_vacuous(st)
    print("%s: %s%s" % (state, info, "" if clear else "  [V within the margin only on steps below %g]" % S.H_TINY))
    assert not ill, "LM decisions on a knife edge: %s" % ill
    assert not vac, "vacuous case: %s" % vac


@pytest.mark.parametrize("state", list(S.ERV))
def test_ext_rot_vel_state(base, state):
    st = base.erv_state(state)
    sp = st["sp"]
    info = base.erv_hits(st)
    print("%s: ok %s %s" % (state, st["ok"], info))
    if sp["kind"] == "z_inf":
        assert not st["ok"]
        return
    if sp.get("n") == 0:
        assert info["matched"] == 0
        return
    assert st["ok"]
    # singular values a factor 10 from the cut on both sides (kept: s * 1e9 > 10 smax; dropped: s * 1e9 < smax / 10)
    assert info["cut_margin"] >= 10, info
    if sp["kind"] == "count":
        assert info["matched"] == sp["n"]
        if sp["n"] > 1:
            assert info["blocks"] >= 2, info
    elif sp["kind"] == "rank":
        assert info["kept"] == sp["rank"], info
    elif sp["kind"] == "cond":
        assert info["kept"] == 6 and 0.5 * sp["cond"] <= info["cond"] <= 2 * sp["cond"], info
    if "huber" in sp["want"]:
        assert info["huber"] >= S.MIN_HITS, info

"""The IMU-mode device stages against the reference on the seeded states of tests/imu_states.py (their validity, hit counts
and LM margins are checked on the CPU by tests/test_cpu_imu_states.py):

- rb_try_vel (k_tv_eval + k_blocks_finish<10>): m_id_f and the whole in-place residual buffer bit for bit, at every evaluation of
  a chain whose residuals feed the next evaluation's reweighting.  Misses inherit the fi of the last match before them
  across warps, blocks and gated keylines, or 0 before the first match.  The per-keyline arithmetic is sequential double
  on both sides; the sums differ only in order: score rel 1e-11, JtJ(a,b) within 1e-11 sqrt(JtJ(a,a) JtJ(b,b)), JtF(a)
  within 1e-11 sqrt(JtJ(a,a) score) (Cauchy-Schwarz bounds on the sums of |terms|).
- rb_minimizer_v: V abs 1e-10 / rel 1e-8 where every LM decision clears the margin, F rel 1e-10, RVel rel 1e-8 where JtJ is
  non-singular (else the same NaN / inf positions), m_id_f of the last evaluation exact.
- rb_ext_rot_vel (k_extrotvel + k_blocks_finish<27>): ok equal, Wx(a,b) within 1e-11 sqrt(Wx(a,a) Wx(b,b)); X and Rx rel 1e-8 where
  cond(Wx) <= 1e6 and rel 1e-14 cond above; on rank-deficient systems the same number of kept singular values and X, Rx
  equal on the kept subspace.
- The IMU pipeline with MatchNumThresh = 3: after vision frames and a reset it runs as a fresh pipeline does, and a fresh
  one follows the reference."""
import numpy as np
import pytest

import imu_states as S
from parity_util import _diff
from pipeline_util import assert_knife_edge, euroc_sequence, raw, run_reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env(built):
    from oracle import refapi
    from rebvo_b200 import capi
    if not refapi.available():
        pytest.skip("oracle/_ref not built")
    b = S.RefBase()
    ctx = capi.Ctx(S.CFG["cam"], S.CFG["sigma0"], S.CFG["ksigma"], kl_capacity=S.KEYLINE_MAX)
    yield b, ctx
    ctx.close()


def _maps(b, ctx, kl, fc):
    new, old = ctx.new_map(), ctx.new_map()
    new.load_keylines(b.kl11, b.mask11)
    new.build_field(S.CFG["radius"], b.rt)
    new.set_frame_count(fc)
    old.load_keylines(kl, b.empty)
    return new, old


def _sum_errs(tag, s_r, J_r, F_r, s_g, J_g, F_g):
    errs = []
    if not abs(s_g - s_r) <= 1e-11 * abs(s_r):
        errs.append("%s score: ref %.17g gpu %.17g" % (tag, s_r, s_g))
    d = np.diag(J_r)
    bad = ~(np.abs(J_g - J_r) <= 1e-11 * np.sqrt(np.outer(d, d)))
    if bad.any():
        errs.append("%s JtJ: ref %s gpu %s" % (tag, J_r[bad][:3], J_g[bad][:3]))
    bad = ~(np.abs(F_g - F_r) <= 1e-11 * np.sqrt(d * s_r))
    if bad.any():
        errs.append("%s JtF: ref %s gpu %s" % (tag, F_r[bad], F_g[bad]))
    return errs


@pytest.mark.parametrize("state", list(S.TV))
def test_try_vel_state(env, state):
    b, ctx = env
    st = b.tv_state(state)
    sp = st["sp"]
    new, old = _maps(b, ctx, st["kl"], sp["fc"])
    msgs = []
    try:
        for k, e in enumerate(st["evals"]):
            s_g, J_g, F_g, res_g = new.try_vel(old, e["V"], sp["mt"], sp["q"], sp["mnt"], e["res_in"], sp["rw"],
                                               sp["min_mod"])
            tag = "eval %d" % k
            msgs += _sum_errs(tag, e["s"], e["JtJ"], e["JtF"], s_g, J_g, F_g)
            for d in (_diff(tag + " residuals", e["res"], res_g), _diff(tag + " m_id_f", e["m_id_f"], old.keylines()["m_id_f"])):
                if d:
                    msgs.append(d)
    finally:
        new.close()
        old.close()
    assert not msgs, "\n".join(msgs[:20])


def _singular(J):
    J = np.asarray(J, np.float64)
    if not np.isfinite(J).all() or not np.abs(J).max() > 0:
        return True
    ev = np.linalg.eigvalsh((J + J.T) / 2)
    return ev[0] <= 1e-12 * ev[-1]


def _same_nonfinite(a, b):
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b)) and \
        np.array_equal(np.isneginf(a), np.isneginf(b))


@pytest.mark.parametrize("state", list(S.MV))
def test_minimizer_v_state(env, state):
    b, ctx = env
    st = b.mv_state(state)
    sp, a, ref = st["sp"], st["a"], st["ref"]
    new, old = _maps(b, ctx, st["kl"], a["fc"])
    try:
        m_g = new.minimizer_v(old, st["V0"], a["mt"], sp["iter_max"], a["q"], a["mnt"], a["rw"], a["min_mod"])
        mf = old.keylines()["m_id_f"]
    finally:
        new.close()
        old.close()
    msgs = []
    _, clear = S.knife(st["tr"])
    if clear:
        dv = np.abs(m_g["V"] - ref["V"])
        if not (dv <= np.maximum(1e-10, 1e-8 * np.abs(ref["V"]))).all():
            msgs.append("V: ref %s gpu %s" % (ref["V"], m_g["V"]))
    else:
        print("%s: a decision within the margin on a step below %g: V not compared" % (state, S.H_TINY))
    if not abs(m_g["F"] - ref["F"]) <= 1e-10 * abs(ref["F"]):
        msgs.append("F: ref %.17g gpu %.17g" % (ref["F"], m_g["F"]))
    if not _same_nonfinite(ref["RVel"], m_g["RVel"]):
        msgs.append("RVel NaN / inf positions: ref %s gpu %s" % (ref["RVel"].ravel(), m_g["RVel"].ravel()))
    elif not _singular(st["drv"]["JtJ"]):
        if not (np.abs(m_g["RVel"] - ref["RVel"]) <= 1e-8 * np.abs(ref["RVel"]).max()).all():
            msgs.append("RVel: ref %s gpu %s" % (ref["RVel"].ravel(), m_g["RVel"].ravel()))
    d = _diff("m_id_f", st["m_id_f"], mf)
    if d:
        msgs.append(d)
    if "empty" in sp["want"] and not np.array_equal(m_g["V"], st["V0"]):
        msgs.append("empty old map: Vel changed to %s" % m_g["V"])
    print("%s: ref V %s F %.6g, gpu V %s F %.6g" % (state, ref["V"], ref["F"], m_g["V"], m_g["F"]))
    assert not msgs, "\n".join(msgs)


def _match(tag, ref, got, tol):
    ref, got = np.asarray(ref, np.float64), np.asarray(got, np.float64)
    bad = ~(np.abs(got - ref) <= tol * np.abs(ref) + 0.1 * tol * np.abs(ref).max())
    return ["%s: ref %s gpu %s (tol %.1e)" % (tag, ref[bad][:3], got[bad][:3], tol)] if bad.any() else []


@pytest.mark.parametrize("state", list(S.ERV))
def test_ext_rot_vel_state(env, state):
    b, ctx = env
    st = b.erv_state(state)
    m = ctx.new_map()
    try:
        m.load_keylines(st["kl"], b.empty)
        ok, Wx, Rx, X = m.ext_rot_vel(st["V"], S.LOC_UNC, S.RW)
    finally:
        m.close()
    assert ok == st["ok"], (ok, st["ok"])
    if not ok:
        return
    Wr, Rr, Xr = st["Wx"], st["Rx"], st["X"]
    msgs = []
    d = np.sqrt(np.outer(np.diag(Wr), np.diag(Wr)))
    bad = ~(np.abs(Wx - Wr) <= 1e-11 * d)
    if bad.any():
        msgs.append("Wx: ref %s gpu %s" % (Wr[bad][:3], Wx[bad][:3]))
    if not np.abs(Wr).max() > 0:   # no matches: every singular value is cut
        assert not msgs and not X.any() and not Rx.any(), (msgs, X, Rx)
        return
    U, s, _ = np.linalg.svd(Wr)
    kept = s * S.CUT > s[0]
    cond = s[0] / s[kept][-1]
    tol = 1e-8 if cond <= 1e6 else 1e-14 * cond
    sr = np.linalg.svd(Rx, compute_uv=False)
    n_gpu = int((sr > 1e-12 * sr[0]).sum())
    if n_gpu != kept.sum():
        msgs.append("kept singular values: ref %d gpu %d (Rx spectrum %s)" % (kept.sum(), n_gpu, sr))
    P = U[:, kept] @ U[:, kept].T
    msgs += _match("X", Xr, P @ X, tol) + _match("Rx", Rr, P @ Rx @ P, tol)
    print("%s: kept %d cond %.3g tol %.1e" % (state, kept.sum(), cond, tol))
    assert not msgs, "\n".join(msgs)


# ---- the IMU pipeline with MatchNumThresh > 0 ---------------------------------------------------------------------------
NV, NF, BATCH = 24, 40, 8   # vision frames (frame 23 sets FrameCount (23-1)/8 = 2), IMU frames, frames per push


def _imu_run(p, ts, fr, imu, vision_first):
    from rebvo_b200 import capi
    pl = capi.Pipeline(p, max_batch=BATCH)
    navs, odo = [], []
    try:
        pl.set_odometry(True)
        if vision_first:
            for s in range(0, NV, BATCH):
                pl.push(fr[s:s + BATCH], ts[s:s + BATCH])
        pl.set_imu(imu, capi.default_imu_params(InitBias=1, InitBiasFrameNum=5))
        if vision_first:
            pl.reset()
        for s in range(0, NF, BATCH):
            navs.append(pl.push(fr[s:s + BATCH], ts[s:s + BATCH]))
            odo.append(pl.odometry())
    finally:
        pl.close()
    return np.concatenate(navs), np.concatenate(odo)


def test_imu_after_vision_and_reset(built):
    """Vision frames leave each ring map's FrameCount at (frame-1)/8; the reference's IMU flow never raises FrameCount
    (only Minimizer_RV does), so its m_num gate min(MatchNumThresh, FrameCount) stays off.  After set_imu and reset, the
    IMU pushes must gate nothing a fresh pipeline keeps: nav and odometry records equal byte for byte."""
    from rebvo_b200 import capi, synth
    seq = euroc_sequence()
    ts, fr = seq.frames(max(NV, NF))
    imu = synth.imu_samples(seq, max(NV, NF))
    p = capi.default_params(synth.EUROC, MatchNumThresh=3)
    nav_f, odo_f = _imu_run(p, ts, fr, imu, False)
    nav_r, odo_r = _imu_run(p, ts, fr, imu, True)
    diff = np.nonzero((raw(nav_f) != raw(nav_r)).reshape(len(nav_f), -1).any(1))[0]
    assert len(diff) == 0, "nav records differ from frame %d (matches fresh %s, after reset %s)" % (
        diff[0], nav_f["matches"][diff[:5]], nav_r["matches"][diff[:5]])
    assert np.array_equal(raw(odo_f), raw(odo_r)), "odometry records"


def test_imu_pipeline_match_num_thresh_vs_reference(built, tmp_path):
    """A fresh IMU pipeline with MatchNumThresh = 3 against the reference's CPU build with the same parameters"""
    from rebvo_b200 import capi, synth
    seq = euroc_sequence()
    ts, fr = seq.frames(NF)
    imu = synth.imu_samples(seq, NF)
    p = capi.default_params(synth.EUROC, MatchNumThresh=3)
    _, ref = run_reference(tmp_path, ts, fr, p, imu=imu)
    nav, _ = _imu_run(p, ts, fr, imu, False)
    n = min(len(ref), len(nav))
    assert np.isfinite(nav["Pos"][:n]).all()
    assert_knife_edge(ref, nav, NF - 2, "IMU pipeline, MatchNumThresh 3")
    assert np.allclose(ref["K"][1:n], nav["K"][1:n], rtol=1e-6, atol=1e-12)

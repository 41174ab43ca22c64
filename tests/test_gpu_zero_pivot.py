"""The LDL^T sites that meet a zero pivot on degenerate edge maps, against the reference, on the device and end to end.

TooN's Cholesky<6>(JtJ).get_inverse() stops at the first zero pivot and keeps finite entries after it; a factor that
goes on past it (1/0 = inf) makes them NaN (tests/test_cpu_zero_pivot.py).  These tests run the states that reach such a
pivot and compare by class: the same NaN, +inf and -inf positions, and finite values within the usual bars.

test_minimiser_cov runs Minimizer_RV (the covariance RVel / RW0 of lm_finalize_cov, and W_X) on seeded old maps in three
kernel forms: every keyline gated by s_rho (JtJ = 0), and old and new maps of exactly vertical or horizontal edges, whose
field gradients leave the Vy or the Vx column of the Jacobian exactly zero.  Each state proves it reached its zero pivot
on the reference's own W_X.

test_imu_stream runs IMU mode (ImuMode=2) through the pipeline, the reference (ref_rebvo) and the reference on the
library's stages (shim_rebvo) on EuRoC-like streams with a stretch of vertical-stripe frames, before and after the
scale filter starts, and compares the odometry records with the reference's pose graph.  test_vision_stripes runs the
stretch in vision mode.  These streams reach no zero pivot (the tests print the pivots they measure): they check the
stretch by class, while the zero pivots themselves are reached on the seeded states of test_minimiser_cov and of
tests/test_cpu_zero_pivot.py.  No stream has a black frame: the reference's IMU branch aborts on one (DESIGN.md section 3).

test_contexts_of_different_slices runs the minimiser of a context after a second context with a smaller shared-memory
slice was created."""
import os

import numpy as np
import pytest

from pipeline_util import assert_knife_edge, euroc_sequence, run_pipeline, run_reference, shim_exe, trim
from test_cpu_zero_pivot import class_errors, zero_pivot
from test_gpu_minimiser_forms import BARS, CFG, CLUSTERS, Base, _ctx, _set_form_env, _tile

pytestmark = pytest.mark.gpu

FORMS = ("four_clusters", "one_cluster", "spill_g4")


# ---- Minimizer_RV on maps that leave a Jacobian column zero ------------------------------------------------------------
def _axis(kl, axis):
    """every gradient turned onto one image axis (its sign and modulus kept): axis 0 = vertical edges (gradient along x)"""
    kl = kl.copy()
    s = np.where(kl["m_m"][:, axis] < 0, -1.0, 1.0).astype(np.float32)
    kl["m_m"][:] = 0
    kl["u_m"][:] = 0
    kl["m_m"][:, axis] = s * kl["n_m"]
    kl["u_m"][:, axis] = s
    return kl


# state -> (gradient axis of both maps or None, s_rho of every old keyline or None, pivot TooN stops at)
STATES = {"all_gated": (None, 10.0, 0), "vertical": (0, None, 1), "horizontal": (1, None, 0)}
Q = 1e3


@pytest.fixture(scope="module")
def base(built):
    b = Base()
    yield b
    for c in b.ctx.values():
        c.close()
    b.b.close()


def _maps(base, state):
    axis, s_rho, _ = STATES[state]
    old = _tile(base.kl10, 4000, np.random.default_rng(11))
    new = base.kl11
    if axis is not None:
        old, new = _axis(old, axis), _axis(new, axis)
    if s_rho is not None:
        old["s_rho"] = s_rho * Q
    return old, new


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("state", list(STATES))
def test_minimiser_cov(base, monkeypatch, state, form):
    _set_form_env(monkeypatch, form)
    old_kl, new_kl = _maps(base, state)
    args = (CFG["match_thresh"], 5, 2, 2.0, Q, 0, 2)
    r_new = base.refmap()
    r_new.set_keylines(new_kl)
    r_new.set_mask(base.mask11, len(new_kl))
    r_new.build_field(CFG["radius"], base.rt)
    r_old = base.refmap()
    r_old.set_keylines(old_kl)
    r_old.set_mask(base.empty, len(old_kl))
    m_r = r_new.minimizer_rv(r_old, np.zeros(3), np.zeros(3), *args)
    # the state reaches its target: TooN's factor of the reference's JtJ stops at the pivot the state aims at
    piv = zero_pivot(np.asarray(m_r["W_X"], np.float64).reshape(6, 6))
    print("%s / %s: TooN stops at pivot %s; finite RVel %d, RW0 %d" % (state, form, piv, np.isfinite(m_r["RVel"]).sum(),
                                                                      np.isfinite(m_r["RW0"]).sum()))
    assert piv == STATES[state][2], "vacuous state: the factor stops at pivot %s" % piv
    if state != "all_gated":
        assert np.isfinite(m_r["RW0"]).any(), "the reference's covariance has no finite entry: nothing to tell apart"

    ctx = _ctx(base, form)
    assert ctx.minimizer_clusters() == CLUSTERS[form]
    new, old = ctx.new_map(), ctx.new_map()
    try:
        new.load_keylines(new_kl, base.mask11)
        new.build_field(CFG["radius"], base.rt)
        old.load_keylines(old_kl, base.empty)
        m_g = new.minimizer_rv(old, np.zeros(3), np.zeros(3), *args)
    finally:
        new.close()
        old.close()
    errs = []
    for k, rtol, atol, scaled in BARS:
        if k in ("F", "rel_err_score"):
            continue
        ref = np.asarray(m_r[k], np.float64)
        amax = np.abs(ref[np.isfinite(ref)]).max() if np.isfinite(ref).any() else 0.0
        errs += class_errors(k, ref, m_g[k], rtol, atol * amax if scaled else atol)
    assert not errs, "\n".join(errs)


# ---- whole streams ------------------------------------------------------------------------------------------------------
NF = 30
FIRST_FILTERED = 4 + 5 + 1   # est_ka_gmek_bias runs from frame 4 + InitBiasFrameNum + 1


def _stripes(h, w, shift):
    """vertical step edges only: 24-px bands of two grey levels, moved `shift` px to the right"""
    x = (np.arange(w) + shift) // 24
    row = np.where(x % 2 == 0, 60, 190).astype(np.uint8)
    img = np.broadcast_to(row[None, :, None], (h, w, 3))
    return np.ascontiguousarray(img)


# (a black frame is not among them: the reference's IMU branch aborts on one, in SO3::coerce's assertion)
STREAMS = {"stripes": dict(stripes=range(FIRST_FILTERED + 3, FIRST_FILTERED + 9)),
           "stripes_before_filter": dict(stripes=range(4, 8))}


def _stream(name):
    from rebvo_b200 import synth
    seq = euroc_sequence()
    ts, fr = seq.frames(NF)
    fr = fr.copy()
    sp = STREAMS[name]
    for k, i in enumerate(sp["stripes"]):
        fr[i] = _stripes(fr.shape[1], fr.shape[2], 2 * k)
    return ts, fr, synth.imu_samples(seq, NF)


def _classes(a, b, fields, what):
    """per record: the same NaN, +inf and -inf positions in every field"""
    errs = []
    for f in fields:
        for cls, fn in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
            d = (fn(a[f]) != fn(b[f])).reshape(len(a), -1).any(1)
            if d.any():
                errs.append("%s %s: %s positions differ at records %s" % (what, f, cls, np.nonzero(d)[0][:6]))
    return errs


def _compare_nav(ref, got, what, imu):
    """by class, then the bars of test_gpu_imu_mode.py on the finite values: assert_knife_edge (kn, est_ok, matches
    within 0.5 %, ATE and largest position error <= 1e-3 m) and K within 1e-6"""
    ref, got = trim(ref, got)
    fields = ("Pos", "Pose", "Vel", "RotLie") + (("K",) if imu else ())
    errs = _classes(ref, got, fields, what)
    assert not errs, "\n".join(errs)
    assert_knife_edge(ref, got, NF - 2, what)
    if imu:
        assert np.allclose(ref["K"][1:], got["K"][1:], rtol=1e-6, atol=1e-12, equal_nan=True), what


def _compare_odometry(ref, odo, what):
    """the pipeline's odometry records (record r: frame r) against the reference's pose graph (record r: frame r + 1), by
    class and with test_gpu_odometry.py's bars on the finite values"""
    got = odo[1:]
    # (the reference's last record depends on its shutdown: test_gpu_odometry.py)
    n = min(len(ref) - 1, len(got))
    assert n >= NF - 3
    ref, got = ref[:n], got[:n]
    fields = ("relPosPose", "WrelPosPose", "Rs", "Rv", "Rg", "K")
    errs = _classes(ref, got, fields, what)
    for r in range(n):
        w = ref["WrelPosPose"][r]
        amax = np.abs(w[np.isfinite(w)]).max() if np.isfinite(w).any() else 0.0
        errs += class_errors("%s record %d WrelPosPose" % (what, r), w, got["WrelPosPose"][r], 0.0, 1e-5 * amax)
        errs += class_errors("%s record %d relPosPose" % (what, r), ref["relPosPose"][r], got["relPosPose"][r], 0.0, 1e-6)
        for k in ("Rs", "Rv", "Rg"):   # covariances: each entry also against its own scale sqrt(|C_ii C_jj|)
            c = np.asarray(ref[k][r], np.float64)
            with np.errstate(invalid="ignore"):
                sc = np.nan_to_num(np.sqrt(np.abs(np.outer(np.diag(c), np.diag(c)))), nan=0.0, posinf=0.0)
            errs += class_errors("%s record %d %s" % (what, r, k), c, got[k][r], 1e-6, 1e-6 * sc)
        errs += class_errors("%s record %d K" % (what, r), ref["K"][r], got["K"][r], 1e-6, 0.0)
    assert not errs, "\n".join(errs[:12])


def _pivots(ref_pg, frames):
    """{frame: the pivot TooN's factor of the reference's information matrix stops at} for the frames of a stretch"""
    return {i: zero_pivot(ref_pg["WrelPosPose"][i - 1]) for i in frames if i - 1 < len(ref_pg)}


def _pose_graph(tmp_path, p, ts, fr, **kw):
    from oracle import build_pose_graph
    from rebvo_b200 import capi
    ps = str(tmp_path / "poses_list.ps")
    run_reference(tmp_path, ts, fr, p, exe=build_pose_graph.EXE, timeout=1500, PoseGraphFile=ps, **kw)
    return capi.read_pose_graph(ps)


@pytest.mark.parametrize("stream", list(STREAMS))
def test_imu_stream(built, tmp_path, stream):
    """A stretch of vertical-stripe frames, the nearest a rendered stream comes to the degenerate maps of
    test_minimiser_cov and test_bias_correct: nav records of the reference, its shim and the pipeline, and the odometry
    records (Rv = P_V / dt^4 is R_Xgv's velocity block) of the reference and the pipeline, by class.  Measured: no frame
    of these streams leaves the reference's W_Xgv a zero pivot (ExtRotVel's information keeps every row), so these are
    parity cases of the stretch, not of the zero-pivot sites; the zero pivots are reached on seeded states instead."""
    from oracle import refapi
    from rebvo_b200 import capi, synth
    if not (os.path.exists(shim_exe()) and os.path.exists(refapi.EXE)):
        pytest.skip("oracle/_ref/shim_rebvo / ref_rebvo not built")
    ts, fr, imu = _stream(stream)
    p = capi.default_params(synth.EUROC)
    _, ref = run_reference(tmp_path, ts, fr, p, imu=imu)
    _, shim = run_reference(tmp_path, ts, fr, p, exe=shim_exe(), imu=imu)
    pg = _pose_graph(tmp_path, p, ts, fr, imu=imu)
    r = run_pipeline(p, ts, fr, 10, imu=imu, odometry=True, collect=("odometry",))
    hit = list(STREAMS[stream]["stripes"])
    piv = _pivots(pg, hit)
    print("%s: matches %s, zero pivots %s, finite Rv entries %s" % (stream, ref["matches"][hit], piv,
                                                                   [int(np.isfinite(pg["Rv"][i - 1]).sum()) for i in hit]))
    _compare_nav(ref, shim, "shim", True)
    _compare_nav(ref, r.nav, "pipeline", True)
    _compare_odometry(pg, r.odometry, "odometry")


def test_vision_stripes(built, tmp_path):
    """Vision mode on the same stretch, against the reference's nav records and pose graph by class.  Measured: the pose
    graph's information matrices of the stretch have no zero pivot either (they are W_X moved into the frame's axes)."""
    from rebvo_b200 import capi, synth
    ts, fr, _ = _stream("stripes")
    p = capi.default_params(synth.EUROC)
    _, ref = run_reference(tmp_path, ts, fr, p)
    pg = _pose_graph(tmp_path, p, ts, fr)
    r = run_pipeline(p, ts, fr, 10, odometry=True, collect=("odometry",))
    hit = list(STREAMS["stripes"]["stripes"])
    piv = _pivots(pg, hit)
    print("vision: matches %s, zero pivots %s" % (ref["matches"][hit], piv))
    _compare_nav(ref, r.nav, "vision", False)
    _compare_odometry(pg, r.odometry, "vision odometry")


def test_contexts_of_different_slices(built, monkeypatch):
    """The minimiser's shared-memory limit belongs to its kernel, not to a context: a context created after another with a
    smaller shared-memory slice (REBVO_B200_MIN_KPC=32) must leave the first one able to launch."""
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    seq = euroc_sequence()
    _, fr = seq.frames(2)
    out = []
    _set_form_env(monkeypatch, "four_clusters")
    big = capi.Ctx(cam, CFG["sigma0"], CFG["ksigma"], kl_capacity=50000)
    monkeypatch.setenv("REBVO_B200_MIN_KPC", "32")
    small = capi.Ctx(cam, CFG["sigma0"], CFG["ksigma"], kl_capacity=2000)
    maps = []
    try:
        det = capi.DetectParams(2, 0.4, 0.095259868922420, 2000, 1500, 0.0, 1.0, 0.0)
        for ctx in (big, small):
            ms = [ctx.new_map(), ctx.new_map()]
            maps.append(ms)
            for m, f in zip(ms, fr):
                m.upload_rgb(f)
                m.dog_build()
                m.detect(det, 0.01, 0)
            ms[1].build_field(CFG["radius"], 0.01)
        for ms in maps:   # the first context launches after the second was created
            out.append(ms[1].minimizer_rv(ms[0], np.zeros(3), np.zeros(3), CFG["match_thresh"], 5, 2, 2.0, Q, 0, 2))
    finally:
        for ms in maps:
            for m in ms:
                m.close()
        small.close()
        big.close()
    # both contexts minimise the same maps: the same pose
    assert np.isfinite(out[0]["V"]).all() and np.allclose(out[0]["V"], out[1]["V"], rtol=0, atol=1e-8), out

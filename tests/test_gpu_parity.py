"""GPU parity tests: the CUDA path (through the C ABI) against the UNMODIFIED reference compiled into
oracle/_ref (SURVEY.md section 8(c)), stage by stage, on seeded synthetic frames at the benchmark resolutions.

Bars: float32 scale space, keyline records, id mask and match field bit-exact; float64 per-keyline results
rel 1e-12; reductions over keylines (JtJ, JtF, score) rel 1e-10 (different, fixed summation order);
minimiser outputs abs 1e-9."""
import numpy as np
import pytest

from parity_util import (BIG_CFG, DOG_THRESH, EUROC_CFG, KL_EXACT_DETECT, PLANE_FIT, POS_NEG, TUM_CFG, Report,
                         compare_keylines)

pytestmark = pytest.mark.gpu


def _frames(cfg):
    from rebvo_b200 import synth
    cam = cfg["cam"]
    if cfg["name"] == "tum":
        return synth.frame_pair(seed=42, w=cam["w"], h=cam["h"], nrect=220, shift=(1.5, 0.7))
    if cfg["name"] == "big":
        seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=100, zf=cam["zfx"], nrect_bg=1500, nrect_fg=200)
        return seq.frame(10)[1], seq.frame(11)[1]
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=7, zf=cam["zfx"])
    return seq.frame(10)[1], seq.frame(11)[1]


def _seed_depth(kl):
    kl = kl.copy()
    kl["rho"] = 1.0
    kl["s_rho"] = 0.2
    kl["m_num"] = 5
    return kl


def _run_stage_parity(cfg):
    from oracle import refapi
    from rebvo_b200 import capi
    cam = cfg["cam"]
    rep = Report(cfg["name"])
    f0, f1 = _frames(cfg)
    refs = [refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], cfg["sigma0"],
                          cfg["ksigma"]) for _ in range(2)]
    ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)
    gm = [ctx.new_map(), ctx.new_map()]
    det = capi.DetectParams(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["kl_ref"], cfg["gain"], cfg["tmax"],
                            cfg["tmin"])
    # ---------------- scale space + detector, two frames with the threshold feedback chained -------------
    t_ref, l_ref = cfg["thresh"], 0
    t_gpu, l_gpu = cfg["thresh"], 0
    for i, fr in enumerate((f0, f1)):
        r, g = refs[i], gm[i]
        r.rgb2bw(fr)
        r.build()
        g.upload_rgb(fr)
        g.dog_build()
        rep.exact("f%d gray" % i, r.plane("gray"), g.plane("gray"))
        rep.exact("f%d Img(0)" % i, r.plane("img0"), g.plane("img0"))
        rep.exact("f%d Img(1)" % i, r.plane("img1"), g.plane("img1"))
        rep.exact("f%d DoG" % i, r.plane("dog"), g.plane("dog"))
        rep.exact("f%d Dx interior" % i, r.plane("dx")[1:-1, 1:-1], g.plane("dx")[1:-1, 1:-1])
        rep.exact("f%d Dy interior" % i, r.plane("dy")[1:-1, 1:-1], g.plane("dy")[1:-1, 1:-1])
        kn_r, t_ref, l_ref = r.detect(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], t_ref, l_ref, cfg["kl_ref"],
                                      cfg["gain"], cfg["tmax"], cfg["tmin"])
        kn_g, t_gpu, l_gpu = g.detect(det, t_gpu, l_gpu)
        rep.add("f%d detect kn/tresh" % i, kn_r == kn_g and t_ref == t_gpu and l_ref == l_gpu,
                "ref kn=%d t=%.9g | gpu kn=%d t=%.9g" % (kn_r, t_ref, kn_g, t_gpu))
        compare_keylines(rep, "f%d detect" % i, r.keylines(), g.keylines(), KL_EXACT_DETECT)
        rep.exact("f%d mask" % i, r.mask(), g.mask())
        _, rt = r.reestimate(cfg["track_points"], 100)
        gt = g.reestimate(cfg["track_points"], 100)
        rep.add("f%d reEstimateThresh" % i, np.float32(rt) == np.float32(gt), "ref %.9g gpu %.9g" % (rt, gt))
    # ---------------- truncation at kl_max -----------------------------------------------------------------
    small = 5000
    kn_r, _, _ = refs[1].detect(PLANE_FIT, POS_NEG, DOG_THRESH, small, t_ref, l_ref, cfg["kl_ref"], 0.0, 1, 0)
    det_small = capi.DetectParams(PLANE_FIT, POS_NEG, DOG_THRESH, small, cfg["kl_ref"], 0.0, 1.0, 0.0)
    kn_g, _, _ = gm[1].detect(det_small, t_ref, l_ref)
    compare_keylines(rep, "kl_max cut", refs[1].keylines(), gm[1].keylines(), KL_EXACT_DETECT)
    rep.exact("kl_max cut mask", refs[1].mask(), gm[1].mask())
    # restore frame 1
    refs[1].detect(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], t_ref, l_ref, cfg["kl_ref"], 0.0, 1, 0)
    gm[1].detect(capi.DetectParams(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["kl_ref"], 0.0, 1.0, 0.0),
                 t_ref, l_ref)
    _, rt = refs[1].reestimate(cfg["track_points"], 100)
    gm[1].reestimate(cfg["track_points"], 100)

    m_r = _tracker_parity(rep, cfg, refs, gm, rt)
    old_r, new_r, old_g, new_g = refs[0], refs[1], gm[0], gm[1]
    # FordwardMatch
    old_r.forward_match(new_r)
    old_g.forward_match(new_g)
    fm_fields = ["rho", "s_rho", "m_num", "m_id", "p_m_0"]
    compare_keylines(rep, "FordwardMatch new", new_r.keylines(), new_g.keylines(), fm_fields)
    mk = new_r.keylines()["m_id"] >= 0
    rep.exact("FordwardMatch m_m0 (matched)", new_r.keylines()["m_m0"][mk], new_g.keylines()["m_m0"][mk])
    rep.exact("FordwardMatch n_m0 (matched)", new_r.keylines()["n_m0"][mk], new_g.keylines()["n_m0"][mk])
    # rotate_keylines with the reference's rotation
    R0 = refapi.so3_exp(m_r["W"])
    old_r.rotate(R0)
    old_g.rotate(R0)
    compare_keylines(rep, "rotate_keylines old", old_r.keylines(), old_g.keylines(), ["p_m", "m_m", "rho", "s_rho"])
    # directed_matching from identical state
    old_g.load_keylines(old_r.keylines(), old_r.mask())
    new_g.load_keylines(new_r.keylines(), new_r.mask())
    R = R0.T.copy()
    n_r = new_r.directed_matching(old_r, m_r["V"], m_r["RVel"], R, cfg["thr_mod"], cfg["thr_ang"], cfg["radius"],
                                  cfg["loc_unc_match"])
    n_g = new_g.directed_matching(old_g, m_r["V"], m_r["RVel"], R, cfg["thr_mod"], cfg["thr_ang"], cfg["radius"],
                                  cfg["loc_unc_match"])
    rep.add("directed_matching count", n_r == n_g, "ref %d gpu %d" % (n_r, n_g))
    compare_keylines(rep, "directed_matching new", new_r.keylines(), new_g.keylines(),
                     ["rho", "s_rho", "m_num", "m_id", "p_m_0"])
    mk = new_r.keylines()["m_id"] >= 0
    rep.exact("directed_matching m_m0 (matched)", new_r.keylines()["m_m0"][mk], new_g.keylines()["m_m0"][mk])
    # Regularize_1_iter
    new_g.load_keylines(new_r.keylines(), new_r.mask())
    r_r = new_r.regularize(cfg["reg_thresh"])
    r_g = new_g.regularize(cfg["reg_thresh"])
    rep.add("Regularize_1_iter count", r_r == r_g, "ref %d gpu %d" % (r_r, r_g))
    compare_keylines(rep, "Regularize_1_iter", new_r.keylines(), new_g.keylines(), ["rho", "s_rho"])
    # EKF
    new_r.ekf(m_r["V"], m_r["RVel"], m_r["RW0"], cfg["q_abs"], 1.6968e-4, cfg["loc_unc"])
    new_g.ekf(m_r["V"], cfg["q_abs"], cfg["loc_unc"])
    compare_keylines(rep, "EKF", new_r.keylines(), new_g.keylines(), [], ["rho", "s_rho", "rho0", "s_rho0"], rtol=1e-13)
    compare_keylines(rep, "EKF (bitwise)", new_r.keylines(), new_g.keylines(), ["rho", "s_rho", "rho0", "s_rho0"])
    # EstimateReScalingOpt
    kp_r, rkp_r = new_r.rescale(20.0, 1, False)
    kp_g, rkp_g = new_g.rescale(20.0, 1, False)
    rep.close("EstimateReScalingOpt Kp", kp_r, kp_g, 1e-12)
    rep.close("EstimateReScalingOpt RKp", rkp_r, rkp_g, 1e-11)
    rep.dump()
    for g in gm:
        g.close()
    ctx.close()
    return rep


def _tracker_parity(rep, cfg, refs, gm, rt):
    """TryVelRot at three poses x three (reweight, procjf) pairs, then Minimizer_RV; returns the reference's result."""
    # old = frame 0 with seeded depth, new = frame 1
    old_r, new_r, old_g, new_g = refs[0], refs[1], gm[0], gm[1]
    old_r.set_keylines(_seed_depth(old_r.keylines()))
    old_g.load_keylines(old_r.keylines(), old_r.mask())
    new_g.load_keylines(new_r.keylines(), new_r.mask())
    q_r = old_r.quantile(1e-3, 20.0, 0.9, 100)
    q_g = old_g.quantile(1e-3, 20.0, 0.9, 100)
    rep.add("EstimateQuantile", q_r == q_g, "ref %.17g gpu %.17g" % (q_r, q_g))
    new_r.build_field(cfg["radius"], rt)
    new_g.build_field(cfg["radius"], rt)
    fr_, fg_ = new_r.field(), new_g.field()
    rep.exact("field ikl", fr_[:, :, 1], fg_[:, :, 1])
    has = fr_[:, :, 1] >= 0
    rep.exact("field dist (where set)", fr_[:, :, 0][has], fg_[:, :, 0][has])
    # single evaluations of TryVelRot
    k0 = old_r.knum()
    pnum = (k0 + 3) & ~3
    rng = np.random.default_rng(3)
    res_prev = np.zeros(pnum)
    Xs = [np.zeros(6), np.array([0.002, -0.001, 0.0005, 0.001, -0.002, 0.003]),
          np.array([-0.004, 0.003, -0.001, -0.003, 0.001, -0.004])]
    for xi, X in enumerate(Xs):
        for (rw, pj) in ((False, True), (True, True), (False, False)):
            s_r, J_r, F_r, res_r = new_r.try_vel_rot(old_r, X, rw, pj, cfg["match_thresh"], q_r,
                                                     cfg["match_num_thresh"], cfg["reweight"], res_prev)
            mf_r = old_r.keylines()["m_id_f"].copy()
            s_g, J_g, F_g, res_g = new_g.try_vel_rot(old_g, X, rw, pj, cfg["match_thresh"], q_r,
                                                     cfg["match_num_thresh"], cfg["reweight"], res_prev)
            mf_g = old_g.keylines()["m_id_f"]
            tag = "TryVelRot X%d rw=%d pj=%d" % (xi, rw, pj)
            rep.close(tag + " score", s_r, s_g, 1e-10)
            if pj:
                rep.close(tag + " JtJ", J_r, J_g, 1e-9, atol=1e-9 * np.abs(J_r).max())
                rep.close(tag + " JtF", F_r, F_g, 1e-9, atol=1e-9 * np.abs(F_r).max())
            rep.exact(tag + " m_id_f", mf_r, mf_g)
            kl0 = old_r.keylines()
            used = (kl0["s_rho"] <= q_r)
            rep.close(tag + " DResidualNew", res_r[:k0][used], res_g[used], 1e-12, atol=1e-12)
            if pj and not rw:
                res_prev = res_r.copy()
                res_prev[~np.isfinite(res_prev)] = 0
    # full minimisation
    V0, W0 = np.zeros(3), np.zeros(3)
    old_r.set_keylines(_seed_depth(old_r.keylines()))
    m_r = new_r.minimizer_rv(old_r, V0, W0, cfg["match_thresh"], cfg["iter_max"], cfg["init_type"], cfg["reweight"],
                             q_r, cfg["match_num_thresh"], cfg["init_iter"])
    new_g.set_frame_count(0)
    m_g = new_g.minimizer_rv(old_g, V0, W0, cfg["match_thresh"], cfg["iter_max"], cfg["init_type"], cfg["reweight"],
                             q_r, cfg["match_num_thresh"], cfg["init_iter"])
    rep.add("Minimizer_RV values", True, "ref V=%s W=%s F=%.6g" % (m_r["V"], m_r["W"], m_r["F"]))
    rep.close("Minimizer_RV V", m_r["V"], m_g["V"], 0.0, atol=1e-9)     # SURVEY 8(c): abs 1e-9
    rep.close("Minimizer_RV W", m_r["W"], m_g["W"], 0.0, atol=1e-9)
    rep.close("Minimizer_RV F", m_r["F"], m_g["F"], 1e-8)
    rep.close("Minimizer_RV RVel", m_r["RVel"], m_g["RVel"], 1e-8, atol=1e-9 * np.abs(m_r["RVel"]).max())
    rep.close("Minimizer_RV RW0", m_r["RW0"], m_g["RW0"], 1e-8, atol=1e-9 * np.abs(m_r["RW0"]).max())
    rep.close("Minimizer_RV W_X", m_r["W_X"], m_g["W_X"], 1e-8, atol=1e-9 * np.abs(m_r["W_X"]).max())
    rep.close("Minimizer_RV rel_err_score", m_r["rel_err_score"], m_g["rel_err_score"], 1e-8)
    rep.exact("Minimizer_RV m_id_f", old_r.keylines()["m_id_f"], old_g.keylines()["m_id_f"])
    return m_r


@pytest.mark.parametrize("cfg", [TUM_CFG, EUROC_CFG, BIG_CFG], ids=["tum640", "euroc752", "synthetic1280x960"])
def test_stage_parity(built, cfg):
    rep = _run_stage_parity(cfg)
    fails = rep.failures()
    assert not fails, "\n".join("%s: %s" % (f["what"], f["info"]) for f in fails)


def test_box_plan(built):
    """Known-answer constants of iigauss::iigauss (SURVEY.md 8(a) row D2)."""
    from rebvo_b200 import capi
    for sigma0, want in ((1.7818, ([3, 3, 5], [3, 5, 5], 1.825742, 2.160247)),
                         (3.56359, ([7, 7, 7], [9, 9, 9], 3.464102, 4.472136))):
        ctx = capi.Ctx(EUROC_CFG["cam"], sigma0, 1.2599)
        d, s = ctx.box_plan()
        assert d[0].tolist() == want[0] and d[1].tolist() == want[1]
        assert abs(s[0] - want[2]) < 1e-6 and abs(s[1] - want[3]) < 1e-6
        ctx.close()

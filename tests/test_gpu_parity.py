"""GPU parity tests: the CUDA path (through the C ABI) against the UNMODIFIED reference compiled into
oracle/_ref (SURVEY.md section 8(c)), stage by stage, on seeded synthetic frames at the benchmark resolutions.

Bars: float32 scale space, keyline records, id mask and match field bit-exact; float64 per-keyline results
rel 1e-12; reductions over keylines (JtJ, JtF, score) rel 1e-10 (different, fixed summation order);
minimiser outputs abs 1e-9."""
import numpy as np
import pytest

from parity_util import (BIG_CFG, DOG_THRESH, EUROC_CFG, KL_EXACT_DETECT, PLANE_FIT, POS_NEG, TUM_CFG, Report,
                         compare_keylines, parity_frames, tracker_parity)

pytestmark = pytest.mark.gpu


def _run_stage_parity(cfg):
    from oracle import refapi
    from rebvo_b200 import capi
    cam = cfg["cam"]
    rep = Report(cfg["name"])
    f0, f1 = parity_frames(cfg)
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

    m_r = tracker_parity(rep, cfg, refs, gm, rt)
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

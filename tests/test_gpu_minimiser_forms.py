"""Every form of Minimizer_RV against the reference: the four-cluster kernel (the default), the one-cluster kernel
(REBVO_B200_MIN_G=1) and one k_tvr_eval launch per evaluation (REBVO_B200_MIN_PERSIST=0).  All three share the
per-keyline body and the LM steps.  Each form runs test_gpu_parity.py's tracker block on the EuRoC frame pair, with its
bars: the stage-level TryVelRot at three poses x three (reweight, procjf) pairs, then Minimizer_RV, m_id_f exact."""
import pytest

from parity_util import DOG_THRESH, EUROC_CFG, PLANE_FIT, POS_NEG, Report, parity_frames, tracker_parity

pytestmark = pytest.mark.gpu

FORMS = {"four_clusters": {}, "one_cluster": {"REBVO_B200_MIN_G": "1"}, "per_evaluation": {"REBVO_B200_MIN_PERSIST": "0"}}
CLUSTERS = {"four_clusters": 4, "one_cluster": 1, "per_evaluation": 0}


@pytest.mark.parametrize("form", sorted(FORMS))
def test_minimiser_form(built, monkeypatch, form):
    from oracle import refapi
    from rebvo_b200 import capi
    for k in ("REBVO_B200_MIN_G", "REBVO_B200_MIN_PERSIST"):
        monkeypatch.delenv(k, raising=False)
    for k, v in FORMS[form].items():   # read by rb_ctx_create
        monkeypatch.setenv(k, v)
    cfg = EUROC_CFG
    cam = cfg["cam"]
    rep = Report("minimiser " + form)
    refs = [refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], cfg["sigma0"],
                          cfg["ksigma"]) for _ in range(2)]
    ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)
    assert ctx.minimizer_clusters() == CLUSTERS[form]
    gm = [ctx.new_map(), ctx.new_map()]
    # the detector state test_gpu_parity.py's tracker block starts from (its detector stages are checked there)
    det = capi.DetectParams(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["kl_ref"], cfg["gain"], cfg["tmax"],
                            cfg["tmin"])
    t_ref, l_ref = cfg["thresh"], 0
    t_gpu, l_gpu = cfg["thresh"], 0
    for r, g, fr in zip(refs, gm, parity_frames(cfg)):
        r.rgb2bw(fr)
        r.build()
        g.upload_rgb(fr)
        g.dog_build()
        _, t_ref, l_ref = r.detect(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], t_ref, l_ref, cfg["kl_ref"],
                                   cfg["gain"], cfg["tmax"], cfg["tmin"])
        _, t_gpu, l_gpu = g.detect(det, t_gpu, l_gpu)
    refs[1].detect(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], t_ref, l_ref, cfg["kl_ref"], 0.0, 1, 0)
    gm[1].detect(capi.DetectParams(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["kl_ref"], 0.0, 1.0, 0.0),
                 t_ref, l_ref)
    _, rt = refs[1].reestimate(cfg["track_points"], 100)
    gm[1].reestimate(cfg["track_points"], 100)

    m_r = tracker_parity(rep, cfg, refs, gm, rt)
    # the switches took effect: the cluster forms run a minimisation in one launch, the other in one per evaluation
    n0 = ctx.launches()
    gm[1].minimizer_rv(gm[0], m_r["V"], m_r["W"], cfg["match_thresh"], cfg["iter_max"], cfg["init_type"],
                       cfg["reweight"], 1e3, cfg["match_num_thresh"], cfg["init_iter"])
    launches = ctx.launches() - n0
    n_eval = 2 * (cfg["init_iter"] + 1) + cfg["iter_max"] + 1
    assert launches >= n_eval if form == "per_evaluation" else launches <= 2, launches
    for g in gm:
        g.close()
    ctx.close()
    fails = rep.failures()
    assert not fails, "\n".join("%s: %s" % (f["what"], f["info"]) for f in fails)

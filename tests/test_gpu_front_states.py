"""The front end on the device against the unmodified reference, on the states of tests/front_states.py: the detector
(k_update_thresh, k_detect_a<R>, k_seg_scan, k_detect_b, k_join) with thresholds exactly on each of build_mask's
comparisons, kl_max cuts on chosen lanes, segments and scan threads, loaded masks and controller chains;
reEstimateThresh (k_nm_minmax, k_nm_histo) on loaded keylines; build_field (k_build_field) on loaded keyline sets.
Keyline records, mask, kn / threshold state and reTunedThresh bit for bit; the field's winner on every pixel and its
distance where there is one (the reference leaves dist stale on empty pixels).  R = 2 runs the reference in this
process, R = 1, 3 and 4 in one child process each."""
import numpy as np
import pytest

import front_states as fs
from test_cpu_front_states import same_detect

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("R", [1, 2, 3, 4])
def test_detect_states(built, R, tmp_path):
    jobs = fs.detect_jobs(R)
    refs = fs.ref_results(tmp_path, R, jobs)
    ctxs = {}
    try:
        for job, ref in zip(jobs, refs):
            dev = fs.run_dev(job, ctxs)
            port = fs.run_port(job)
            for s, (d, r, p) in enumerate(zip(dev, ref, port)):
                tag = "%s step %d" % (job["name"], s)
                if d["kn"] == 0:
                    # the reference returns its stale kl[0].n_m there; the device returns 0 (DESIGN.md section 3)
                    assert all(x == 0 for x in d["reest"]), tag
                    d = dict(d, reest=r["reest"])
                same_detect(d, r, tag, skip_undefined=p)
    finally:
        for c in ctxs.values():
            c.close()


def test_reestimate_states(built):
    from rebvo_b200 import capi
    cam = fs.CAM
    ctx = capi.Ctx(cam, fs.SIGMA0, fs.KSIGMA, kl_capacity=50000)
    mask = np.full((cam["h"], cam["w"]), -1, np.int32)
    m = ctx.new_map()
    for name, n_m in fs.reest_sets():
        kl = fs.keylines_with(n_m)
        m.load_keylines(kl, mask)
        for k, n in fs.reest_calls(len(kl)):
            want = fs.port_reestimate(n_m, k, n)
            got = np.float32(m.reestimate(k, n))
            assert want.view(np.uint32) == got.view(np.uint32), (name, k, n, want, got)
    for n in (0, 4097):
        with pytest.raises(capi.RbError):
            m.reestimate(10, n)
    m.close()
    ctx.close()


def test_reestimate_matches_reference(built):
    """The same loaded sets on the reference (the restatement is pinned to it by test_cpu_front_states.py; this closes
    the loop on the device directly)."""
    from oracle import refapi
    from rebvo_b200 import capi
    cam = fs.CAM
    ctx = capi.Ctx(cam, fs.SIGMA0, fs.KSIGMA, kl_capacity=50000)
    mask = np.full((cam["h"], cam["w"]), -1, np.int32)
    g = ctx.new_map()
    for name, n_m in fs.reest_sets():
        r = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], fs.SIGMA0, fs.KSIGMA)
        kl = fs.keylines_with(n_m)
        r.set_keylines(kl)
        r.set_mask(mask, len(kl))
        g.load_keylines(kl, mask)
        for k, n in fs.reest_calls(len(kl)):
            want = np.float32(r.reestimate(k, n)[1])
            got = np.float32(g.reestimate(k, n))
            assert want.view(np.uint32) == got.view(np.uint32), (name, k, n, want, got)
    g.close()
    ctx.close()


@pytest.mark.parametrize("kcap", [3000, 50000])
def test_field_states(built, kcap):
    from oracle import refapi
    from rebvo_b200 import capi
    cam = fs.CAM
    w, h = cam["w"], cam["h"]
    ctx = capi.Ctx(cam, fs.SIGMA0, fs.KSIGMA, kl_capacity=kcap)
    mask = np.full((h, w), -1, np.int32)
    g = ctx.new_map()
    for name, kl, runs, _ in fs.field_sets(w, h, 3000):
        r = refapi.RefMap(w, h, cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], fs.SIGMA0, fs.KSIGMA)
        r.set_keylines(kl)
        r.set_mask(mask, len(kl))
        g.load_keylines(kl, mask)
        for radius, min_mod in runs:
            r.build_field(radius, min_mod)
            g.build_field(radius, min_mod)
            want, got = r.field(), g.field()
            assert np.array_equal(want[:, :, 1], got[:, :, 1]), (name, kcap, radius, min_mod)
            won = want[:, :, 1] >= 0
            assert np.array_equal(want[:, :, 0][won], got[:, :, 0][won]), (name, kcap, radius, min_mod)
    g.close()
    ctx.close()


def _pipe_params():
    from rebvo_b200 import capi
    # TrackPoints below kn: reTunedThresh then gates a part of the keylines out of the field
    return capi.default_params(fs.CAM, TrackPoints=1500, **fs.PIPE_DET)


def _stage_chain(p, frames):
    """rb_map_detect + rb_map_reestimate_thresh on each frame with the threshold chained on the host: per frame
    (float(tresh), kn, reTunedThresh)."""
    from rebvo_b200 import capi
    ctx = capi.Ctx(fs.CAM, p.Sigma0, p.KSigma, kl_capacity=p.kl_capacity)
    t, l, out = p.DetectorThresh, 0, []
    m = ctx.new_map()
    for g in frames:
        m.upload_mono(g)
        m.dog_build()
        kn, t, l = m.detect(p.det, t, l)
        out.append((np.float32(t), kn, np.float32(m.reestimate(p.TrackPoints, p.QCutOffNumBins))))
    m.close()
    ctx.close()
    return out


@pytest.mark.parametrize("batch", [5, 8])
def test_pipeline_controller_chain(built, batch):
    """The fused pipeline keeps the detector's feedback (DetChain) on the device across pushes and graph replays: on a
    stream that clamps the threshold at both ends, its per-frame thresh, kn and retuned_thresh are the stage-level
    chain's, bit for bit."""
    from pipeline_util import run_pipeline
    p = _pipe_params()
    ts, frames = fs.pipe_stream()
    want = _stage_chain(p, frames)
    t = np.array([w[0] for w in want])
    assert (t == np.float32(p.det.thresh_max)).sum() >= 3 and (t == np.float32(p.det.thresh_min)).sum() >= 3, t
    nav = run_pipeline(p, ts, frames, batch).nav
    assert len(nav) == len(want)
    for i, (n, w) in enumerate(zip(nav, want)):
        got = (np.float32(n["thresh"]), int(n["kn"]), np.float32(n["retuned_thresh"]))
        assert got[1] == w[1] and got[0].view(np.uint32) == w[0].view(np.uint32) and \
            got[2].view(np.uint32) == w[2].view(np.uint32), (i, got, w)


def test_pipeline_field_min_mod_from_state(built):
    """pl.map(0).field(): the pipeline builds the newest map's field with min_mod = that map's own reTunedThresh read on
    the device; it equals the reference's build_field on that map's keylines with that threshold."""
    from oracle import refapi
    from pipeline_util import push
    from rebvo_b200 import capi
    p = _pipe_params()
    ts, frames = fs.pipe_stream()
    cam = fs.CAM
    pl = capi.Pipeline(p, max_batch=8)
    try:
        for s in range(0, len(ts), 8):
            nav = push(pl, frames[s:s + 8], ts[s:s + 8])
        m = pl.map(0)
        kl, mask, fld = m.keylines(), m.mask(), m.field()
    finally:
        pl.close()
    retuned = np.float32(nav[-1]["retuned_thresh"])
    assert len(kl) == nav[-1]["kn"] > 1000
    dropped = int((kl["n_m"] < retuned).sum())
    assert 100 <= dropped < len(kl) - 100, (dropped, len(kl))   # the gate takes some keylines and keeps others
    r = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], p.Sigma0, p.KSigma)
    r.set_keylines(kl)
    r.set_mask(mask, len(kl))
    r.build_field(p.SearchRange, float(retuned))
    want = r.field()
    assert np.array_equal(want[:, :, 1], fld[:, :, 1])
    won = want[:, :, 1] >= 0
    assert won.sum() > 1000
    assert np.array_equal(want[:, :, 0][won], fld[:, :, 0][won])

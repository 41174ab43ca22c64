"""DetectorPlaneFitSize 1..4 on the device (k_detect_a<R>): the detector, the edge map's mask state, argument checks, the
fused pipeline, the unmodified REBVO on the shim and IMU mode, against the unmodified reference.

The reference caches its plane-fit pseudo inverse per process (edge_finder.cpp:83-84), so every reference result for a
window other than 5x5 comes from a child process (tests/plane_fit.py) or from a whole reference run (ref_rebvo), one
window size per process."""
import os

import numpy as np
import pytest

from parity_util import BIG_CFG, DOG_THRESH, EUROC_CFG, KL_EXACT_DETECT, POS_NEG, TUM_CFG, Report, compare_keylines
from plane_fit import ref_detect_child

pytestmark = pytest.mark.gpu
NF = 60
ERR = "DetectorPlaneFitSize must be 1..4"


def _frames3(cfg):
    from rebvo_b200 import synth
    cam = cfg["cam"]
    if cfg["name"] == "big":
        seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=100, zf=cam["zfx"], nrect_bg=1500, nrect_fg=200)
    else:
        seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=7 if cfg["name"] == "euroc" else 42, zf=cam["zfx"])
    return np.stack([seq.frame(i)[1] for i in (10, 11, 12)])


def border_frame(cam, seed=5):
    """A stream-like frame whose outer 6 rows and columns carry 255 / 0 stripes 7 pixels wide, across the border: edges
    that reach the first interior row and column of every window size."""
    from rebvo_b200 import synth
    rng = np.random.default_rng(seed)
    w, h = cam["w"], cam["h"]
    g = synth.rect_canvas(rng, w, h, 120)
    yy, xx = np.mgrid[0:h, 0:w]
    ring = (np.minimum(xx, w - 1 - xx) < 6) | (np.minimum(yy, h - 1 - yy) < 6)
    stripes = np.where(((xx // 7) + (yy // 7)) % 2 == 0, 255.0, 0.0)
    g = np.where(ring, stripes, g)
    return synth.to_rgb_u8(g, rng)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _det(capi, R, cfg, kl_max=None, gain=None):
    return capi.DetectParams(R, POS_NEG, DOG_THRESH, kl_max or cfg["kl_max"], cfg["kl_ref"],
                             cfg["gain"] if gain is None else gain, cfg["tmax"], cfg["tmin"])


def _ref(tmp_path, cfg, frames, R, **kw):
    return ref_detect_child(tmp_path, frames, R, cfg["cam"], cfg["sigma0"], cfg["ksigma"], cfg["thresh"],
                            kw.pop("kl_max", cfg["kl_max"]), cfg["kl_ref"], kw.pop("gain", cfg["gain"]), cfg["tmax"],
                            cfg["tmin"], POS_NEG, DOG_THRESH, cfg["track_points"], **kw)


@pytest.mark.parametrize("cfg", [TUM_CFG, EUROC_CFG, BIG_CFG], ids=["tum640", "euroc752", "synthetic1280x960"])
def test_stage_parity(built, cfg, tmp_path):
    """rb_map_detect + reEstimateThresh at R = 1, 3, 4 over three frames with the auto-gain feedback chained, and a kl_max
    cut at R = 3: keylines (n_id / p_id included), mask, kn, threshold state bit for bit."""
    from rebvo_b200 import capi
    cam = cfg["cam"]
    frames = _frames3(cfg)
    ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)
    rep = Report("plane_fit_" + cfg["name"])
    small = 5000
    for R in (1, 3, 4):
        ref = _ref(tmp_path, cfg, frames, R, cut=small if R == 3 else None)
        t, l = cfg["thresh"], 0
        maps = []
        for i, fr in enumerate(frames):
            g = ctx.new_map()
            maps.append(g)
            g.upload_rgb(fr)
            g.dog_build()
            kn, t, l = g.detect(_det(capi, R, cfg), t, l)
            want = ref["f%d_kn_tresh" % i].tolist()
            rep.add("R%d f%d kn/tresh/l_kl_num" % (R, i), [kn, t, l] == want, "ref %s gpu %s" % (want, [kn, t, l]))
            compare_keylines(rep, "R%d f%d" % (R, i), ref["f%d_kl" % i], g.keylines(), KL_EXACT_DETECT)
            rep.exact("R%d f%d mask" % (R, i), ref["f%d_mask" % i], g.mask())
            gt = g.reestimate(cfg["track_points"], 100)
            rep.add("R%d f%d reEstimateThresh" % (R, i), np.float32(gt) == ref["f%d_retuned" % i][0],
                    "ref %.9g gpu %.9g" % (ref["f%d_retuned" % i][0], gt))
            assert kn > 1000
        if R == 3:
            kn, _, _ = maps[-1].detect(_det(capi, R, cfg, kl_max=small, gain=0.0), t, l)
            rep.add("R3 cut kn", kn == int(ref["cut_kn"][0]) == small, "ref %d gpu %d" % (ref["cut_kn"][0], kn))
            compare_keylines(rep, "R3 cut", ref["cut_kl"], maps[-1].keylines(), KL_EXACT_DETECT)
            rep.exact("R3 cut mask", ref["cut_mask"], maps[-1].mask())
        for g in maps:
            g.close()
    rep.dump()
    ctx.close()
    fails = rep.failures()
    assert not fails, "\n".join("%s: %s" % (f["what"], f["info"]) for f in fails)


def test_border_rows_and_columns(built, tmp_path):
    """Strong edges across the border: the keylines on the first interior row / column (x = R or y = R) are the
    reference's, and nothing outside the interior is marked."""
    from rebvo_b200 import capi
    cfg = EUROC_CFG
    cam = cfg["cam"]
    fr = border_frame(cam)
    ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)
    for R in (1, 3, 4):
        ref = _ref(tmp_path, cfg, fr[None], R, gain=0.0)
        g = ctx.new_map()
        g.upload_rgb(fr)
        g.dog_build()
        kn, _, _ = g.detect(_det(capi, R, cfg, gain=0.0), cfg["thresh"], 0)
        kl, mask = g.keylines(), g.mask()
        x, y = kl["p_inx"] % cam["w"], kl["p_inx"] // cam["w"]
        edge = (x == R) | (y == R) | (x == cam["w"] - 1 - R) | (y == cam["h"] - 1 - R)
        assert edge.sum() > 20, (R, int(edge.sum()))
        rk = ref["f0_kl"]
        assert kn == len(rk)
        for f in KL_EXACT_DETECT:
            assert np.array_equal(_bits(rk[f]), _bits(kl[f])), (R, f)
        assert np.array_equal(ref["f0_mask"], mask)
        inner = np.zeros_like(mask, bool)
        inner[R:-R, R:-R] = True
        assert (mask[~inner] == -1).all()
        g.close()
    ctx.close()


def test_window_switch_on_one_map(built):
    """R = 1 then R = 3 on one map (and on a clone of the R = 1 map) gives a fresh map's R = 3 result: the ids the 3x3
    window left between the two margins are cleared.  R = 3 then R = 1 likewise."""
    from rebvo_b200 import capi
    cfg = EUROC_CFG
    cam = cfg["cam"]
    fr = border_frame(cam, seed=9)
    ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)

    def run(seq):
        m = ctx.new_map()
        m.upload_rgb(fr)
        m.dog_build()
        for R in seq:
            m.detect(_det(capi, R, cfg, gain=0.0), cfg["thresh"], 0)
        return m

    def detect_ss(m, src, R):   # (a clone has no scale space of its own: it detects on its source's planes)
        import ctypes as C
        t, l, kn = C.c_double(cfg["thresh"]), C.c_int(0), C.c_int(0)
        det = _det(capi, R, cfg, gain=0.0)
        ctx.check(ctx.L.rb_map_detect_ss(m.h_, src.h_, C.byref(det), C.byref(t), C.byref(l), C.byref(kn)))

    for a, b in ((1, 3), (3, 1), (1, 4)):
        fresh = run([b])
        want_kl, want_mask = fresh.keylines(), fresh.mask()
        one = run([a, b])
        assert np.array_equal(one.mask(), want_mask), (a, b)
        assert one.keylines().tobytes() == want_kl.tobytes(), (a, b)
        # clone of the R = a map: the radius of the last detect travels with the copy
        m = run([a])
        c = m.clone()
        detect_ss(c, m, b)
        assert np.array_equal(c.mask(), want_mask), ("clone", a, b)
        assert c.keylines().tobytes() == want_kl.tobytes(), ("clone", a, b)
        for x in (fresh, one, m, c):
            x.close()
    ctx.close()


def test_rejected_sizes(built):
    """R outside 1..4: RB_ERR_ARG with the message before anything is enqueued (the map is untouched), and the context
    then detects at R = 2 like the reference.  A pipeline refuses such a size at creation."""
    from oracle import refapi
    from rebvo_b200 import capi
    cfg = TUM_CFG
    cam = cfg["cam"]
    fr = _frames3(cfg)[0]
    ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)
    m = ctx.new_map()
    m.upload_rgb(fr)
    m.dog_build()
    kn0, _, _ = m.detect(_det(capi, 3, cfg, gain=0.0), cfg["thresh"], 0)
    kl0, mask0 = m.keylines(), m.mask()
    launches = ctx.launches()
    for R in (0, -1, 5):
        with pytest.raises(capi.RbError, match=ERR):
            m.detect(_det(capi, R, cfg, gain=0.0), cfg["thresh"], 0)
    assert ctx.launches() == launches
    assert m.knum() == kn0 and np.array_equal(m.mask(), mask0) and m.keylines().tobytes() == kl0.tobytes()
    kn, _, _ = m.detect(_det(capi, 2, cfg, gain=0.0), cfg["thresh"], 0)
    if refapi.available():
        r = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], cfg["sigma0"], cfg["ksigma"])
        r.rgb2bw(fr)
        r.build()
        knr, _, _ = r.detect(2, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["thresh"], 0, cfg["kl_ref"], 0.0, cfg["tmax"],
                             cfg["tmin"])
        assert knr == kn
        assert np.array_equal(r.mask(), m.mask())
        rk, gk = r.keylines(), m.keylines()
        for f in KL_EXACT_DETECT:
            assert np.array_equal(_bits(rk[f]), _bits(gk[f])), f
    m.close()
    ctx.close()
    from rebvo_b200 import synth
    for R in (0, 5):
        with pytest.raises(capi.RbError, match="rb_pipeline_create failed"):
            capi.Pipeline(capi.default_params(synth.EUROC, plane_fit_size=R), max_batch=4)


def _stream(nf=NF):
    from rebvo_b200 import synth
    cam = synth.EUROC
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=7, zf=cam["zfx"])
    ts, fr = seq.frames(nf)
    return cam, seq, ts, fr


def _run(p, ts, fr, batch):
    from rebvo_b200 import capi
    pl = capi.Pipeline(p, max_batch=batch)
    nav = np.concatenate([pl.push(fr[s:s + batch], ts[s:s + batch]) for s in range(0, len(ts), batch)])
    pl.close()
    return nav


@pytest.mark.parametrize("R", [1, 3])
def test_pipeline_vs_reference(built, R, tmp_path):
    """The fused pipeline at R against the reference's whole REBVO run with the same DetectorPlaneFitSize."""
    from oracle import refapi
    from rebvo_b200 import capi, synth
    if not os.path.exists(refapi.EXE):
        pytest.skip("oracle/_ref/ref_rebvo not built")
    cam, _, ts, fr = _stream()
    p = capi.default_params(cam, plane_fit_size=R)
    nav = _run(p, ts, fr, 20)
    nav7 = _run(p, ts, fr, 7)
    assert nav.tobytes() == nav7.tobytes()
    path = str(tmp_path / "frames.bin")
    synth.write_frames_file(path, ts, fr)
    _, ref = refapi.run_full_rebvo(path, path + ".ref", refapi.ref_params_from(p))
    n = min(len(ref), len(nav))
    assert n >= NF - 2
    e = np.sqrt(((ref["Pos"][:n] - nav["Pos"][:n]) ** 2).sum(1))
    ate = float(np.sqrt((e ** 2).mean()))
    first = int(np.nonzero(e > 1e-9)[0][0]) if (e > 1e-9).any() else -1
    dm = np.abs(ref["matches"][1:n].astype(int) - nav["matches"][1:n].astype(int))
    print("R=%d pipeline vs reference: ATE %.3e m over %d frames, first frame above 1e-9 m: %d, max |d matches| %d, "
          "kn %d..%d" % (R, ate, n, first, dm.max(), nav["kn"][:n].min(), nav["kn"][:n].max()))
    assert np.array_equal(ref["kn"][:n], nav["kn"][:n])
    assert np.array_equal(ref["est_ok"][1:n] != 0, nav["estimation_ok"][1:n] != 0)
    # the detector is bit-exact; the tracker's sums run in another order, so a frame whose LM decision sits on a knife
    # edge may take the other branch (as in test_gpu_dropin.py): matches within 0.5 %, poses within north_star's bar
    assert dm.max() <= 0.005 * ref["matches"][1:n].max(), dm.max()
    assert ate <= 1e-3 and e.max() <= 1e-3


def test_dropin_shim_at_r3(built, tmp_path):
    """The unmodified REBVO on include/rebvo_b200_shim.hpp with DetectorPlaneFitSize=3 equals the fused pipeline at R = 3."""
    from oracle import refapi
    from rebvo_b200 import capi, synth
    shim_exe = os.path.join(os.path.dirname(refapi.EXE), "shim_rebvo")
    if not os.path.exists(shim_exe):
        pytest.skip("oracle/_ref/shim_rebvo not built")
    cam, _, ts, fr = _stream()
    p = capi.default_params(cam, plane_fit_size=3)
    path = str(tmp_path / "frames.bin")
    synth.write_frames_file(path, ts, fr)
    _, rec = refapi.run_full_rebvo(path, path + ".shim", refapi.ref_params_from(p), exe=shim_exe)
    nav = _run(p, ts, fr, 20)
    n = min(len(rec), len(nav))
    assert n >= NF - 2
    assert np.array_equal(nav["kn"][:n], rec["kn"][:n])
    assert np.array_equal(nav["matches"][1:n], rec["matches"][1:n])
    assert np.abs(nav["Pos"][:n] - rec["Pos"][:n]).max() <= 1e-9


def test_imu_mode_kn_at_r3(built):
    """IMU mode (rb_pipeline_set_imu) at R = 3: the same kn per frame as vision only -- kn depends on the detector and its
    threshold feedback alone."""
    from rebvo_b200 import capi, synth
    nf = 50
    cam, seq, ts, fr = _stream(nf)
    p = capi.default_params(cam, plane_fit_size=3)
    vis = _run(p, ts, fr, 10)
    pl = capi.Pipeline(p, max_batch=10)
    pl.set_imu(synth.imu_samples(seq, nf), capi.default_imu_params(InitBias=1, InitBiasFrameNum=5))
    nav = np.concatenate([pl.push(fr[s:s + 10], ts[s:s + 10]) for s in range(0, nf, 10)])
    pl.close()
    assert np.array_equal(vis["kn"], nav["kn"])
    assert np.isfinite(nav["Pos"]).all()

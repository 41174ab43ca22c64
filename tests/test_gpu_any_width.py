"""Frames of any width (w % 4 != 0): the scale-space planes are row-pitched (rows of w rounded up to 4 floats) and the input
stage reads packed frames whose rows and frames start at any byte.  KITTI odometry's 1241x376 and 1226x370, and geometries
with w = 1, 2, 3 (mod 4) and w * h odd or even, against the reference (compiled from its sources into oracle/_ref, which
takes any size): scale-space planes and the detector bit for bit, the fused pipeline and the unmodified REBVO on the shim
against the reference's three-thread run, and every way of feeding frames byte-identical to the host RGB push."""
import numpy as np
import pytest

from parity_util import DOG_THRESH, KL_EXACT_DETECT, POS_NEG
from pipeline_util import (assert_knife_edge, assert_runs_identical, assert_shim_equals, push, run_pipeline,
                           run_reference, shim_exe)
from plane_fit import ref_detect_child

pytestmark = pytest.mark.gpu

GEOMETRIES = [(1241, 376), (1226, 370), (750, 97), (37, 33), (331, 244)]
KITTI = [(1241, 376), (1226, 370)]
NF = 60
KC = (-0.12, 0.03, 0.0, 1e-4, 2e-5)   # a mild rad-tan model for UseUndistort=1


def _cam(w, h):
    return dict(w=w, h=h, zfx=718.856, zfy=718.856, ppx=w / 2.0 - 13.3, ppy=h / 2.0 - 2.8)


def _seq(w, h, seed=7):
    from rebvo_b200 import synth
    return synth.Sequence(w=w, h=h, seed=seed, zf=718.0)


def _u32(a):
    return np.ascontiguousarray(a).view(np.uint32)


# ---- 1. scale space -------------------------------------------------------------------------------------------------
def _inputs(w, h, seed):
    rng = np.random.default_rng(seed)
    rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    rgb[h // 3:, w // 4:] //= 3   # an edge, so that the planes are not just noise
    mono = rng.integers(0, 256, (h, w), dtype=np.uint8)
    mono[: h // 2, w // 3:] //= 4
    gray = (rng.random((h, w)) * 765.0).astype(np.float32)
    return rgb, mono, gray


def _ref_planes(w, h, sigma0, how, img):
    from oracle import refapi
    r = refapi.RefMap(w, h, w / 2.0, h / 2.0, 300.0, 300.0, sigma0, 1.2599)
    if how == "gray":
        r.set_gray(img)
    else:
        r.rgb2bw(img if how == "rgb" else np.repeat(img[:, :, None], 3, axis=2))
    r.build()
    return {k: r.plane(k).copy() for k in ("gray", "img0", "img1", "dog")}


def _gpu_planes(w, h, sigma0, how, img):
    from rebvo_b200 import capi
    cam = dict(w=w, h=h, zfx=300.0, zfy=300.0, ppx=w / 2.0, ppy=h / 2.0)
    ctx = capi.Ctx(cam, sigma0, 1.2599, kl_capacity=20000)
    m = ctx.new_map()
    getattr(m, "upload_" + how)(img)
    m.dog_build()
    out = {k: m.plane(k).copy() for k in ("gray", "img0", "img1", "dog")}
    m.close()
    ctx.close()
    return out


@pytest.mark.parametrize("env", [{}], ids=["tma"])
@pytest.mark.parametrize("sigma0", [1.7818, 3.56359])
def test_scale_space_bitwise(built, monkeypatch, sigma0, env):
    """gray, Img(0), Img(1), DoG of RGB, mono and float uploads equal the reference's sspace::build bit for bit (the TMA
    kernels, whose tensor maps serve every width)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for gi, (w, h) in enumerate(GEOMETRIES):
        rgb, mono, gray = _inputs(w, h, 100 + gi)
        for how, img in (("rgb", rgb), ("mono", mono), ("gray", gray)):
            ref = _ref_planes(w, h, sigma0, how, img)
            got = _gpu_planes(w, h, sigma0, how, img)
            for k in ref:
                assert ref[k].shape == got[k].shape == (h, w)
                bad = int((_u32(ref[k]) != _u32(got[k])).sum())
                assert bad == 0, "%dx%d sigma0 %.2f %s upload, plane %s: %d pixels differ" % (w, h, sigma0, how, k, bad)
            if how == "mono":
                assert np.array_equal(got["gray"], 3.0 * mono.astype(np.float32))


def test_context_size_limits(built):
    """Any width and height from 32 up is accepted, narrower or shorter frames are not."""
    from rebvo_b200 import capi
    for w, h in ((32, 32), (33, 32), (34, 35), (35, 32), (1241, 376)):
        capi.Ctx(_cam(w, h), 1.7818, 1.2599, kl_capacity=1000).close()
    for w, h in ((31, 64), (64, 31)):
        with pytest.raises(capi.RbError):
            capi.Ctx(_cam(w, h), 1.7818, 1.2599, kl_capacity=1000)


# ---- 2. detector ----------------------------------------------------------------------------------------------------
def _det_cfg(w, h):
    return dict(name="kitti", cam=_cam(w, h), sigma0=3.56359, ksigma=1.2599, thresh=0.01, gain=5e-7, tmax=0.5,
                tmin=0.005, kl_max=40000, kl_ref=15000, track_points=12000)


def _frames3(w, h):
    seq = _seq(w, h, seed=21)
    return np.stack([seq.frame(i)[1] for i in (10, 11, 12)])


def _det(capi, R, cfg):
    return capi.DetectParams(R, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["kl_ref"], cfg["gain"], cfg["tmax"], cfg["tmin"])


def _gpu_detect(cfg, frames, R):
    """detect + reEstimateThresh on each frame, the threshold chained: [(kn, tresh, l_kl_num, keylines, mask, retuned)]"""
    from rebvo_b200 import capi
    ctx = capi.Ctx(cfg["cam"], cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)
    t, l, out = cfg["thresh"], 0, []
    for fr in frames:
        m = ctx.new_map()
        m.upload_rgb(fr)
        m.dog_build()
        kn, t, l = m.detect(_det(capi, R, cfg), t, l)
        out.append((kn, t, l, m.keylines(), m.mask(), m.reestimate(cfg["track_points"], 100)))
        m.close()
    ctx.close()
    return out


def _assert_detect(got, ref_kn_t_l, ref_kl, ref_mask, ref_retuned, what):
    kn, t, l, kl, mask, retuned = got
    assert [kn, t, l] == list(ref_kn_t_l), "%s: kn/tresh/l_kl_num gpu %s ref %s" % (what, [kn, t, l], list(ref_kn_t_l))
    assert kn > 1000, what
    assert len(kl) == len(ref_kl), what
    for f in KL_EXACT_DETECT:
        assert np.array_equal(np.ascontiguousarray(ref_kl[f]).view(np.uint8), np.ascontiguousarray(kl[f]).view(np.uint8)), \
            "%s: keyline field %s" % (what, f)
    assert np.array_equal(ref_mask, mask), "%s: mask" % what
    assert np.float32(retuned) == np.float32(ref_retuned), "%s: reTunedThresh gpu %r ref %r" % (what, retuned, ref_retuned)


@pytest.mark.parametrize("wh", KITTI, ids=["1241x376", "1226x370"])
def test_detector_r2_vs_reference(built, wh):
    """DetectorPlaneFitSize 2 against the in-process reference: keylines, mask, kn and the threshold feedback over three
    chained frames, and reEstimateThresh."""
    from oracle import refapi
    cfg = _det_cfg(*wh)
    cam = cfg["cam"]
    frames = _frames3(*wh)
    got = _gpu_detect(cfg, frames, 2)
    t, l = cfg["thresh"], 0
    for i, fr in enumerate(frames):
        r = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], cfg["sigma0"], cfg["ksigma"])
        r.rgb2bw(fr)
        r.build()
        kn, t, l = r.detect(2, POS_NEG, DOG_THRESH, cfg["kl_max"], t, l, cfg["kl_ref"], cfg["gain"], cfg["tmax"], cfg["tmin"])
        retuned = r.reestimate(cfg["track_points"], 100)[1]
        _assert_detect(got[i], (kn, t, l), r.keylines(), r.mask(), retuned, "%dx%d R2 frame %d" % (wh + (i,)))


@pytest.mark.parametrize("wh", KITTI, ids=["1241x376", "1226x370"])
def test_detector_other_windows_vs_reference(built, wh, tmp_path):
    """DetectorPlaneFitSize 1, 3 and 4, each against the reference in a process of its own (its pseudo inverse is cached
    per process)."""
    cfg = _det_cfg(*wh)
    frames = _frames3(*wh)
    for R in (1, 3, 4):
        ref = ref_detect_child(tmp_path, frames, R, cfg["cam"], cfg["sigma0"], cfg["ksigma"], cfg["thresh"], cfg["kl_max"],
                               cfg["kl_ref"], cfg["gain"], cfg["tmax"], cfg["tmin"], POS_NEG, DOG_THRESH,
                               cfg["track_points"])
        got = _gpu_detect(cfg, frames, R)
        for i in range(len(frames)):
            k = ref["f%d_kn_tresh" % i].tolist()
            _assert_detect(got[i], (int(k[0]), k[1], int(k[2])), ref["f%d_kl" % i], ref["f%d_mask" % i],
                           ref["f%d_retuned" % i][0], "%dx%d R%d frame %d" % (wh + (R, i)))


# ---- 3. / 4. whole pipeline against the reference ----------------------------------------------------------------------
@pytest.fixture(scope="module")
def kitti_stream():
    w, h = KITTI[0]
    ts, fr = _seq(w, h, seed=13).frames(NF)
    return _cam(w, h), ts, fr


@pytest.mark.parametrize("kc", [None, KC], ids=["plain", "undistort"])
def test_pipeline_vs_reference(built, kitti_stream, kc, tmp_path):
    """The fused pipeline at 1241x376 against the reference's three-thread REBVO: identical keyline counts, match counts and
    poses within the bars of the drop-in test (a frame whose LM decision sits on a knife edge may take the other branch),
    equal estimation_ok."""
    from rebvo_b200 import capi
    cam, ts, fr = kitti_stream
    p = capi.default_params(cam)
    _, ref = run_reference(tmp_path, ts, fr, p, kc=kc)
    nav = run_pipeline(p, ts, fr, 20, kc=kc).nav
    assert_knife_edge(ref, nav, NF - 2, "1241x376 " + ("undistorted" if kc else "plain"))
    assert nav["kn"][:len(ref)].min() > 1000


def test_unmodified_rebvo_on_the_gpu_library(built, kitti_stream, tmp_path):
    """The reference's own REBVO class on include/rebvo_b200_shim.hpp at 1241x376: it initialises, is identical run after
    run, and equals the fused pipeline."""
    from rebvo_b200 import capi
    cam, ts, fr = kitti_stream
    p = capi.default_params(cam)
    runs = [run_reference(tmp_path, ts, fr, p, exe=shim_exe())[1].copy() for _ in range(2)]
    n = min(len(r) for r in runs)
    assert n >= NF - 2
    for f in ("kn", "matches", "Pos", "PoseLie", "Kp", "est_ok"):
        assert np.array_equal(runs[0][f][:n], runs[1][f][:n]), f
    assert_shim_equals(run_pipeline(p, ts, fr, 20).nav[:n], runs[0][:n])


# ---- 5. every way of feeding frames --------------------------------------------------------------------------------
FEED_NF = 20
# the two KITTI sizes (w * h % 4 == 0) and one with w = 3 (mod 4) and w * h odd, so that mono frames after the first start
# at odd bytes of a device buffer
FEED_GEOMETRIES = KITTI + [(1239, 375)]


@pytest.fixture(scope="module", params=FEED_GEOMETRIES, ids=["%dx%d" % g for g in FEED_GEOMETRIES])
def feed(request):
    w, h = request.param
    ts, rgb = _seq(w, h, seed=5).frames(FEED_NF)
    assert np.array_equal(rgb[..., 0], rgb[..., 1]) and np.array_equal(rgb[..., 0], rgb[..., 2])
    return _cam(w, h), ts, rgb


def _feed(feed, fmt="rgb", how="host", batch=FEED_NF, offset=0, kc=None, mirror=0):
    from rebvo_b200 import capi
    cam, ts, rgb = feed
    return run_pipeline(capi.default_params(cam), ts, rgb, batch, how, fmt, offset, kc, mirror,
                        check_mirror=bool(mirror))


@pytest.mark.parametrize("kc", [None, KC], ids=["plain", "undistort"])
def test_feeds_byte_identical(built, feed, monkeypatch, kc):
    """Host / device, RGB / mono (mono = RGB of the replicated frames), batches 20, 7 and 1, the 5-frame head / rest cut of
    host pushes, and device buffers whose frames start at odd bytes: one set of nav records."""
    ref = _feed(feed, kc=kc)
    assert np.isfinite(ref.nav["Pos"]).all() and ref.nav["kn"].min() > 500
    assert_runs_identical(ref, _feed(feed, "rgb", "device", kc=kc), "device RGB")
    assert_runs_identical(ref, _feed(feed, "mono", kc=kc), "host mono")
    assert_runs_identical(ref, _feed(feed, "mono", "device", kc=kc), "device mono")
    for batch in (7, 1):
        assert_runs_identical(ref, _feed(feed, "rgb", batch=batch, kc=kc), "host RGB batch %d" % batch)
        assert_runs_identical(ref, _feed(feed, "mono", "device", batch=batch, kc=kc), "device mono batch %d" % batch)
    for off in (1, 3):
        assert_runs_identical(ref, _feed(feed, "rgb", "device", offset=off, kc=kc),
                              "device RGB at byte offset %d" % off)
    monkeypatch.setenv("REBVO_B200_SUB", "5")
    assert_runs_identical(ref, _feed(feed, "rgb", kc=kc), "host RGB, SUB=5")
    assert_runs_identical(ref, _feed(feed, "mono", kc=kc), "host mono, SUB=5")


def test_misaligned_mono_device_base_refused(built, feed):
    """The device mono entry point keeps its rule: a base pointer that is not 4-byte aligned is refused."""
    from rebvo_b200 import capi
    cam, ts, rgb = feed
    mono = rgb[:4, ..., 0]
    pl = capi.Pipeline(capi.default_params(cam), max_batch=4)
    for off in (1, 2, 3):
        with pytest.raises(capi.RbError):
            push(pl, mono, ts[:4], "device", offset=4 + off)
    pl.close()


@pytest.mark.parametrize("mode", [1, 2])
def test_mirror(built, feed, mode):
    """Mirror modes 1 and 2 with one-frame pushes: every frame's records equal rb_map_sync_host_keylines /
    rb_map_pack_net_keylines of the same map, and the mirror leaves the nav records unchanged."""
    ref = _feed(feed, batch=1)
    assert_runs_identical(ref, _feed(feed, "rgb", batch=1, mirror=mode), "RGB, mirror %d" % mode)
    assert_runs_identical(ref, _feed(feed, "mono", batch=1, mirror=mode), "mono, mirror %d" % mode)


def test_imu_mode_mono_equals_rgb(built, feed):
    from rebvo_b200 import capi, synth
    cam, ts, rgb = feed
    n, B = 10, 5
    imu = synth.imu_samples(_seq(cam["w"], cam["h"], seed=5), n)
    out = [run_pipeline(capi.default_params(cam), ts[:n], rgb[:n], B, fmt=fmt, imu=imu) for fmt in ("rgb", "mono")]
    assert_runs_identical(out[0], out[1], "IMU mode")
    assert np.isfinite(out[0].nav["Pos"]).all()

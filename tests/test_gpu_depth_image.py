"""The dense inverse-depth image of the viewer's depth grid (depth_filler::getImgRho at every pixel) on the device:
rb_depth_image and the pipeline's per-frame images, bit for bit against the header's own getImgRho on the unmodified
reference depth_filler (oracle/_ref/libref_depth_image.so, built by oracle/ref_depth_image.py)."""
import numpy as np
import pytest

import pipeline_util as pu
from test_gpu_depth_fill import CAM_1280, KITTI, in_grid, make_records, params, tracked_records

pytestmark = pytest.mark.gpu


def _ref():
    from oracle import ref_depth, ref_depth_image
    if not ref_depth_image.available():
        if ref_depth.available():   # the reference was compiled here, so this library must have been too
            pytest.fail("oracle/_ref/libref_depth.so was built but oracle/_ref/libref_depth_image.so was not")
        pytest.skip("oracle/_ref/libref_depth_image.so not built")
    return ref_depth_image


def _cams():
    from rebvo_b200 import synth
    return {"euroc": synth.EUROC, "tum": synth.TUM, "kitti": KITTI, "1280": CAM_1280}


def float_exact(ref):
    """getImgRho returns a float widened to double: the float32 planes hold it exactly."""
    f = ref.astype(np.float32)
    assert np.array_equal(f.astype(np.float64), ref)
    return f


def assert_plane_equal(got, want, what):
    assert got.shape == want.shape and got.dtype == np.float32, (what, got.shape, want.shape)
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert len(bad) == 0, "%s: %d pixels differ, first %s: %r vs %r" % (what, len(bad), bad[0], got[tuple(bad[0])],
                                                                      want[tuple(bad[0])])


def assert_image_equal(img, ref, what):
    """img: (rho, s_rho or None) float32; ref: (rho, s_rho) float64 of the reference."""
    assert_plane_equal(img[0], float_exact(ref[0]), what + " rho")
    if img[1] is not None:
        assert_plane_equal(img[1], float_exact(ref[1]), what + " s_rho")


@pytest.fixture(scope="module")
def ctxs(built):
    from rebvo_b200 import capi
    out = {n: capi.Ctx(c, 3.56359, 1.2599, kl_capacity=40000) for n, c in _cams().items()}
    yield out
    for c in out.values():
        c.close()


# ---- 1. one-shot on tracked maps, against the reference ------------------------------------------------------------------
def blocks_of(cam):
    """10x10, 16x16, 7x13, one block as large as the frame (gw = gh = 1: every pixel takes the negative-dx path), and a
    block that leaves remainder columns and rows on this camera."""
    w, h = cam["w"], cam["h"]
    rem = next((bw, bh) for bw, bh in ((9, 7), (11, 7), (13, 11), (9, 13)) if w % bw and h % bh)
    return [(10, 10), (16, 16), (7, 13), (w, h), rem]


@pytest.mark.parametrize("cam", ["euroc", "tum", "kitti", "1280"])
def test_one_shot_tracked_maps(ctxs, cam):
    ref = _ref()
    c = _cams()[cam]
    for bw, bh in blocks_of(c):
        for age, rec in enumerate(tracked_records(cam)):
            rec = in_grid(rec, c, bw, bh)
            for thr, mnum, iters in ((1.0, 5, 10), (1e9, 0, 3)):
                p = params(bw, bh, thr, mnum, iters)
                cells, _ = ctxs[cam].depth_fill_net(rec, p)
                img = ctxs[cam].depth_image(cells, p)
                what = "%s %dx%d map %d (%g, %d, %d)" % (cam, bw, bh, age, thr, mnum, iters)
                assert_image_equal(img, ref.depth_image_net(c, rec, bw, bh, thr, mnum, iters), what)
                rho_only, none = ctxs[cam].depth_image(cells, p, s_rho=False)
                assert none is None and rho_only.tobytes() == img[0].tobytes(), what


# ---- 2. crafted grids -----------------------------------------------------------------------------------------------------
def crafted(rng, gw, gh, kind):
    """Values a fill produces: fused cells (rho up to 65535 / 1e4, small s_rho), the prior of an empty grid (1, 40),
    zeros, and doubles that round when cast to float, including ones below float's normal range."""
    if kind == "random":
        return rng.uniform(0, 6.5535, (gh, gw)), rng.uniform(1e-5, 40, (gh, gw))
    rho = rng.choice([0.0, 1e-4, 6.5535, 1.0, 1 / 3, 5e-324, 1e-40, 1e20], (gh, gw))
    s_rho = rng.choice([1e-4 / np.sqrt(200), 40.0, 1e-4, 1e10, 0.0, 2.0 / 3], (gh, gw))
    return rho, s_rho


def cells_of(rho, s_rho):
    from rebvo_b200 import capi
    cells = np.zeros(rho.shape, capi.DEPTH_CELL)
    cells["rho"], cells["s_rho"], cells["dist"], cells["fixed"] = rho, s_rho, 7.0, 1
    return cells


# (camera, block): first / last rows and columns with and without remainders, gw = 1, gh = 1, and grids too large for
# shared memory (2x2, 3x3 and 1x1 blocks: as many cells as the frame has pixels), read in place from global memory
CRAFTED = [("euroc", 10, 10), ("euroc", 9, 7), ("euroc", 752, 3), ("euroc", 5, 480), ("euroc", 752, 480), ("euroc", 4, 4),
           ("euroc", 3, 3), ("euroc", 2, 2), ("euroc", 1, 1), ("kitti", 16, 16), ("kitti", 1241, 9), ("1280", 10, 10),
           ("1280", 6, 5), ("tum", 13, 11)]


@pytest.mark.parametrize("kind", ["random", "extremes"])
@pytest.mark.parametrize("cam,bw,bh", CRAFTED, ids=["%s_%dx%d" % c for c in CRAFTED])
def test_crafted_grids(ctxs, cam, bw, bh, kind):
    ref = _ref()
    c = _cams()[cam]
    gw, gh = c["w"] // bw, c["h"] // bh
    rng = np.random.default_rng(gw * 31 + gh)
    rho, s_rho = crafted(rng, gw, gh, kind)
    img = ctxs[cam].depth_image(cells_of(rho, s_rho), params(bw, bh))
    assert_image_equal(img, ref.depth_image_cells(c["w"], c["h"], bw, bh, rho, s_rho), "%s %dx%d %s" % (cam, bw, bh, kind))


def test_one_shot_arguments(ctxs):
    from rebvo_b200 import capi
    ctx = ctxs["euroc"]
    cells = cells_of(np.ones((48, 75)), np.ones((48, 75)))
    for bad in (params(0, 10), params(10, 0), params(753, 10), params(10, 481), params(iters=-1)):
        with pytest.raises(capi.RbError, match="-2"):
            ctx.depth_image(cells, bad)
    for shape in ((48, 74), (47, 75), (75, 48)):   # not the grid size of the parameters on this camera
        with pytest.raises(capi.RbError, match="-2"):
            ctx.depth_image(cells_of(np.ones(shape), np.ones(shape)), params())
    ctx.depth_image(cells, params())


# ---- 3. the pipeline's per-frame images ---------------------------------------------------------------------------------
def run_image(prm, ts, frames, batch, how="host", fmt="rgb", mirror=2, mode=2, depth=True, odometry=False):
    """Pushes of `batch` frames with the depth grid (viewer parameters) and images of `mode`; per frame: nav, mirror
    records, (cells, min_dist), (rho, s_rho) copies; the launches of each push; odometry records."""
    from rebvo_b200 import capi
    pl = capi.Pipeline(prm, max_batch=batch)
    navs, mirrors, grids, images, launches, odo = [], [], [], [], [], []
    try:
        if mirror:
            pl.set_mirror(mirror)
        if mode:
            pl.set_depth_image(mode)
        if depth:
            pl.set_depth(params())
        if odometry:
            pl.set_odometry(True)
        for s in range(0, len(ts), batch):
            src = frames[s:s + batch, ..., 0] if fmt == "mono" else frames[s:s + batch]
            l0 = pl.launches()
            nav = pu.push(pl, src, ts[s:s + batch], how)
            launches.append(pl.launches() - l0)
            navs.append(nav)
            for i in range(len(nav)):
                if mirror:
                    mirrors.append(pl.mirror(i).copy())
                if depth:
                    grids.append(pl.depth(i))
                if depth and mode:
                    r, sr = pl.depth_image(i)
                    images.append((r.copy(), None if sr is None else sr.copy()))
            if odometry:
                odo.append(pl.odometry())
    finally:
        pl.close()
    return dict(nav=np.concatenate(navs), mirrors=mirrors, grids=grids, images=images, launches=launches,
                odometry=np.concatenate(odo) if odo else None)


def assert_images_match(run, ctx, cam, mode, what):
    """Every frame's image equals rb_depth_image on that frame's cells, byte for byte, and the reference: on that frame's
    records (mirror mode 2) or on its cells."""
    ref = _ref()
    assert len(run["images"]) == len(run["grids"]) == len(run["nav"])
    p = params()
    for f, ((cells, _), img) in enumerate(zip(run["grids"], run["images"])):
        assert img[0].shape == (cam["h"], cam["w"]) and (img[1] is None) == (mode == 1), (what, f)
        one = ctx.depth_image(cells, p, s_rho=mode == 2)
        assert img[0].tobytes() == one[0].tobytes(), "%s frame %d: rho against rb_depth_image" % (what, f)
        if mode == 2:
            assert img[1].tobytes() == one[1].tobytes(), "%s frame %d: s_rho against rb_depth_image" % (what, f)
        if run["mirrors"] and run["mirrors"][f].dtype == np.uint8:
            want = ref.depth_image_net(cam, in_grid(run["mirrors"][f], cam, 10, 10), 10, 10, 1.0, 5, 10)
        else:
            want = ref.depth_image_cells(cam["w"], cam["h"], 10, 10, cells["rho"], cells["s_rho"])
        assert_image_equal(img, want, "%s frame %d" % (what, f))


@pytest.mark.parametrize("batch,n,how,fmt,mirror,mode", [
    (1, 4, "host", "rgb", 2, 2), (7, 14, "dev", "rgb", 0, 1), (7, 14, "host", "mono", 1, 2), (7, 14, "dev", "mono", 2, 1),
    (64, 64, "host", "rgb", 2, 2), (64, 64, "dev", "mono", 0, 2), (64, 64, "dev", "rgb", 1, 1)])
def test_pipeline_images_equal_one_shot_and_reference(ctxs, monkeypatch, batch, n, how, fmt, mirror, mode):
    from rebvo_b200 import capi, synth
    _ref()
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(n, seed=9)
    prm = capi.default_params(cam)
    run = run_image(prm, ts, fr, batch, how, fmt, mirror, mode)
    what = "batch %d %s %s mirror %d mode %d" % (batch, how, fmt, mirror, mode)
    assert_images_match(run, ctxs["euroc"], cam, mode, what)
    if batch == 7 and fmt == "rgb":   # eager launches give the same images
        monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
        eager = run_image(prm, ts, fr, batch, how, fmt, mirror, mode)
        monkeypatch.delenv("REBVO_B200_NO_GRAPH")
        for f, (a, b) in enumerate(zip(run["images"], eager["images"])):
            assert a[0].tobytes() == b[0].tobytes() and (a[1] is None) == (b[1] is None), f
            assert a[1] is None or a[1].tobytes() == b[1].tobytes(), f


def test_pipeline_images_other_camera(ctxs):
    """A frame that is not a multiple of the block (1241 x 376 with 10 x 10 blocks: remainder columns and rows)."""
    from rebvo_b200 import capi, synth
    cam = KITTI
    ts, fr = synth.Sequence(w=cam["w"], h=cam["h"], seed=5, zf=cam["zfx"]).frames(6)
    run = run_image(capi.default_params(cam), ts, fr, 3, mirror=2, mode=2)
    assert_images_match(run, ctxs["kitti"], cam, 2, "kitti")


# ---- 4. nothing else changes --------------------------------------------------------------------------------------------
def as_run(r):
    return pu.Run(r["nav"], None, r["mirrors"] or None, None, r["odometry"], r["launches"])


@pytest.mark.parametrize("mirror", [0, 1, 2])
def test_images_change_no_other_record(built, mirror):
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(16, seed=11)
    prm = capi.default_params(cam)
    on = run_image(prm, ts, fr, 8, mirror=mirror, mode=2, odometry=True)
    off = run_image(prm, ts, fr, 8, mirror=mirror, mode=0, odometry=True)
    pu.assert_runs_identical(as_run(on), as_run(off), "images on / off, mirror %d" % mirror)
    assert len(on["grids"]) == len(off["grids"]) == 16
    for f, ((ca, ma), (cb, mb)) in enumerate(zip(on["grids"], off["grids"])):
        assert ca.tobytes() == cb.tobytes() and np.float64(ma).tobytes() == np.float64(mb).tobytes(), "grid of frame %d" % f
    assert [a - b for a, b in zip(on["launches"], off["launches"])] == [8, 8]   # the image pass: one launch per frame


def test_images_off_restores_batches(built):
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(16, seed=12)
    prm = capi.default_params(cam)

    def run(toggle):
        pl = capi.Pipeline(prm, max_batch=4)
        navs, launches, grids = [], [], []
        try:
            pl.set_depth(params())
            for k, s in enumerate(range(0, 16, 4)):
                if toggle and k == 1:
                    pl.set_depth_image(2)
                if toggle and k == 2:
                    pl.set_depth_image(1)
                if toggle and k == 3:
                    pl.set_depth_image(0)
                l0 = pl.launches()
                navs.append(pl.push(fr[s:s + 4], ts[s:s + 4]))
                launches.append(pl.launches() - l0)
                grids += [pl.depth(i)[0].tobytes() for i in range(4)]
                if toggle and k in (1, 2):
                    rho, srho = pl.depth_image(3)
                    assert rho.shape == (cam["h"], cam["w"]) and (srho is None) == (k == 2)
                else:
                    with pytest.raises(capi.RbError):
                        pl.depth_image(0)
        finally:
            pl.close()
        return np.concatenate(navs), launches, grids

    nav0, l0, g0 = run(False)
    nav1, l1, g1 = run(True)
    assert pu.raw(nav0).tobytes() == pu.raw(nav1).tobytes() and g0 == g1
    assert l1 == [l0[0], l0[1] + 4, l0[2] + 4, l0[3]]


def test_set_before_or_after_depth(built):
    """The image mode may be set before the grid is switched on, and stays while the grid is switched off and on."""
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(6, seed=14)
    pl = capi.Pipeline(capi.default_params(cam), max_batch=2)
    try:
        pl.set_depth_image(1)
        pl.push(fr[0:2], ts[0:2])
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth_image(0)   # no grid, no image
        pl.set_depth(params())
        pl.push(fr[2:4], ts[2:4])
        first = pl.depth_image(1)[0].copy()
        assert np.isfinite(first).all() and first.shape == (cam["h"], cam["w"])
        pl.set_depth(params(16, 16))   # another grid: the image pass follows it
        pl.push(fr[4:6], ts[4:6])
        one = pl.depth_image(1)[0].copy()
        cells, _ = pl.depth(1)
        assert cells.shape == (30, 47)
        ctx = capi.Ctx(cam, 3.56359, 1.2599, kl_capacity=40000)
        try:
            assert one.tobytes() == ctx.depth_image(cells, params(16, 16), s_rho=False)[0].tobytes()
        finally:
            ctx.close()
    finally:
        pl.close()


# ---- 5. argument and state errors ---------------------------------------------------------------------------------------
def test_pipeline_arguments(built):
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(3, seed=15)
    pl = capi.Pipeline(capi.default_params(cam), max_batch=2)
    try:
        for bad in (-1, 3):
            with pytest.raises(capi.RbError, match="-2"):
                pl.set_depth_image(bad)
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth_image(0)   # nothing pushed
        pl.set_depth(params())
        pl.push(fr[0:2], ts[0:2])
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth_image(0)   # mode 0: the push made no image
        pl.set_depth_image(2)
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth_image(0)   # set after the push
        pl.push(fr[2:3], ts[2:3])
        pl.depth_image(0)
        for i in (-1, 1):
            with pytest.raises(capi.RbError, match="-2"):
                pl.depth_image(i)
        pl.set_depth(None)
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth_image(0)
    finally:
        pl.close()
    seq = pu.euroc_sequence()
    pl = capi.Pipeline(capi.default_params(cam), max_batch=2)
    try:
        pl.set_imu(synth.imu_samples(seq, 4))
        for mode in (0, 1, 2):
            with pytest.raises(capi.RbError, match="-2"):
                pl.set_depth_image(mode)
    finally:
        pl.close()


def test_smaller_plans_do_not_break_a_pipeline(built, monkeypatch):
    """The image kernel's shared-memory limit is one value per process and device: an image of a smaller grid made
    later (a stage call, another pipeline) must not break a pipeline whose grid needs more.  Eager launches check the
    limit at each launch."""
    from rebvo_b200 import capi, synth
    _ref()
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    cam = CAM_1280
    ts, fr = synth.Sequence(w=cam["w"], h=cam["h"], seed=5, zf=cam["zfx"]).frames(4)
    pl = capi.Pipeline(capi.default_params(cam), max_batch=2)
    other = capi.Pipeline(capi.default_params(synth.TUM), max_batch=2)
    ctx = capi.Ctx(synth.TUM, 3.56359, 1.2599, kl_capacity=40000)
    ctx_big = capi.Ctx(cam, 3.56359, 1.2599, kl_capacity=40000)
    try:
        pl.set_mirror(2)
        pl.set_depth(params())                      # 128 x 96 cells: 96 KB of shared memory per CTA
        pl.set_depth_image(2)
        rec = make_records([100, 300], [100, 200], 9000, 500, 9)
        small, _ = ctx.depth_fill_net(rec, params(16, 12))
        ctx.depth_image(small, params(16, 12))      # 40 x 40 cells: a smaller plan
        other.set_depth(params(16, 12))             # and another pipeline's
        other.set_depth_image(1)
        run = dict(nav=[], mirrors=[], grids=[], images=[])
        for s in range(0, 4, 2):
            nav = pl.push(fr[s:s + 2], ts[s:s + 2])
            run["nav"].append(nav)
            for i in range(len(nav)):
                run["grids"].append(pl.depth(i))
                run["mirrors"].append(pl.mirror(i).copy())
                r, sr = pl.depth_image(i)
                run["images"].append((r.copy(), sr.copy()))
            ctx.depth_image(small, params(16, 12))   # between pushes too
        run["nav"] = np.concatenate(run["nav"])
        assert_images_match(run, ctx_big, cam, 2, "after smaller plans")
    finally:
        ctx_big.close()
        ctx.close()
        other.close()
        pl.close()

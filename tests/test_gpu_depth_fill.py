"""The viewer's per-frame depth grid (depth_filler on each frame's net_keyline records, visualizer.cpp:436-440) on the device:
rb_depth_fill_net and the pipeline's per-frame grids, bit for bit against the unmodified reference depth_filler
(oracle/_ref/libref_depth.so, built by oracle/ref_depth.py)."""
import numpy as np
import pytest

import pipeline_util as pu

pytestmark = pytest.mark.gpu

KITTI = dict(w=1241, h=376, zfx=718.856, zfy=718.856, ppx=607.1928, ppy=185.2157)
CAM_1280 = dict(w=1280, h=960, zfx=900.0, zfy=900.0, ppx=640.5, ppy=479.5)
BLOCKS = [(10, 10), (8, 8), (16, 12), (7, 5), (2, 2)]
ITERS = [0, 1, 10, 30]
THRESH = [(1.0, 5), (0.2, 0), (1e9, 255)]


def _ref():
    from oracle import refapi, ref_depth
    if not ref_depth.available():
        if refapi.available():   # the reference was compiled here, so its depth_filler must have been too
            pytest.fail("oracle/_ref/libref_mtrack.so was built but oracle/_ref/libref_depth.so was not")
        pytest.skip("oracle/_ref/libref_depth.so not built")
    return ref_depth


def _cams():
    from rebvo_b200 import synth
    return {"euroc": synth.EUROC, "tum": synth.TUM, "kitti": KITTI, "1280": CAM_1280}


def fields(rec):
    r = rec.astype(np.uint32)
    return dict(qx=r[:, 0] | (r[:, 1] << 8), qy=r[:, 2] | (r[:, 3] << 8), rho=r[:, 4] | (r[:, 5] << 8),
                s_rho=r[:, 6] | (r[:, 7] << 8), m_num=r[:, 12])


def make_records(qx, qy, rho, s_rho, m_num):
    qx, qy, rho, s_rho, m_num = np.broadcast_arrays(*(np.asarray(v, np.int64) for v in (qx, qy, rho, s_rho, m_num)))
    rec = np.zeros((len(qx), 15), np.uint8)
    for col, v in ((0, qx), (2, qy), (4, rho), (6, s_rho)):
        rec[:, col], rec[:, col + 1] = v & 0xff, (v >> 8) & 0xff
    rec[:, 8:12] = 0xff   # n_kl = -1
    rec[:, 12] = m_num
    rec[:, 13:15] = 127
    return rec


def in_grid(rec, cam, bw, bh):
    """The records whose cell index (GetIndex of the float quotients) lies inside the grid: the others write out of bounds in
    the reference, so they are left out of every comparison."""
    f = fields(rec)
    gw, gh = cam["w"] // bw, cam["h"] // bh
    x = (f["qx"].astype(np.float32) / np.float32(bw)).astype(np.uint32)
    y = (f["qy"].astype(np.float32) / np.float32(bh)).astype(np.uint32)
    return rec[y * np.uint32(gw) + x < gw * gh]


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


def assert_grid_equal(cells, min_dist, ref, what):
    assert cells.shape == ref["rho"].shape, (what, cells.shape, ref["rho"].shape)
    for k in ("rho", "s_rho", "dist"):
        bad = np.argwhere(bits(cells[k]) != bits(ref[k]))
        assert len(bad) == 0, "%s: %s differs in %d cells, first %s: %r vs %r" % (
            what, k, len(bad), bad[0], cells[k][tuple(bad[0])], ref[k][tuple(bad[0])])
    assert np.array_equal(cells["fixed"], ref["fixed"]), what
    assert bits(min_dist) == bits(ref["min_dist"]), (what, min_dist, ref["min_dist"])


def params(bw=10, bh=10, thr=1.0, mnum=5, iters=10):
    from rebvo_b200 import capi
    return capi.depth_params(bw, bh, thr, mnum, iters)


_records = {}


def tracked_records(name):
    """net_keyline records of the two newest maps of a short pipeline run of the synthetic stream with this camera, each
    packed at its frame's K."""
    if name not in _records:
        from rebvo_b200 import capi, synth
        cam = _cams()[name]
        ts, fr = synth.Sequence(w=cam["w"], h=cam["h"], seed=5, zf=cam["zfx"]).frames(10)
        pl = capi.Pipeline(capi.default_params(cam), max_batch=10)
        try:
            nav = pl.push(fr, ts)
            _records[name] = [pl.map(a).pack_net(float(nav[-1 - a]["K"])) for a in (0, 1)]
        finally:
            pl.close()
        assert len(_records[name][0]) > 3000
    return _records[name]


@pytest.fixture(scope="module")
def ctxs(built):
    from rebvo_b200 import capi
    out = {n: capi.Ctx(c, 3.56359, 1.2599, kl_capacity=40000) for n, c in _cams().items()}
    yield out
    for c in out.values():
        c.close()


# ---- 1. stage parity on tracked maps ------------------------------------------------------------------------------------
@pytest.mark.parametrize("block", BLOCKS, ids=["%dx%d" % b for b in BLOCKS])
@pytest.mark.parametrize("cam", ["euroc", "tum", "kitti", "1280"])
def test_stage_parity_tracked_maps(ctxs, cam, block):
    ref = _ref()
    c = _cams()[cam]
    bw, bh = block
    for age, rec in enumerate(tracked_records(cam)):
        rec = in_grid(rec, c, bw, bh)
        for iters in ITERS:
            for thr, mnum in THRESH:
                if block == (2, 2) and iters not in (0, 10):
                    continue   # (the 2x2 grid is the slow single-CTA global-memory case: two sweep counts suffice)
                cells, md = ctxs[cam].depth_fill_net(rec, params(bw, bh, thr, mnum, iters))
                want = ref.depth_fill_net(c, rec, bw, bh, thr, mnum, iters)
                assert_grid_equal(cells, md, want, "%s %dx%d map %d iter %d thr (%g, %d)" % (cam, bw, bh, age, iters, thr, mnum))
        # every record through both gates: a grid with fused and filled cells
        cells, md = ctxs[cam].depth_fill_net(rec, params(bw, bh, 1e9, 0, 10))
        assert_grid_equal(cells, md, ref.depth_fill_net(c, rec, bw, bh, 1e9, 0, 10), "%s %dx%d map %d, no gates" % (cam, bw, bh, age))
        assert 0 < cells["fixed"].sum() < cells["fixed"].size


# ---- 2. crafted records -------------------------------------------------------------------------------------------------
def _check(ctx, cam, rec, p, what):
    ref = _ref()
    cells, md = ctx.depth_fill_net(rec, p)
    want = ref.depth_fill_net(cam, rec, p.block_w, p.block_h, p.thresh_rel_rho, p.thresh_match_num, p.iter_num)
    assert_grid_equal(cells, md, want, what)
    return cells, md


def test_crafted_one_cell_order(ctxs):
    from rebvo_b200 import synth
    cam, ctx = synth.EUROC, ctxs["euroc"]
    rng = np.random.default_rng(3)
    n = 60
    rho = rng.integers(500, 60000, n)
    one = make_records(rng.integers(300, 310, n), rng.integers(200, 210, n), rho, rng.integers(50, 3000, n), 9)
    bg = make_records(rng.integers(0, 740, 400), rng.integers(0, 470, 400), rng.integers(500, 60000, 400),
                      rng.integers(50, 3000, 400), 9)
    rec = np.concatenate([bg[:200], one, bg[200:]])
    a, _ = _check(ctx, cam, rec, params(), "60 records in one cell")
    # the fusion is order sensitive in the last bits: the reversed records give another grid, equal to the reference's too
    rev = np.concatenate([bg[:200], one[::-1], bg[200:]])
    b, _ = _check(ctx, cam, rev, params(), "60 records in one cell, reversed")
    assert a["fixed"][20, 30] == 1


def test_crafted_gates(ctxs):
    from rebvo_b200 import synth
    cam, ctx = synth.EUROC, ctxs["euroc"]
    # s_rho / rho exactly at thresh_rel_rho (kept: the gate is >), just above (skipped); m_num at the threshold (kept), below
    rec = make_records([15, 35, 55, 75, 95, 115, 135, 155], 45, [10000, 10000, 5000, 5000, 20000, 20000, 4000, 4000],
                       [10000, 10001, 1000, 1001, 4000, 4001, 800, 801], [5, 5, 5, 4, 5, 4, 6, 3])
    for thr, mnum in ((1.0, 5), (0.2, 5), (0.2, 0), (1.0, 6)):
        cells, _ = _check(ctx, cam, rec, params(thr=thr, mnum=mnum), "gates (%g, %d)" % (thr, mnum))
        assert cells["fixed"].sum() > 0 or mnum == 6


def test_crafted_remainder_column(ctxs):
    from rebvo_b200 import synth
    cam, ctx = synth.EUROC, ctxs["euroc"]
    # qx >= 750 at 752 px with 10-px blocks: qx / 10 == gw, the first cell of the next row
    rec = make_records([750, 751, 751, 5, 749], [33, 100, 250, 101, 330], [3000, 7000, 12000, 9000, 15000], 500, 9)
    cells, _ = _check(ctx, cam, rec, params(), "remainder column")
    assert cells["fixed"][4, 0] == 1 and cells["fixed"][11, 0] == 1 and cells["fixed"][26, 0] == 1
    # 7x5 blocks at 752x480: columns 749..751 wrap
    _check(ctx, cam, make_records([749, 750, 751], [100, 200, 300], 8000, 400, 9), params(7, 5), "remainder column 7x5")


def test_crafted_empty_and_all_fixed(ctxs):
    from rebvo_b200 import synth
    cam, ctx = synth.EUROC, ctxs["euroc"]
    for iters in (0, 10):
        cells, md = _check(ctx, cam, np.zeros((0, 15), np.uint8), params(iters=iters), "kn = 0")
        assert cells["fixed"].sum() == 0 and np.all(cells["rho"] == 1.0) and np.all(cells["s_rho"] == 40.0)
    ys, xs = np.mgrid[0:48, 0:75]
    rng = np.random.default_rng(4)
    rec = make_records(xs.ravel() * 10 + 3, ys.ravel() * 10 + 6, rng.integers(1000, 50000, xs.size), 700, 9)
    cells, _ = _check(ctx, cam, rec, params(), "every cell fixed")
    assert cells["fixed"].all()


def test_crafted_out_of_grid_rows_dropped(ctxs):
    from rebvo_b200 import synth
    cam, ctx = synth.EUROC, ctxs["euroc"]
    rng = np.random.default_rng(6)
    base = make_records(rng.integers(0, 745, 300), rng.integers(0, 470, 300), rng.integers(1000, 50000, 300), 700, 9)
    # 7x7 blocks at 480 px: gh = 68, rows 476..479 give qy / 7 == gh; qy = 600 lies past the frame.  Undefined behaviour in
    # the reference (an out-of-bounds write), dropped on the device: they change nothing.
    oob = make_records([10, 300, 700, 100], [476, 479, 478, 600], 20000, 300, 9)
    p = params(7, 7)
    assert len(in_grid(oob, cam, 7, 7)) == 0 and len(in_grid(base, cam, 7, 7)) == len(base)
    want, wmd = _check(ctx, cam, base, p, "in-grid records")
    mixed = np.concatenate([base[:150], oob, base[150:]])
    got, gmd = ctx.depth_fill_net(mixed, p)
    for k in ("rho", "s_rho", "dist"):
        assert np.array_equal(bits(got[k]), bits(want[k])), k
    assert np.array_equal(got["fixed"], want["fixed"]) and bits(gmd) == bits(wmd)


def test_invalid_arguments(ctxs):
    from rebvo_b200 import capi, synth
    ctx = ctxs["euroc"]
    rec = np.zeros((1, 15), np.uint8)
    for bad in (params(0, 10), params(10, 0), params(753, 10), params(10, 481), params(iters=-1)):
        with pytest.raises(capi.RbError, match="-2"):
            ctx.depth_fill_net(rec, bad)
    cam = synth.EUROC
    pl = capi.Pipeline(capi.default_params(cam), max_batch=2)
    try:
        for bad in (params(0, 10), params(10, 481), params(iters=-1)):
            with pytest.raises(capi.RbError, match="-2"):
                pl.set_depth(bad)
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth(0)   # off
        pl.set_depth(params())
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth(0)   # nothing pushed yet
    finally:
        pl.close()
    seq = pu.euroc_sequence()
    pl = capi.Pipeline(capi.default_params(cam), max_batch=2)
    try:
        pl.set_imu(synth.imu_samples(seq, 4))
        with pytest.raises(capi.RbError, match="-2"):
            pl.set_depth(params())
    finally:
        pl.close()


# ---- 3. the pipeline's per-frame grids ----------------------------------------------------------------------------------
def run_depth(prm, ts, frames, batch, how="host", fmt="rgb", mirror=2, depth=True, odometry=False):
    """Pushes of `batch` frames with depth (viewer parameters) and the mirror on; per frame: nav, mirror records,
    (cells, min_dist); plus the launches of each push."""
    from rebvo_b200 import capi
    pl = capi.Pipeline(prm, max_batch=batch)
    navs, mirrors, grids, launches, odo = [], [], [], [], []
    try:
        if mirror:
            pl.set_mirror(mirror)
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
            if odometry:
                odo.append(pl.odometry())
    finally:
        pl.close()
    return dict(nav=np.concatenate(navs), mirrors=mirrors, grids=grids, launches=launches,
                odometry=np.concatenate(odo) if odo else None)


def assert_grids_match_reference(run, cam, what):
    ref = _ref()
    assert len(run["grids"]) == len(run["mirrors"]) == len(run["nav"])
    for f, (rec, (cells, md)) in enumerate(zip(run["mirrors"], run["grids"])):
        assert len(rec) == run["nav"][f]["kn"]
        rec = in_grid(rec, cam, 10, 10)
        assert_grid_equal(cells, md, ref.depth_fill_net(cam, rec, 10, 10, 1.0, 5, 10), "%s frame %d" % (what, f))


def assert_same_grids(a, b, what):
    assert len(a) == len(b)
    for f, ((ca, ma), (cb, mb)) in enumerate(zip(a, b)):
        assert ca.tobytes() == cb.tobytes() and bits(ma) == bits(mb), "%s: frame %d" % (what, f)


@pytest.mark.parametrize("batch,n,how,fmt", [(1, 4, "host", "rgb"), (7, 14, "dev", "rgb"), (7, 14, "host", "mono"),
                                             (64, 64, "host", "rgb"), (64, 64, "dev", "mono")])
def test_pipeline_grids_equal_reference(built, monkeypatch, batch, n, how, fmt):
    from rebvo_b200 import capi, synth
    _ref()
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(n, seed=9)
    prm = capi.default_params(cam)
    run = run_depth(prm, ts, fr, batch, how, fmt)
    assert_grids_match_reference(run, cam, "batch %d %s %s" % (batch, how, fmt))
    if batch != 64 or fmt == "rgb":
        monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
        eager = run_depth(prm, ts, fr, batch, how, fmt)
        monkeypatch.delenv("REBVO_B200_NO_GRAPH")
        assert_same_grids(run["grids"], eager["grids"], "graph replay vs eager")
        assert pu.raw(run["nav"]).tobytes() == pu.raw(eager["nav"]).tobytes()


# ---- 4. nothing else changes ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mirror", [0, 1, 2])
def test_depth_changes_no_other_record(built, mirror):
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(16, seed=11)
    prm = capi.default_params(cam)
    prm.kl_capacity = 40000
    on = run_depth(prm, ts, fr, 8, mirror=mirror, depth=True, odometry=True)
    off = run_depth(prm, ts, fr, 8, mirror=mirror, depth=False, odometry=True)
    assert pu.raw(on["nav"]).tobytes() == pu.raw(off["nav"]).tobytes()
    assert pu.raw(on["odometry"]).tobytes() == pu.raw(off["odometry"]).tobytes()
    assert len(on["mirrors"]) == len(off["mirrors"])
    for f, (a, b) in enumerate(zip(on["mirrors"], off["mirrors"])):   # (mode 1: field by field, the padding is not written)
        ok = np.array_equal(a, b) if mirror == 2 else pu.keylines_equal(a, b)
        assert ok, "mirror %d frame %d" % (mirror, f)
    # the pack (when the mirror's records cannot be read) and the fill: two launches per frame, one with mirror mode 2
    per_frame = 1 if mirror == 2 else 2
    assert [a - b for a, b in zip(on["launches"], off["launches"])] == [per_frame * 8, per_frame * 8]
    if mirror == 0:   # the grids do not depend on where the records were packed
        with_mirror = run_depth(prm, ts, fr, 8, mirror=2, depth=True)
        assert_same_grids(on["grids"], with_mirror["grids"], "own pack vs mirror records")


def test_depth_off_restores_batches(built):
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(12, seed=12)
    prm = capi.default_params(cam)

    def run(toggle):
        pl = capi.Pipeline(prm, max_batch=4)
        navs, launches = [], []
        try:
            for k, s in enumerate(range(0, 12, 4)):
                if toggle and k == 1:
                    pl.set_depth(params())
                if toggle and k == 2:
                    pl.set_depth(None)
                l0 = pl.launches()
                navs.append(pl.push(fr[s:s + 4], ts[s:s + 4]))
                launches.append(pl.launches() - l0)
            with pytest.raises(capi.RbError):
                pl.depth(0)
        finally:
            pl.close()
        return np.concatenate(navs), launches

    nav0, l0 = run(False)
    nav1, l1 = run(True)
    assert pu.raw(nav0).tobytes() == pu.raw(nav1).tobytes()
    assert l1[0] == l0[0] and l1[2] == l0[2] and l1[1] == l0[1] + 2 * 4


def test_smaller_plans_do_not_break_a_pipeline(built, monkeypatch):
    """The fill kernel's shared-memory limit is one value per process and device: fills planned later with smaller grids (a
    stage call on another camera, another pipeline's set_depth) must not break a pipeline whose grid needs more.  Eager
    launches (every push with REBVO_B200_NO_GRAPH=1) check the limit at each launch."""
    from rebvo_b200 import capi, synth
    _ref()
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    cam = synth.EUROC
    ts, fr = pu.euroc_stream(8, seed=13)
    pl = capi.Pipeline(capi.default_params(cam), max_batch=4)
    other = capi.Pipeline(capi.default_params(synth.TUM), max_batch=2)
    ctx = capi.Ctx(synth.TUM, 3.56359, 1.2599, kl_capacity=40000)
    try:
        pl.set_mirror(2)
        pl.set_depth(params())                      # 75x48 cells: ~64 KB of shared memory
        rec = make_records([100, 300], [100, 200], 9000, 500, 9)
        ctx.depth_fill_net(rec, params(16, 12))     # 40x40 cells: a smaller plan
        other.set_depth(params(16, 12))             # and another pipeline's
        grids, mirrors, navs = [], [], []
        for s in range(0, 8, 4):
            nav = pl.push(fr[s:s + 4], ts[s:s + 4])
            navs.append(nav)
            for i in range(len(nav)):
                grids.append(pl.depth(i))
                mirrors.append(pl.mirror(i).copy())
            ctx.depth_fill_net(rec, params(8, 8))   # between pushes too
        assert_grids_match_reference(dict(nav=np.concatenate(navs), mirrors=mirrors, grids=grids), cam, "after smaller plans")
    finally:
        ctx.close()
        other.close()
        pl.close()


def test_long_cell_lists_and_many_sweeps(ctxs):
    """Block sizes near the frame's put most records into one cell (the long-list sort), and many sweeps run the wavefront
    far past its first sweep."""
    ref = _ref()
    from rebvo_b200 import synth
    cam, ctx = synth.EUROC, ctxs["euroc"]
    rec = tracked_records("euroc")[0]
    for bw, bh, iters in ((752, 480, 3), (376, 240, 10), (300, 200, 200), (10, 10, 150)):
        r = in_grid(rec, cam, bw, bh)
        cells, md = ctx.depth_fill_net(r, params(bw, bh, 1e9, 0, iters))
        assert_grid_equal(cells, md, ref.depth_fill_net(cam, r, bw, bh, 1e9, 0, iters), "%dx%d, %d sweeps" % (bw, bh, iters))

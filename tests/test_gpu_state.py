"""Session checkpoints (rb_pipeline_save_state / rb_pipeline_load_state): a session saved at any frame and loaded into
another pipeline -- new object, other max_batch, other push sizes -- continues with the bytes of the uninterrupted run:
nav and odometry records, mirrors, depth grids and images, the trajectory text.  In every input layout, in IMU dataset
and live mode, rewound in place, on four pipelines at once, and after every kind of refused blob, which leaves the
target as it was."""
import hashlib
import threading

import numpy as np
import pytest

from pipeline_util import EUROC_KC, euroc_sequence, push, raw

pytestmark = pytest.mark.gpu
NF = 32
CUTS = (0, 1, 2, 3, 20)     # nothing pushed yet, "ring only initialised", each ring phase, and a converged map
RB_ERR_ARG = -2


@pytest.fixture(scope="module")
def stream(built):
    from rebvo_b200 import capi, synth
    seq = euroc_sequence()
    ts, fr = seq.frames(NF)
    return capi.default_params(synth.EUROC), ts, fr, synth.imu_samples(seq, NF)


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).view(np.uint8).tobytes()).hexdigest()


def _pipeline(params, max_batch, mirror):
    from rebvo_b200 import capi
    pl = capi.Pipeline(params, max_batch=max_batch)
    pl.set_undistort(EUROC_KC)
    pl.set_mirror(mirror)
    pl._mirror_mode = mirror
    pl.set_depth(capi.depth_params())
    pl.set_depth_image(2)
    pl.set_odometry(True)
    return pl


def _push(pl, layout, frames, ts):
    if layout == "rgb":
        return pl.push(frames, ts)
    if layout == "mono":
        return pl.push_mono(np.ascontiguousarray(frames[..., 0]), ts)
    if layout == "dev":
        return push(pl, frames, ts, "dev")
    import torch   # strided device frames: rows 48 bytes longer than the frame's
    n, h, w, _ = frames.shape
    buf = torch.zeros((n, h, w + 16, 3), dtype=torch.uint8, device="cuda")
    buf[:, :, :w] = torch.from_numpy(frames).cuda()
    return pl.push_frames(buf[:, :, :w], ts)


def _outputs(pl, nav):
    """Per frame of the last push: digests of its nav and odometry records, mirror, depth grid and depth image."""
    odom = pl.odometry()
    out = []
    for i in range(len(nav)):
        cells, md = pl.depth(i)
        rho, s_rho = pl.depth_image(i)
        out.append({"nav": _digest(nav[i:i + 1]), "odometry": _digest(odom[i:i + 1]), "mirror": _digest(pl.mirror(i)),
                    "depth": _digest(cells) + repr(md), "image": _digest(rho) + _digest(s_rho)})
    return out


def _run(pl, layout, frames, ts, start, end, sizes):
    """Frames [start, end) in pushes of the given sizes, taken in turn: (nav records, per-frame outputs)."""
    navs, outs, s, k = [], [], start, 0
    while s < end:
        e = min(end, s + sizes[k % len(sizes)])
        nav = _push(pl, layout, frames[s:e], ts[s:e])
        navs.append(nav)
        outs += _outputs(pl, nav)
        s, k = e, k + 1
    from rebvo_b200 import capi
    return (np.concatenate(navs) if navs else np.zeros(0, capi.NAV)), outs


def _assert_same(want, got, first, what):
    from rebvo_b200 import capi
    (nav_w, out_w), (nav_g, out_g) = want, got
    assert len(nav_w) == len(nav_g), what
    bad = np.nonzero((raw(nav_w) != raw(nav_g)).reshape(len(nav_w), -1).any(1))[0]
    assert not len(bad), "%s: nav record of frame %d differs" % (what, first + bad[0])
    for i, (a, b) in enumerate(zip(out_w, out_g)):
        for k in a:
            assert a[k] == b[k], "%s: %s of frame %d differs" % (what, k, first + i)
    assert capi.format_trajectory(nav_w) == capi.format_trajectory(nav_g), what


# layout, mirror mode, and the push sizes of the uninterrupted run and of the continuations
LAYOUTS = [("rgb", 1), ("mono", 2), ("dev", 2), ("strided", 1)]


@pytest.mark.parametrize("layout,mirror", LAYOUTS)
def test_continuation_is_the_uninterrupted_run(stream, layout, mirror):
    from rebvo_b200 import capi
    params, ts, fr, _ = stream
    base = _pipeline(params, 8, mirror)
    try:
        full = _run(base, layout, fr, ts, 0, NF, [8])
    finally:
        base.close()
    # the source pushes up to each cut and saves there; a save changes none of its later outputs
    src = _pipeline(params, 20, mirror)
    blobs, navs, outs, at = {}, [], [], 0
    try:
        for cut in CUTS + (NF,):
            if cut > at:
                nav, out = _run(src, layout, fr, ts, at, cut, [cut - at])
                navs.append(nav)
                outs += out
                at = cut
            if cut in CUTS:
                blobs[cut] = src.save_state()
    finally:
        src.close()
    _assert_same(full, (np.concatenate(navs), outs), 0, "%s: source that saved at %s" % (layout, CUTS))
    for cut, blob in blobs.items():
        info = capi.state_info(blob)
        assert info["n_pushed"] == cut and info["mode"] == capi.STATE_VISION
        assert info["kn"] == (full[0][cut - 1]["kn"] if cut else 0)
        dst = _pipeline(params, 5, mirror)
        try:
            dst.load_state(blob)
            got = _run(dst, layout, fr, ts, cut, NF, [5, 3])
        finally:
            dst.close()
        _assert_same((full[0][cut:], full[1][cut:]), got, cut, "%s: cut at frame %d" % (layout, cut))


def test_round_trip_and_fork(stream):
    from rebvo_b200 import capi
    params, ts, fr, _ = stream
    a = capi.Pipeline(params, max_batch=8)
    try:
        a.set_undistort(EUROC_KC)
        for s in range(0, 20, 8):
            a.push(fr[s:min(20, s + 8)], ts[s:min(20, s + 8)])
        blob = a.save_state()
        assert a.save_state() == blob
    finally:
        a.close()
    info = capi.state_info(blob)
    assert info["bytes"] == len(blob) and info["n_pushed"] == 20 and info["w"] == params.cam.w
    print("blob: %d bytes, %d keylines, %.1f bytes per keyline" % (len(blob), info["kn"], len(blob) / max(info["kn"], 1)))
    assert len(blob) <= 128 + 1024 + 120 * info["kn"]
    # other tracker settings: accepted, and the blob round-trips
    for p2 in (params, _forked_params(params)):
        b = capi.Pipeline(p2, max_batch=3)
        try:
            b.load_state(blob)
            assert b.save_state() == blob
            b.push(fr[20:23], ts[20:23])
        finally:
            b.close()


def _forked_params(params):
    import copy
    p = copy.copy(params)
    p.TrackerIterNum = params.TrackerIterNum + 3
    p.MatchThreshold = params.MatchThreshold + 5
    p.DetectorThresh = params.DetectorThresh * 1.5
    return p


def test_rewind_in_place(stream):
    from rebvo_b200 import capi
    params, ts, fr, _ = stream
    pl = _pipeline(params, 8, 2)
    try:
        _run(pl, "rgb", fr, ts, 0, 20, [8])
        blob = pl.save_state()
        first = _run(pl, "rgb", fr, ts, 20, NF, [8])
        pl.load_state(blob)
        with pytest.raises(capi.RbError):   # the outputs of the last push are gone
            pl.mirror(0)
        with pytest.raises(capi.RbError):
            pl.odometry()
        second = _run(pl, "rgb", fr, ts, 20, NF, [8])
    finally:
        pl.close()
    _assert_same(first, second, 20, "rewound to frame 20")


def test_stage_level_view_after_load(stream):
    from rebvo_b200 import capi
    params, ts, fr, _ = stream
    a = capi.Pipeline(params, max_batch=8)
    b = capi.Pipeline(params, max_batch=8)
    try:
        for s in range(0, 21, 7):
            a.push(fr[s:s + 7], ts[s:s + 7])
        m = a.map(0)
        kl, mask = m.keylines(), m.mask()
        b.push(fr[:2], ts[:2])   # stale maps in every slot the load does not write
        b.push(fr[2:4], ts[2:4])
        b.load_state(a.save_state())
        assert b.map(1) is None
        m2 = b.map(0)
        assert m2.knum() == len(kl)
        assert np.ascontiguousarray(m2.keylines()).tobytes() == np.ascontiguousarray(kl).tobytes()
        assert np.array_equal(m2.mask(), mask)
        b.push(fr[21:22], ts[21:22])
        assert b.map(1) is not None
    finally:
        a.close()
        b.close()


def _imu_params():
    from rebvo_b200 import capi
    return capi.default_imu_params(InitBias=1, InitBiasFrameNum=5)


@pytest.mark.parametrize("cut", [3, 14])   # inside the InitBiasFrameNum window; after the filter starts (frame > 9)
def test_imu_dataset_continuation(stream, cut):
    from rebvo_b200 import capi
    params, ts, fr, imu = stream

    def make():
        pl = capi.Pipeline(params, max_batch=8)
        pl.set_imu(imu, _imu_params())
        pl.set_odometry(True)
        return pl
    a = make()
    try:
        navs, odos = [], []
        for s in range(0, NF, 8):
            navs.append(a.push(fr[s:s + 8], ts[s:s + 8]))
            odos.append(a.odometry())
        nav, odo = np.concatenate(navs), np.concatenate(odos)
    finally:
        a.close()
    b, c = make(), make()
    try:
        for s in range(0, cut, 8):
            b.push(fr[s:min(cut, s + 8)], ts[s:min(cut, s + 8)])
        blob = b.save_state()
        assert capi.state_info(blob)["mode"] == capi.STATE_IMU_DATASET
        c.load_state(blob)
        for s in range(cut, NF, 5):
            e = min(NF, s + 5)
            assert raw(c.push(fr[s:e], ts[s:e])).tobytes() == raw(nav[s:e]).tobytes(), "frames %d..%d" % (s, e)
            assert raw(c.odometry()).tobytes() == raw(odo[s:e]).tobytes(), "odometry %d..%d" % (s, e)
    finally:
        b.close()
        c.close()


def test_imu_live_carries_unreleased_samples(stream):
    from rebvo_b200 import capi
    params, ts, fr, imu = stream
    tsample = (imu[-1, 0] - imu[0, 0]) / (len(imu) - 1)

    def make():
        pl = capi.Pipeline(params, max_batch=8)
        pl.set_imu_live(_imu_params(), sample_time=tsample, buffer_size=len(imu) + 1)
        pl.set_odometry(True)
        return pl
    a = make()
    try:
        a.push_imu(imu)
        nav = np.concatenate([a.push(fr[s:s + 8], ts[s:s + 8]) for s in range(0, NF, 8)])
    finally:
        a.close()
    for cut in (4, 14):
        # the source has the samples up to three frames past the cut: those after frame cut-1 are not released
        k = int(np.searchsorted(imu[:, 0], ts[min(NF - 1, cut + 3)], side="right")) + 1
        b, c = make(), make()
        try:
            b.push_imu(imu[:k])
            for s in range(0, cut, 8):
                b.push(fr[s:min(cut, s + 8)], ts[s:min(cut, s + 8)])
            blob = b.save_state()
            assert capi.state_info(blob)["mode"] == capi.STATE_IMU_LIVE
            small = capi.Pipeline(params, max_batch=8)
            try:   # a ring too small for the pending samples refuses the blob
                small.set_imu_live(_imu_params(), sample_time=tsample, buffer_size=2)
                with pytest.raises(capi.RbError):
                    small.load_state(blob)
            finally:
                small.close()
            c.load_state(blob)
            c.push_imu(imu[k:])   # only what the source had not received
            got = np.concatenate([c.push(fr[s:s + 6], ts[s:s + 6]) for s in range(cut, NF, 6)])
            assert raw(got).tobytes() == raw(nav[cut:]).tobytes(), "live cut at %d" % cut
        finally:
            b.close()
            c.close()


def _checkpoint_at_20(params, ts, fr):
    """(blob saved at frame 20, nav records of frames 20.. of the source that went on)"""
    from rebvo_b200 import capi
    a = capi.Pipeline(params, max_batch=10)
    try:
        a.push(fr[:10], ts[:10])
        a.push(fr[10:20], ts[10:20])
        blob = a.save_state()
        return blob, np.concatenate([a.push(fr[s:s + 6], ts[s:s + 6]) for s in range(20, NF, 6)])
    finally:
        a.close()


def _continue_on(params, ts, fr, blob, device=0):
    from rebvo_b200 import capi
    pl = capi.Pipeline(params, max_batch=6, device=device)
    try:
        pl.load_state(blob)
        return np.concatenate([pl.push(fr[s:s + 6], ts[s:s + 6]) for s in range(20, NF, 6)])
    finally:
        pl.close()


def test_independent_pipelines(stream):
    params, ts, fr, _ = stream
    blob, want = _checkpoint_at_20(params, ts, fr)
    res, errs = [None] * 4, []

    def work(k):
        try:
            res[k] = _continue_on(params, ts, fr, blob)
        except Exception as e:   # reported below
            errs.append(e)
    th = [threading.Thread(target=work, args=(k,)) for k in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for k in range(4):
        assert raw(res[k]).tobytes() == raw(want).tobytes(), "pipeline %d" % k


def test_load_on_another_gpu(stream):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    params, ts, fr, _ = stream
    blob, want = _checkpoint_at_20(params, ts, fr)
    assert raw(_continue_on(params, ts, fr, blob, device=1)).tobytes() == raw(want).tobytes()


def test_refusals_leave_the_target_untouched(stream):
    import copy
    import ctypes as C

    from rebvo_b200 import capi
    params, ts, fr, imu = stream
    src = capi.Pipeline(params, max_batch=8)
    t, twin = capi.Pipeline(params, max_batch=8), capi.Pipeline(params, max_batch=8)
    others = []
    try:
        src.push(fr[:8], ts[:8])
        src.push(fr[8:12], ts[8:12])
        good = src.save_state()
        for pl in (t, twin):
            pl.push(fr[:6], ts[:6])
        at = 6

        def blob_of(imu_mode=False, **over):
            p = copy.copy(params)
            cam = copy.copy(params.cam)
            for k, v in over.items():
                if hasattr(cam, k):
                    setattr(cam, k, v)
                else:
                    setattr(p, k, v)
            p.cam = cam
            o = capi.Pipeline(p, max_batch=2)
            others.append(o)
            if imu_mode:
                o.set_imu(imu, _imu_params())
            return o
        bad = {}
        # another camera, Sigma0, KSigma, kl_capacity: blobs of pipelines that never pushed (their geometry is in the header)
        for name, over in (("w", dict(w=params.cam.w - 32)), ("ppx", dict(ppx=params.cam.ppx + 1)),
                           ("zfx", dict(zfx=params.cam.zfx * 1.01)), ("Sigma0", dict(Sigma0=params.Sigma0 * 1.1)),
                           ("KSigma", dict(KSigma=params.KSigma * 1.1)),
                           ("kl_capacity", dict(kl_capacity=(params.kl_capacity or 50000) - 1000))):
            bad[name] = blob_of(**over).save_state()
        bad["mode"] = blob_of(imu_mode=True).save_state()
        bad["flipped byte"] = bytearray(good)
        bad["flipped byte"][len(good) // 2] ^= 0x10
        bad["truncated"] = good[:-8]
        bad["header only"] = good[:128]
        v = bytearray(good)
        v[8] += 1   # version
        bad["version"] = v
        for name, blob in bad.items():
            l0 = t.launches()
            with pytest.raises(capi.RbError) as e:
                t.load_state(bytes(blob))
            assert "error -2" in str(e.value), (name, str(e.value))
            assert t.launches() == l0, name
            a, b = t.push(fr[at:at + 1], ts[at:at + 1]), twin.push(fr[at:at + 1], ts[at:at + 1])
            assert raw(a).tobytes() == raw(b).tobytes(), "after the refused blob: %s" % name
            at += 1
        # IMU samples other than the target's
        i1, i2 = capi.Pipeline(params, max_batch=4), capi.Pipeline(params, max_batch=4)
        others += [i1, i2]
        i1.set_imu(imu, _imu_params())
        i2.set_imu(imu[:-1], _imu_params())
        i1.push(fr[:3], ts[:3])
        with pytest.raises(capi.RbError):
            i2.load_state(i1.save_state())
        # cap too small: RB_ERR_ARG with the size needed
        need = C.c_size_t(0)
        buf = C.create_string_buffer(64)
        r = t.L.rb_pipeline_save_state(t.h_, buf, C.c_size_t(64), C.byref(need))
        assert r == RB_ERR_ARG and need.value == len(t.save_state())
        # a save or a load changes no later push's launch count
        d0 = [twin.launches()]
        twin.push(fr[at:at + 2], ts[at:at + 2])
        d0 = twin.launches() - d0[0]
        t.load_state(t.save_state())
        l0 = t.launches()
        a = t.push(fr[at:at + 2], ts[at:at + 2])
        assert t.launches() - l0 == d0
    finally:
        for pl in [src, t, twin] + others:
            pl.close()

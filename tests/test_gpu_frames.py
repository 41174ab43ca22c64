"""Strided frame input (rb_pipeline_push_frames / rb_pipeline_push_frames_dev, Pipeline.push_frames): frames with a row step,
one buffer per frame, from host or device memory.  Every case compares a strided push byte for byte with a packed push of
the same pixels on a twin pipeline: raw nav and odometry records, the keyline mirror (modes 1 and 2), the depth grid and
image of every frame, and the keylines and mask of the two newest maps after the last push."""

import numpy as np
import pytest

import pipeline_util as pu

pytestmark = pytest.mark.gpu
RB_ERR_ARG, RB_ERR_STATE = -2, -4
KC = (-0.12, 0.03, 0.0, 1e-4, 2e-5)   # a mild rad-tan model for the KITTI sizes


def _cams():
    from rebvo_b200 import synth

    def kitti(w, h):
        return dict(w=w, h=h, zfx=718.856, zfy=718.856, ppx=w / 2.0 - 13.3, ppy=h / 2.0 - 2.8)
    return {"euroc": synth.EUROC, "1241": kitti(1241, 376), "1226": kitti(1226, 370)}


_streams = {}


def stream(cam, n):
    """(ts, RGB frames) of a seeded sequence on camera `cam`, the first n frames (rendered once per module)."""
    from rebvo_b200 import synth
    if cam not in _streams or len(_streams[cam][0]) < n:
        c = _cams()[cam]
        _streams[cam] = synth.Sequence(w=c["w"], h=c["h"], seed=11, zf=c["zfx"]).frames(max(n, 15))
    ts, fr = _streams[cam]
    return ts[:n], fr[:n]


def _kc(cam, und):
    return None if not und else (pu.EUROC_KC if cam == "euroc" else KC)


# row steps, from the tight one (w * bytes per pixel) of frame i
STEPS = {
    "tight": lambda i, r: r,
    "+1": lambda i, r: r + 1,
    "+3": lambda i, r: r + 3,
    "+61": lambda i, r: r + 61,
    "512": lambda i, r: -(-r // 512) * 512,   # a GpuMat's pitch
    "mixed": lambda i, r: [r, r + 1, r + 3, r + 61, -(-r // 512) * 512][i % 5],
}


def _filled(size, fill, seed):
    if fill == "random":
        return np.random.default_rng(seed).integers(0, 256, size, dtype=np.uint8)
    return np.full(size, fill, np.uint8)


def place(frames, mem, step="mixed", fill="random", seed=0):
    """Each frame of `frames` (RGB [n, h, w, 3] or mono [n, h, w]) in a buffer of its own, at byte offset i % 4 of it, rows
    STEPS[step](i) bytes apart; `fill` (a byte value or "random") in the row padding and around the frame.  A list of
    NumPy views (mem "host") or torch CUDA views (mem "dev")."""
    import torch
    n, h, w = frames.shape[:3]
    bpp = 3 if frames.ndim == 4 else 1
    out = []
    for i in range(n):
        s, off = STEPS[step](i, w * bpp), i % 4
        buf = _filled(off + h * s + 5, fill, seed * 1000 + i)
        buf[off:off + h * s].reshape(h, s)[:, :w * bpp] = frames[i].reshape(h, w * bpp)
        shape, strides = ((h, w, 3), (s, 3, 1)) if bpp == 3 else ((h, w), (s, 1))
        if mem == "host":
            out.append(np.lib.stride_tricks.as_strided(buf[off:], shape, strides))
        else:
            out.append(torch.from_numpy(buf).cuda()[off:].as_strided(shape, strides))
    return out


def new_pipeline(cam, batch, kc, mirror, imu=None, live=False):
    from rebvo_b200 import capi
    pl = capi.Pipeline(capi.default_params(_cams()[cam]), max_batch=batch)
    if kc is not None:
        pl.set_undistort(kc)
    if imu is None:
        if mirror:
            pl.set_mirror(mirror)
        pl.set_depth(capi.depth_params())
        pl.set_depth_image(2)
    elif live:
        pl.set_imu_live(capi.default_imu_params(InitBias=1, InitBiasFrameNum=5),
                        (imu[-1, 0] - imu[0, 0]) / (len(imu) - 1), len(imu) + 8)
        pl.push_imu(imu)
    else:
        pl.set_imu(imu, capi.default_imu_params(InitBias=1, InitBiasFrameNum=5))
    pl.set_odometry(True)
    return pl


def products(pl, n, mirror):
    out = []
    for i in range(n):
        rec = pl.mirror(i).tobytes() if mirror else None
        cells, md = pl.depth(i)
        r, s = pl.depth_image(i)
        out.append((rec, cells.tobytes() + np.float64(md).tobytes(), r.tobytes() + s.tobytes()))
    return out


def run(cam, sizes, pushes, fmt="rgb", und=False, mirror=1, imu=None, live=False):
    """The frames of `cam` in pushes of `sizes` frames on one pipeline; pushes[k % len(pushes)](pl, frames, ts) makes push
    k.  nav, odometry, per-frame products, launches per push, and the two newest maps after the last push."""
    n = sum(sizes)
    ts, fr = stream(cam, n)
    src = fr[..., 0] if fmt == "mono" else fr
    pl = new_pipeline(cam, max(sizes), _kc(cam, und), mirror, imu, live)
    navs, odo, prods, launches = [], [], [], []
    try:
        s = 0
        for k, m in enumerate(sizes):
            l0 = pl.launches()
            nav = pushes[k % len(pushes)](pl, src[s:s + m], ts[s:s + m])
            launches.append(pl.launches() - l0)
            navs.append(nav)
            odo.append(pl.odometry())
            if imu is None:
                prods += products(pl, m, mirror)
            s += m
        maps = [(m.keylines(), m.mask()) for m in (pl.map(0), pl.map(1))]
    finally:
        pl.close()
    return dict(nav=np.concatenate(navs), odometry=np.concatenate(odo), products=prods, launches=launches, maps=maps)


def packed(mem):
    return lambda pl, frames, ts: pu.push(pl, frames, ts, mem)


def strided(mem, step="mixed", fill="random"):
    return lambda pl, frames, ts: pl.push_frames(place(frames, mem, step, fill, seed=int(ts[0] * 20)), ts)


def assert_same(a, b, what, launches=True):
    assert pu.raw(a["nav"]).tobytes() == pu.raw(b["nav"]).tobytes(), what + ": nav records"
    assert pu.raw(a["odometry"]).tobytes() == pu.raw(b["odometry"]).tobytes(), what + ": odometry records"
    assert len(a["products"]) == len(b["products"])
    for f, (x, y) in enumerate(zip(a["products"], b["products"])):
        for k, name in enumerate(("mirror", "grid", "image")):
            assert x[k] == y[k], "%s: %s of frame %d" % (what, name, f)
    for age, ((ka, ma), (kb, mb)) in enumerate(zip(a["maps"], b["maps"])):
        assert pu.keylines_equal(ka, kb), "%s: keylines of map %d" % (what, age)
        assert np.array_equal(ma, mb), "%s: mask of map %d" % (what, age)
    if launches:
        assert a["launches"] == b["launches"], "%s: launches per push %s against %s" % (what, a["launches"], b["launches"])


# ---- 1. format x memory x undistortion x size x step x push size ---------------------------------------------------------
# (camera, format, memory, undistortion, step, push sizes, mirror mode).  A host push of 64 frames runs as a head and a rest
# sub-batch; the first push of a pipeline is eager, the later ones replay captured batches.
CASES = [
    ("euroc", "rgb", "host", False, "tight", (1, 7, 7), 1),
    ("euroc", "rgb", "host", True, "+61", (1, 64), 2),
    ("euroc", "rgb", "dev", False, "512", (1, 7, 7), 2),
    ("euroc", "rgb", "dev", True, "mixed", (1, 64), 1),
    ("euroc", "mono", "host", False, "+3", (1, 7, 7), 2),
    ("euroc", "mono", "host", True, "mixed", (7, 7), 1),
    ("euroc", "mono", "dev", False, "+1", (1, 7, 7), 1),
    ("euroc", "mono", "dev", True, "512", (1, 64), 2),
    ("1241", "rgb", "host", True, "+1", (1, 7, 7), 1),
    ("1241", "rgb", "dev", False, "+3", (1, 7, 7), 2),
    ("1241", "rgb", "dev", True, "tight", (1, 7, 7), 1),
    ("1241", "mono", "dev", True, "mixed", (1, 7, 7), 2),
    ("1226", "rgb", "dev", False, "mixed", (1, 7, 7), 1),
    ("1226", "rgb", "host", False, "512", (7, 7), 2),
    ("1226", "mono", "host", True, "+61", (1, 7, 7), 1),
    ("1226", "mono", "dev", False, "tight", (1, 7, 7), 2),
    ("1226", "mono", "dev", True, "+61", (1, 7, 7), 1),
]


@pytest.mark.parametrize("cam,fmt,mem,und,step,sizes,mirror", CASES,
                         ids=["-".join(map(str, c[:5])) + "-%s-m%d" % ("x".join(map(str, c[5])), c[6]) for c in CASES])
def test_strided_equals_packed(built, cam, fmt, mem, und, step, sizes, mirror):
    want = run(cam, sizes, [packed(mem)], fmt, und, mirror)
    got = run(cam, sizes, [strided(mem, step)], fmt, und, mirror)
    assert_same(got, want, "%s %s %s und=%s step %s" % (cam, fmt, mem, und, step))


# ---- 2. placement: frames in reverse order in one buffer, crop views of larger frames ------------------------------------
def _reversed_buffer(frames, mem):
    """The frames in one buffer, frame i in slot n-1-i, rows padded by 7 bytes: one array with a negative frame stride (a
    NumPy view, or a __cuda_array_interface__ object over a torch buffer)."""
    import torch
    from rebvo_b200 import capi
    n, h, w = frames.shape[:3]
    bpp = 3 if frames.ndim == 4 else 1
    s = w * bpp + 7
    buf = _filled(n * h * s + 3, "random", 5)
    body = buf[3:].reshape(n, h, s)
    for i in range(n):
        body[n - 1 - i, :, :w * bpp] = frames[i].reshape(h, w * bpp)
    shape, strides = (n, h, w) + ((3,) if bpp == 3 else ()), (-h * s, s) + ((3, 1) if bpp == 3 else (1,))
    if mem == "host":
        return np.lib.stride_tricks.as_strided(body[n - 1], shape, strides)
    dev = torch.from_numpy(buf).cuda()
    keep.append(dev)
    return capi._CudaArray(dev.data_ptr() + 3 + (n - 1) * h * s, shape, "|u1", strides)


def _crops(frames, mem):
    """The frames as one crop view [:, 5:5+h, 6:6+w] of larger frames (7 more rows, 13 more columns)."""
    import torch
    n, h, w = frames.shape[:3]
    big = _filled(n * (h + 7) * (w + 13) * (frames.size // (n * h * w)), "random", 9).reshape(
        (n, h + 7, w + 13) + frames.shape[3:])
    big[:, 5:5 + h, 6:6 + w] = frames
    if mem == "dev":
        big = torch.from_numpy(big).cuda()
    return big[:, 5:5 + h, 6:6 + w]


keep = []


@pytest.mark.parametrize("mem", ["host", "dev"])
@pytest.mark.parametrize("fmt", ["rgb", "mono"])
def test_placement(built, mem, fmt):
    want = run("1241", (1, 7, 7), [packed(mem)], fmt, True, 1)
    try:
        got = run("1241", (1, 7, 7), [lambda pl, f, ts: pl.push_frames(_reversed_buffer(f, mem), ts),
                                      lambda pl, f, ts: pl.push_frames(_crops(f, mem), ts)], fmt, True, 1)
    finally:
        keep.clear()
    assert_same(got, want, "%s %s: reversed buffer, crops" % (fmt, mem))


# ---- 3. row padding never changes a result -------------------------------------------------------------------------------
@pytest.mark.parametrize("mem,fmt,cam,und", [("dev", "rgb", "1241", True), ("dev", "mono", "1226", False),
                                             ("host", "rgb", "euroc", True)])
def test_row_padding(built, mem, fmt, cam, und):
    a = run(cam, (1, 7), [strided(mem, "+61", 0)], fmt, und, 2)
    b = run(cam, (1, 7), [strided(mem, "+61", 255)], fmt, und, 2)
    assert_same(a, b, "%s %s: padding 0x00 against 0xff" % (mem, fmt))


# ---- 4. IMU mode, dataset and live -------------------------------------------------------------------------------------
@pytest.mark.parametrize("live", [False, True], ids=["dataset", "live"])
@pytest.mark.parametrize("mem,fmt", [("host", "rgb"), ("dev", "mono"), ("dev", "rgb")])
def test_imu_mode(built, live, mem, fmt):
    from rebvo_b200 import synth
    c = _cams()["euroc"]
    imu = synth.imu_samples(synth.Sequence(w=c["w"], h=c["h"], seed=11, zf=c["zfx"]), 15)
    want = run("euroc", (1, 7, 7), [packed(mem)], fmt, True, imu=imu, live=live)
    got = run("euroc", (1, 7, 7), [strided(mem)], fmt, True, imu=imu, live=live)
    assert_same(got, want, "IMU %s %s %s" % ("live" if live else "dataset", mem, fmt))


def test_imu_live_coverage(built):
    """Live IMU mode: a strided push the samples do not cover fails with RB_ERR_STATE and changes nothing."""
    from rebvo_b200 import capi, synth
    c = _cams()["euroc"]
    imu = synth.imu_samples(synth.Sequence(w=c["w"], h=c["h"], seed=11, zf=c["zfx"]), 15)
    ts, fr = stream("euroc", 8)
    navs = []
    for how in ("packed", "strided"):
        pl = capi.Pipeline(capi.default_params(c), max_batch=7)
        try:
            pl.set_imu_live(capi.default_imu_params(InitBias=1, InitBiasFrameNum=5),
                            (imu[-1, 0] - imu[0, 0]) / (len(imu) - 1), len(imu) + 8)
            cut = int(np.searchsorted(imu[:, 0], ts[3]))
            pl.push_imu(imu[:cut])
            out = [pu.push(pl, fr[:1], ts[:1], "dev") if how == "packed" else
                   pl.push_frames(place(fr[:1], "dev"), ts[:1])]
            if how == "strided":
                with pytest.raises(capi.RbError) as e:
                    pl.push_frames(place(fr[1:8], "dev"), ts[1:8])
                assert "error %d" % RB_ERR_STATE in str(e.value)
            pl.push_imu(imu[cut:])
            out.append(pu.push(pl, fr[1:8], ts[1:8], "dev") if how == "packed" else
                       pl.push_frames(place(fr[1:8], "dev"), ts[1:8]))
            navs.append(np.concatenate(out))
        finally:
            pl.close()
    assert pu.raw(navs[0]).tobytes() == pu.raw(navs[1]).tobytes()


# ---- 5. packed and strided pushes on one pipeline -----------------------------------------------------------------------
@pytest.mark.parametrize("mem,fmt,und", [("dev", "rgb", True), ("dev", "mono", False), ("host", "rgb", False)])
def test_alternation(built, mem, fmt, und):
    want = run("1241", (1, 7, 7, 7, 7), [packed(mem)], fmt, und, 2)
    got = run("1241", (1, 7, 7, 7, 7), [packed(mem), strided(mem)], fmt, und, 2)
    assert_same(got, want, "alternating %s %s" % (mem, fmt))   # (launches per push compared in every position)


# ---- 6. a frame written by a torch kernel right before the push ----------------------------------------------------------
def test_torch_stream_order(built):
    import torch
    ts, fr = stream("euroc", 8)
    n, h, w = fr.shape[:3]
    s = -(-3 * w // 512) * 512
    src = torch.from_numpy(fr).cuda()
    navs = []
    for sync_first in (True, False):
        pl = new_pipeline("euroc", 7, pu.EUROC_KC, 0)
        try:
            out = []
            for a, b in ((0, 1), (1, 8)):
                big = torch.zeros((b - a) * h * s, dtype=torch.uint8, device="cuda")
                view = big.as_strided((b - a, h, w, 3), (h * s, s, 3, 1))
                view.copy_(src[a:b])           # a kernel on torch's current stream
                if sync_first:
                    torch.cuda.synchronize()
                out.append(pl.push_frames(view, ts[a:b]))
            navs.append(np.concatenate(out))
        finally:
            pl.close()
    assert pu.raw(navs[0]).tobytes() == pu.raw(navs[1]).tobytes()


# ---- 7. errors ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mem", ["host", "dev"])
def test_bad_arguments(built, mem):
    """RB_ERR_ARG for every bad argument, before anything is enqueued: the next good push gives the twin's records."""
    from rebvo_b200 import capi
    ts, fr = stream("1226", 5)
    w = fr.shape[2]
    want = run("1226", (1, 2, 2), [packed(mem)], "rgb", True, 0)["nav"]
    pl = new_pipeline("1226", 2, KC, 0)
    try:
        got = [pl.push_frames(place(fr[:1], mem), ts[:1]), pl.push_frames(place(fr[1:3], mem), ts[1:3])]
        fn = pl.L.rb_pipeline_push_frames_dev if mem == "dev" else pl.L.rb_pipeline_push_frames
        views = place(fr[3:5], mem)
        good = [capi.frame_table([v], w, fr.shape[1])[2][0] for v in views]   # (data, step)
        tsa = np.ascontiguousarray(ts[3:5])
        nav = np.zeros(3, capi.NAV)

        def call(fmt, table, n, t=tsa):
            fr_arr = None if table is None else capi._p(np.array([(p or 0, s) for p, s in table], capi.FRAME))
            return fn(pl.h_, fmt, fr_arr, None if t is None else capi._p(t), n, capi._p(nav))
        bad = [
            call(2, good, 2), call(-1, good, 2),                           # format
            call(0, good, 0), call(0, good + good[:1], 3),                 # n outside 1..max_batch (2)
            call(0, None, 2), call(0, good, 2, None),                      # NULL frames, ts
            call(0, [good[0], (None, good[1][1])], 2),                     # NULL data
            call(0, [good[0], (good[1][0], 3 * w - 1)], 2),                # step shorter than an RGB row
            call(1, [good[0], (good[1][0], w - 1)], 2),                    # ... than a mono row
        ]
        assert bad == [RB_ERR_ARG] * len(bad), bad
        got.append(pl.push_frames(views, ts[3:5]))
        with pytest.raises(ValueError):   # a pixel stride of 6 bytes
            pl.push_frames([np.zeros((fr.shape[1], 2 * w, 3), np.uint8)[:, ::2]], ts[:1])
        with pytest.raises(ValueError):   # host and device frames in one push
            pl.push_frames([place(fr[:1], "host")[0], place(fr[:1], "dev")[0]], ts[:2])
    finally:
        pl.close()
    assert pu.raw(np.concatenate(got)).tobytes() == pu.raw(want).tobytes()

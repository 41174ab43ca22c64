"""Asynchronous pushes (rb_pipeline_set_async / enqueue / wait / poll): every ticket's records and outputs are byte for byte
those of a twin pipeline fed the same frames by synchronous pushes of the same sizes, whatever the depth, input layout,
output memory and order of the waits; a full queue, the calls refused while tickets are outstanding and the consumer-stream
fence leave the run as it would have been; and with the feature off the pushes launch what they launched before."""
import ctypes as C

import numpy as np
import pytest

import pipeline_util as pu

pytestmark = pytest.mark.gpu

KITTI = dict(w=1241, h=376, zfx=718.856, zfy=718.856, ppx=607.1928, ppy=185.2157)   # a width that is not a multiple of 4
RB_ERR_ARG, RB_ERR_STATE = -2, -4
BATCH = 4
# push sizes: 1, 3 and max_batch mixed, 27 frames in 12 pushes, so that the tickets cross the three ring phases and both
# scale-space workspaces several times
SIZES = [1, 3, 4, 1, 1, 3, 4, 1, 3, 1, 1, 4]

_streams = {}


def stream(cam, n=sum(SIZES)):
    from rebvo_b200 import synth
    if cam not in _streams:
        c = synth.EUROC if cam == "euroc" else KITTI
        _streams[cam] = synth.Sequence(w=c["w"], h=c["h"], seed=21, zf=c["zfx"]).frames(max(n, sum(SIZES)))
    ts, fr = _streams[cam]
    return ts[:n], fr[:n]


def chunks(cam, fmt, sizes=SIZES):
    ts, fr = stream(cam, sum(sizes))
    if fmt == "mono":
        fr = np.ascontiguousarray(fr[..., 0])
    out, s = [], 0
    for n in sizes:
        out.append((ts[s:s + n], fr[s:s + n]))
        s += n
    return out


def enq(pl, chunk):
    """Enqueue one (ts, frames) chunk from host memory."""
    ts, fr = chunk
    return pl.enqueue(fr, ts, "mono" if fr.ndim == 3 else "rgb")


def new_pipeline(cam, where="host", mirror=0, mode=0, kc=False, depth=True, odometry=True):
    from rebvo_b200 import capi, synth
    pl = capi.Pipeline(capi.default_params(synth.EUROC if cam == "euroc" else KITTI), max_batch=BATCH)
    if kc:
        pl.set_undistort(pu.EUROC_KC)
    if mirror:
        pl.set_mirror(mirror)
    if mode:
        pl.set_depth_image(mode)
    if depth:
        pl.set_depth(capi.depth_params())
    if odometry:
        pl.set_odometry(True)
    if where == "device":
        pl.set_output_memory("device")
    return pl


def feed(frames, how):
    """The frames of one enqueue as the layout `how` passes them: packed host, packed device, or strided device frames
    (each frame in a buffer with padded rows)."""
    import torch
    if how == "host":
        return frames
    if how == "device":
        return torch.from_numpy(frames).cuda()
    pad = torch.zeros((len(frames), frames.shape[1], frames.shape[2] + 5) + frames.shape[3:], dtype=torch.uint8,
                      device="cuda")
    pad[:, :, 3:3 + frames.shape[2]] = torch.from_numpy(frames).cuda()
    return [pad[i, :, 3:3 + frames.shape[2]] for i in range(len(frames))]


def products(pl, n, where, mirror, mode):
    """The bytes of every output of the last push or waited ticket: odometry, and per frame (mirror, grid, image)."""
    out = [pu.raw(pl.odometry()).tobytes()]
    for i in range(n):
        rec = img = None
        if where == "host":
            rec = pl.mirror(i).tobytes() if mirror else None
            cells, md = pl.depth(i)
            grid = tuple(np.ascontiguousarray(cells[k]).tobytes() for k in ("rho", "s_rho", "dist", "fixed"))
            grid += (np.float64(md).tobytes(),)
            if mode:
                r, s = pl.depth_image(i)
                img = r.tobytes() + (b"" if s is None else s.tobytes())
        else:
            rec = pl.mirror_dev(i).cpu().numpy().tobytes() if mirror else None
            grid = tuple(t.contiguous().cpu().numpy().tobytes() for t in pl.depth_dev(i))
            if mode:
                r, s = pl.depth_image_dev(i)
                img = r.cpu().numpy().tobytes() + (b"" if s is None else s.cpu().numpy().tobytes())
        out.append((rec, grid, img))
    return out


def sync_run(cam, fmt, mirror, mode, kc, sizes=SIZES):
    """The twin: host-memory pushes of the same sizes, host outputs; (nav bytes, products) per push and the final blob."""
    pl = new_pipeline(cam, "host", mirror, mode, kc)
    try:
        res = []
        for ts, fr in chunks(cam, fmt, sizes):
            nav = pu.push(pl, fr, ts)
            res.append((pu.raw(nav).tobytes(), products(pl, len(ts), "host", mirror, mode)))
        return res, pl.save_state()
    finally:
        pl.close()


def async_run(pl, cam, fmt, how, where, mirror, mode, depth, pattern, sizes=SIZES):
    """Enqueue every chunk; when `depth` tickets are outstanding (and at the end) wait: the oldest one ("oldest"), all of
    them one at a time ("burst"), or only the newest, which retires the others with it ("newest").  {push index: (nav
    bytes, products)} of the tickets waited."""
    got, pending = {}, []

    def wait(k, t):
        nav = pl.wait(t)
        assert pl.poll() >= t
        got[k] = (pu.raw(nav).tobytes(), products(pl, len(nav), where, mirror, mode))

    def drain(final):
        nonlocal pending
        if pattern == "oldest":
            while pending and (final or len(pending) == depth):
                wait(*pending.pop(0))
        elif pattern == "burst":
            for k, t in pending:
                wait(k, t)
            pending = []
        else:
            wait(*pending[-1])
            pending = []

    for k, (ts, fr) in enumerate(chunks(cam, fmt, sizes)):
        pending.append((k, pl.enqueue(feed(fr, how), ts, fmt)))
        if len(pending) == depth:
            drain(False)
    if pending:
        drain(True)
    return got


def assert_tickets(got, want, what):
    assert got, what
    for k, (nav, prods) in got.items():
        assert nav == want[k][0], "%s: nav records of push %d" % (what, k)
        assert prods[0] == want[k][1][0], "%s: odometry of push %d" % (what, k)
        for f, (a, b) in enumerate(zip(prods[1:], want[k][1][1:])):
            for j, name in enumerate(("mirror", "grid", "image")):
                assert a[j] == b[j], "%s: %s of frame %d of push %d" % (what, name, f, k)


# ---- 1. identity ------------------------------------------------------------------------------------------------------------
# (camera, undistortion, format, input layout, output memory, mirror mode, image mode, depth, wait pattern)
CASES = [
    ("euroc", True, "rgb", "host", "host", 2, 2, 2, "oldest"),
    ("euroc", True, "mono", "device", "device", 1, 1, 4, "burst"),
    ("kitti", False, "rgb", "strided", "device", 2, 2, 8, "newest"),
    ("kitti", False, "mono", "host", "host", 1, 1, 1, "oldest"),
    ("euroc", True, "rgb", "strided", "host", 1, 2, 4, "newest"),
    ("kitti", False, "mono", "device", "device", 2, 1, 2, "burst"),
]


@pytest.mark.parametrize("cam,kc,fmt,how,where,mirror,mode,depth,pattern", CASES)
def test_tickets_are_the_synchronous_pushes(built, cam, kc, fmt, how, where, mirror, mode, depth, pattern):
    want, blob = sync_run(cam, fmt, mirror, mode, kc)
    pl = new_pipeline(cam, where, mirror, mode, kc)
    try:
        pl.set_async(depth)
        got = async_run(pl, cam, fmt, how, where, mirror, mode, depth, pattern)
        assert_tickets(got, want, "%s %s %s depth %d %s" % (cam, fmt, how, depth, pattern))
        if pattern != "newest":
            assert sorted(got) == list(range(len(SIZES)))
        assert pl.save_state() == blob
    finally:
        pl.close()


# ---- 2. a full queue ----------------------------------------------------------------------------------------------------------
def test_enqueue_beyond_depth_changes_nothing(built):
    from rebvo_b200 import capi
    want, blob = sync_run("euroc", "rgb", 2, 1, False)
    pl = new_pipeline("euroc", "host", 2, 1)
    try:
        pl.set_async(2)
        ch = chunks("euroc", "rgb")
        got, k = {}, 0
        while k < len(ch):
            t0 = enq(pl, ch[k])
            t1 = enq(pl, ch[k + 1])
            with pytest.raises(capi.RbError):
                enq(pl, ch[min(k + 2, len(ch) - 1)])   # refused: the run goes on as if it never came
            ts = np.ascontiguousarray(ch[k][0])
            tk = C.c_int64(-1)
            assert pl.L.rb_pipeline_enqueue(pl.h_, 0, 0, capi._p(ch[k][1]), capi._p(ts), len(ts), C.byref(tk)) == RB_ERR_STATE
            assert tk.value == -1
            for j, t in ((k, t0), (k + 1, t1)):
                nav = pl.wait(t)
                got[j] = (pu.raw(nav).tobytes(), products(pl, len(nav), "host", 2, 1))
            k += 2
        assert_tickets(got, want, "full queue")
        assert pl.save_state() == blob
    finally:
        pl.close()


# ---- 3. refusals while tickets are outstanding ----------------------------------------------------------------------------
def test_refusals_leave_the_run_unchanged(built):
    from rebvo_b200 import capi
    _p = capi._p
    want, blob = sync_run("euroc", "rgb", 2, 2, False)
    ch = chunks("euroc", "rgb")
    other = new_pipeline("euroc")
    try:
        pu.push(other, ch[0][1], ch[0][0])
        other_blob = other.save_state()
    finally:
        other.close()
    pl = new_pipeline("euroc", "host", 2, 2)
    try:
        pl.set_async(3)
        L, h = pl.L, pl.h_
        got, k = {}, 0
        while k < len(ch):
            tickets = [(j, enq(pl, ch[j])) for j in range(k, min(k + 3, len(ch)))]
            ts, fr = np.ascontiguousarray(ch[k][0]), ch[k][1]
            nav = np.zeros(len(ts), capi.NAV)
            table = np.array([(fr[i].__array_interface__["data"][0], fr.shape[2] * 3) for i in range(len(ts))], capi.FRAME)
            need, out6, plane = C.c_size_t(0), np.zeros(6, np.float32), np.zeros((480, 752), np.float32)
            refused = {
                "push": L.rb_pipeline_push(h, _p(fr), _p(ts), len(ts), _p(nav)),
                "push_frames": L.rb_pipeline_push_frames(h, 0, _p(table), _p(ts), len(ts), _p(nav)),
                "reset": L.rb_pipeline_reset(h),
                "save_state": L.rb_pipeline_save_state(h, None, C.c_size_t(0), C.byref(need)),
                "load_state": L.rb_pipeline_load_state(h, other_blob, C.c_size_t(len(other_blob))),
                "set_mirror": L.rb_pipeline_set_mirror(h, 1),
                "set_depth": L.rb_pipeline_set_depth(h, None),
                "set_depth_image": L.rb_pipeline_set_depth_image(h, 1),
                "set_odometry": L.rb_pipeline_set_odometry(h, 0),
                "set_output_memory": L.rb_pipeline_set_output_memory(h, 1),
                "set_undistort": L.rb_pipeline_set_undistort(h, None),
                "set_consumer_stream": L.rb_pipeline_set_consumer_stream(h, None),
                "set_async": L.rb_pipeline_set_async(h, 2),
                "batch_plane": L.rb_pipeline_batch_plane(h, 0, 0, _p(plane)),
                "stage_ms": L.rb_pipeline_stage_ms(h, _p(out6)),
            }
            assert all(v == RB_ERR_STATE for v in refused.values()), refused
            for j, t in tickets:
                nav = pl.wait(t)
                got[j] = (pu.raw(nav).tobytes(), products(pl, len(nav), "host", 2, 2))
            k += len(tickets)
        assert_tickets(got, want, "refusals")
        assert pl.save_state() == blob
        # waits on a retired or never issued ticket
        assert L.rb_pipeline_wait(h, C.c_int64(0), None) == RB_ERR_ARG
        assert L.rb_pipeline_wait(h, C.c_int64(1000), None) == RB_ERR_ARG
        assert L.rb_pipeline_wait(h, C.c_int64(-1), None) == RB_ERR_ARG
        # with none outstanding the calls work again
        assert pl.stage_ms().shape == (6,)
        pl.set_async(0)
        tk = C.c_int64(-1)
        ts, fr = np.ascontiguousarray(ch[0][0]), ch[0][1]
        assert L.rb_pipeline_enqueue(h, 0, 0, _p(fr), _p(ts), len(ts), C.byref(tk)) == RB_ERR_ARG   # async off
    finally:
        pl.close()


def test_blob_of_an_async_run_continues_in_a_sync_pipeline(built):
    """Half the pushes through tickets, the blob into a synchronous pipeline, the rest pushed there: the twin's records."""
    half = len(SIZES) // 2
    want, _ = sync_run("kitti", "mono", 1, 1, False)
    pl = new_pipeline("kitti", "device", 1, 1)
    try:
        pl.set_async(2)
        async_run(pl, "kitti", "mono", "device", "device", 1, 1, 2, "burst", SIZES[:half])
        blob = pl.save_state()
    finally:
        pl.close()
    cont = new_pipeline("kitti", "host", 1, 1)
    try:
        cont.load_state(blob)
        for k, (ts, fr) in enumerate(chunks("kitti", "mono")[half:], start=half):
            nav = pu.push(cont, fr, ts)
            assert pu.raw(nav).tobytes() == want[k][0], "push %d" % k
            assert products(cont, len(ts), "host", 1, 1) == want[k][1], "push %d" % k
    finally:
        cont.close()


def test_set_async_is_refused_in_imu_mode(built):
    from rebvo_b200 import capi, synth
    seq = pu.euroc_sequence()
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=2)
    try:
        pl.set_imu(synth.imu_samples(seq, 4), capi.default_imu_params())
        for depth in (0, 2, -1, 9):
            assert pl.L.rb_pipeline_set_async(pl.h_, depth) == RB_ERR_ARG
    finally:
        pl.close()


# ---- 4. off means off ----------------------------------------------------------------------------------------------------------
def test_off_is_the_pipeline_that_never_had_it(built):
    """Never called, set_async(0), and set_async(3) then set_async(0): the same records and launches per push; and a
    ticket launches as many kernels as the synchronous push of its size."""
    import torch
    res = {}
    for arm in ("never", "zero", "on_off", "async"):
        pl = new_pipeline("euroc", "host", 2, 2, kc=True)
        try:
            if arm == "zero":
                pl.set_async(0)
            elif arm == "on_off":
                pl.set_async(3)
                pl.set_async(0)
            elif arm == "async":
                pl.set_async(2)
            navs, launches = [], []
            for ts, fr in chunks("euroc", "rgb"):
                dev = torch.from_numpy(fr).cuda()
                torch.cuda.synchronize()
                l0 = pl.launches()
                if arm == "async":
                    nav = pl.wait(pl.enqueue(dev, ts))
                else:
                    nav = pl.push_dev(dev.data_ptr(), ts)
                launches.append(pl.launches() - l0)
                navs.append(pu.raw(nav).tobytes())
            res[arm] = (navs, launches)
        finally:
            pl.close()
    for arm in ("zero", "on_off", "async"):
        assert res[arm][0] == res["never"][0], arm
        assert res[arm][1] == res["never"][1], arm


# ---- 5. device outputs: the consumer-stream fence ------------------------------------------------------------------------
def test_enqueue_waits_for_the_consumer_stream(built):
    """Depth 1: the ticket after t reuses t's slot.  A torch stream still busy with t's outputs (a long sleep, then clones)
    when that ticket is enqueued: the clones hold t's bytes.  One run, no retries."""
    import torch
    sizes = [BATCH, BATCH]
    want, _ = sync_run("euroc", "rgb", 2, 2, False, sizes)
    ch = chunks("euroc", "rgb", sizes)
    pl = new_pipeline("euroc", "device", 2, 2)
    try:
        pl.set_async(1)
        pl.wait(enq(pl, ch[0]))
        busy = torch.cuda.Stream()
        with torch.cuda.stream(busy):
            torch.cuda._sleep(100_000_000)   # ~50 ms at the H100's clocks
            rho, srho = (t.clone() for t in pl.depth_image_dev(BATCH - 1))
            rec = pl.mirror_dev(BATCH - 1).clone()
            t1 = enq(pl, ch[1])   # waits for `busy`: the current stream
        torch.cuda.synchronize()
        rec0, _, img0 = want[0][1][BATCH]
        assert rec.cpu().numpy().tobytes() == rec0
        assert rho.cpu().numpy().tobytes() + srho.cpu().numpy().tobytes() == img0
        nav = pl.wait(t1)
        assert_tickets({1: (pu.raw(nav).tobytes(), products(pl, BATCH, "device", 2, 2))}, want, "fence")
    finally:
        pl.close()

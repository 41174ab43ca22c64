"""Per-frame outputs in device memory (rb_pipeline_set_output_memory): the keyline mirror, the depth grid and the depth image
of a device-mode pipeline are byte for byte those of a host-mode twin on the same frames, read through zero-copy torch
CUDA tensors; the consumer-stream fence keeps a push from overwriting outputs a torch kernel still reads."""
import ctypes as C

import numpy as np
import pytest

import pipeline_util as pu

pytestmark = pytest.mark.gpu

KITTI = dict(w=1241, h=376, zfx=718.856, zfy=718.856, ppx=607.1928, ppy=185.2157)   # a width that is not a multiple of 4
RB_ERR_ARG, RB_ERR_STATE = -2, -4


def _cams():
    from rebvo_b200 import synth
    return {"euroc": synth.EUROC, "kitti": KITTI}


_streams = {}


def stream(cam, n):
    """(ts, RGB frames) of a seeded sequence on camera `cam`, the first n frames (rendered once per module)."""
    from rebvo_b200 import synth
    if cam not in _streams or len(_streams[cam][0]) < n:
        c = _cams()[cam]
        _streams[cam] = synth.Sequence(w=c["w"], h=c["h"], seed=21, zf=c["zfx"]).frames(max(n, 16))
    ts, fr = _streams[cam]
    return ts[:n], fr[:n]


def new_pipeline(cam, batch, where, mirror=0, depth=True, mode=0, kc=None, odometry=True):
    from rebvo_b200 import capi
    pl = capi.Pipeline(capi.default_params(_cams()[cam]), max_batch=batch)
    if kc is not None:
        pl.set_undistort(kc)
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


def products(pl, n, where, mirror, depth, mode):
    """The bytes of every output of frames 0..n-1 of the last push: (mirror records, cells + min_dist, image planes)."""
    out = []
    for i in range(n):
        rec = grid = img = None
        if where == "host":
            if mirror:
                rec = pl.mirror(i).tobytes()
            if depth:
                cells, md = pl.depth(i)
                grid = cells.tobytes() + np.float64(md).tobytes()
            if depth and mode:
                r, s = pl.depth_image(i)
                img = r.tobytes() + (b"" if s is None else s.tobytes())
        else:
            if mirror:
                rec = pl.mirror_dev(i).cpu().numpy().tobytes()
            if depth:
                g = pl.depth_dev(i)
                gh, gw = g.rho.shape
                grid = raw_dev(g.rho.data_ptr(), gh * gw * 32 + 8).tobytes()
            if depth and mode:
                r, s = pl.depth_image_dev(i)
                img = r.cpu().numpy().tobytes() + (b"" if s is None else s.cpu().numpy().tobytes())
        out.append((rec, grid, img))
    return out


def raw_dev(ptr, nbytes):
    """`nbytes` bytes of device memory at ptr, copied to the host."""
    from rebvo_b200 import capi
    import torch
    return capi._dev_view(ptr, (nbytes,), torch.uint8, (1,), 0).cpu().numpy()


def run(cam, batch, n, where, how="host", fmt="rgb", kc=None, mirror=0, depth=True, mode=0):
    """n frames in pushes of `batch`: nav, odometry, per-frame products and launches per push."""
    ts, fr = stream(cam, n)
    pl = new_pipeline(cam, batch, where, mirror, depth, mode, kc)
    navs, prods, launches = [], [], []
    odo = []
    try:
        for s in range(0, n, batch):
            src = fr[s:s + batch, ..., 0] if fmt == "mono" else fr[s:s + batch]
            l0 = pl.launches()
            nav = pu.push(pl, src, ts[s:s + batch], how)
            launches.append(pl.launches() - l0)
            navs.append(nav)
            odo.append(pl.odometry())
            prods += products(pl, len(nav), where, mirror, depth, mode)
    finally:
        pl.close()
    return dict(nav=np.concatenate(navs), odometry=np.concatenate(odo), products=prods, launches=launches)


def assert_same(dev, host, what):
    assert pu.raw(dev["nav"]).tobytes() == pu.raw(host["nav"]).tobytes(), what + ": nav records"
    assert pu.raw(dev["odometry"]).tobytes() == pu.raw(host["odometry"]).tobytes(), what + ": odometry records"
    assert len(dev["products"]) == len(host["products"]) == len(host["nav"])
    for f, (a, b) in enumerate(zip(dev["products"], host["products"])):
        for k, name in enumerate(("mirror", "grid", "image")):
            assert (a[k] is None) == (b[k] is None), (what, f, name)
            assert a[k] == b[k], "%s: %s of frame %d differs" % (what, name, f)


# ---- 1. device mode gives the host twin's bytes ------------------------------------------------------------------------
# (camera, push size, frames, input memory, format, undistortion, mirror mode, depth grid, image mode).  Full 64-frame
# pushes from host memory run as two sub-batches, the others as one.
CASES = [
    ("euroc", 1, 3, "host", "rgb", False, 1, True, 2),
    ("euroc", 7, 14, "dev", "rgb", True, 2, True, 1),
    ("euroc", 7, 14, "host", "mono", False, 2, True, 2),
    ("euroc", 7, 14, "dev", "mono", True, 0, True, 2),
    ("euroc", 7, 14, "host", "rgb", False, 1, False, 0),
    ("euroc", 64, 64, "host", "rgb", True, 1, True, 2),
    ("euroc", 64, 64, "dev", "mono", False, 2, True, 1),
    ("kitti", 3, 6, "dev", "rgb", False, 1, True, 2),
    ("kitti", 3, 6, "host", "mono", True, 2, True, 1),
]


@pytest.mark.parametrize("cam,batch,n,how,fmt,und,mirror,depth,mode", CASES,
                         ids=["%s-b%d-%s-%s-%s-m%d-%s-i%d" % (c[0], c[1], c[3], c[4], "und" if c[5] else "raw", c[6],
                                                              "grid" if c[7] else "nogrid", c[8]) for c in CASES])
def test_device_outputs_equal_host(built, cam, batch, n, how, fmt, und, mirror, depth, mode):
    kc = pu.EUROC_KC if und else None
    host = run(cam, batch, n, "host", how, fmt, kc, mirror, depth, mode)
    dev = run(cam, batch, n, "device", how, fmt, kc, mirror, depth, mode)
    assert_same(dev, host, "%s batch %d %s %s mirror %d mode %d" % (cam, batch, how, fmt, mirror, mode))
    # no k_mirror_to_host in device mode; every other launch is the same
    fewer = [min(batch, n - s) if mirror else 0 for s in range(0, n, batch)]
    assert dev["launches"] == [h - d for h, d in zip(host["launches"], fewer)]


# ---- 2. switching host -> device -> host on one pipeline ---------------------------------------------------------------
@pytest.mark.parametrize("mirror", [0, 1, 2])
def test_switching_gives_host_twin_bytes(built, mirror):
    batch, n = 4, 16
    ts, fr = stream("euroc", n)
    wheres = ["host", "device", "host", "device"]

    def go(switch):
        pl = new_pipeline("euroc", batch, "host", mirror, True, 2)
        prods, launches, navs = [], [], []
        try:
            for k, s in enumerate(range(0, n, batch)):
                where = wheres[k] if switch else "host"
                if switch:
                    pl.set_output_memory(where)
                l0 = pl.launches()
                navs.append(pl.push(fr[s:s + batch], ts[s:s + batch]))
                launches.append(pl.launches() - l0)
                prods += products(pl, batch, where, mirror, True, 2)
        finally:
            pl.close()
        return dict(nav=np.concatenate(navs), odometry=np.zeros(0), products=prods, launches=launches)

    twin, sw = go(False), go(True)
    assert_same(sw, twin, "switched, mirror %d" % mirror)
    d = batch if mirror else 0
    assert sw["launches"] == [twin["launches"][0], twin["launches"][1] - d, twin["launches"][2], twin["launches"][3] - d]


# ---- 3. the consumer-stream fence ---------------------------------------------------------------------------------------
def test_push_waits_for_the_consumer_stream(built):
    """A torch stream still busy with push k's outputs (a long sleep, then clones of the image and the mirror) when push
    k+1 is made: the clones hold push k's bytes.  One run, no retries."""
    import torch
    batch = 4
    ts, fr = stream("euroc", 2 * batch)
    host = run("euroc", batch, 2 * batch, "host", mirror=2, mode=2)
    pl = new_pipeline("euroc", batch, "device", mirror=2, depth=True, mode=2)
    try:
        pl.push(fr[:batch], ts[:batch])
        busy = torch.cuda.Stream()
        with torch.cuda.stream(busy):
            torch.cuda._sleep(100_000_000)   # ~50 ms at the H100's clocks
            rho, srho = (t.clone() for t in pl.depth_image_dev(batch - 1))
            rec = pl.mirror_dev(batch - 1).clone()
            pl.push(fr[batch:], ts[batch:])   # waits for `busy`: the current stream
        torch.cuda.synchronize()
        want_rec, _, want_img = host["products"][batch - 1]
        assert rec.cpu().numpy().tobytes() == want_rec
        assert rho.cpu().numpy().tobytes() + srho.cpu().numpy().tobytes() == want_img
        # and push k+1's own outputs are the twin's
        assert products(pl, batch, "device", 2, True, 2) == host["products"][batch:]
    finally:
        pl.close()


# ---- 4. the torch views -------------------------------------------------------------------------------------------------
def test_torch_views(built):
    import torch
    from rebvo_b200 import capi
    batch = 5
    ts, fr = stream("kitti", batch)
    cam = KITTI
    for mirror, mode in ((1, 2), (2, 1)):
        pl = new_pipeline("kitti", batch, "device", mirror, True, mode)
        try:
            pl.push(fr, ts)
            rho_all, srho_all = pl.depth_images_dev()
            plane = (cam["w"] * cam["h"] + 63) // 64 * 64
            assert rho_all.shape == (batch, cam["h"], cam["w"]) and rho_all.dtype == torch.float32
            assert rho_all.stride() == (mode * plane, cam["w"], 1) and (srho_all is None) == (mode == 1)
            for i in range(batch):
                p, kn = C.c_void_p(0), C.c_int(0)
                assert pl.L.rb_pipeline_mirror_dev(pl.h_, i, C.byref(p), C.byref(kn)) == 0
                m = pl.mirror_dev(i)
                assert m.data_ptr() == p.value and m.shape == (kn.value, 168 if mirror == 1 else 15)
                assert m.dtype == torch.uint8 and m.is_contiguous() and m.device == torch.device("cuda", 0)
                cp, gw, gh, md = C.c_void_p(0), C.c_int(0), C.c_int(0), C.c_void_p(0)
                assert pl.L.rb_pipeline_depth_dev(pl.h_, i, C.byref(cp), C.byref(gw), C.byref(gh), C.byref(md)) == 0
                g = pl.depth_dev(i)
                assert (gh.value, gw.value) == (cam["h"] // 10, cam["w"] // 10)
                assert g.rho.data_ptr() == cp.value and g.s_rho.data_ptr() == cp.value + 8
                assert g.dist.data_ptr() == cp.value + 16 and g.fixed.data_ptr() == cp.value + 24
                assert md.value == cp.value + gw.value * gh.value * 32 and g.min_dist.data_ptr() == md.value
                for t, dt in ((g.rho, torch.float64), (g.s_rho, torch.float64), (g.dist, torch.float64),
                              (g.fixed, torch.int32)):
                    assert t.shape == (gh.value, gw.value) and t.dtype == dt and t.device.index == 0
                    assert t.stride() == (gw.value * 32 // t.element_size(), 32 // t.element_size())
                assert g.min_dist.shape == () and g.min_dist.dtype == torch.float64
                cells = np.frombuffer(raw_dev(cp.value, gw.value * gh.value * 32).tobytes(), capi.DEPTH_CELL)
                cells = cells.reshape(gh.value, gw.value)
                for f in ("rho", "s_rho", "dist", "fixed"):
                    assert np.array_equal(getattr(g, f).cpu().numpy(), cells[f]), f
                r, s = C.c_void_p(0), C.c_void_p(0)
                assert pl.L.rb_pipeline_depth_image_dev(pl.h_, i, C.byref(r), C.byref(s)) == 0
                rho, srho = pl.depth_image_dev(i)
                assert rho.data_ptr() == r.value and rho.shape == (cam["h"], cam["w"]) and rho.is_contiguous()
                assert torch.equal(rho_all[i], rho)
                if mode == 2:
                    assert srho.data_ptr() == s.value == r.value + 4 * plane and torch.equal(srho_all[i], srho)
                else:
                    assert srho is None and s.value is None
        finally:
            pl.close()


# ---- 5. errors ----------------------------------------------------------------------------------------------------------
def test_errors(built):
    from rebvo_b200 import capi, synth
    ts, fr = stream("euroc", 4)
    pl = new_pipeline("euroc", 2, "host", mirror=1, depth=True, mode=2)
    L, h = pl.L, pl.h_
    p, q, n, gw, gh = C.c_void_p(), C.c_void_p(), C.c_int(), C.c_int(), C.c_int()

    def dev_calls(i):
        return (L.rb_pipeline_mirror_dev(h, i, C.byref(p), C.byref(n)),
                L.rb_pipeline_depth_dev(h, i, C.byref(p), C.byref(gw), C.byref(gh), C.byref(q)),
                L.rb_pipeline_depth_image_dev(h, i, C.byref(p), C.byref(q)))

    def host_calls(i):
        md = C.c_double()
        return (L.rb_pipeline_mirror(h, i, C.byref(p), C.byref(n)),
                L.rb_pipeline_depth(h, i, C.byref(p), C.byref(gw), C.byref(gh), C.byref(md)),
                L.rb_pipeline_depth_image(h, i, C.byref(p), C.byref(q)))
    try:
        pl.push(fr[:2], ts[:2])
        assert dev_calls(0) == (RB_ERR_STATE,) * 3
        assert host_calls(0) == (0, 0, 0)
        for bad in (-1, 2):
            assert L.rb_pipeline_set_output_memory(h, bad) == RB_ERR_ARG
        pl.set_output_memory("device")
        assert host_calls(0) == (RB_ERR_STATE,) * 3
        assert dev_calls(0) == (RB_ERR_ARG,) * 3   # the switch dropped the last push's outputs
        pl.push(fr[2:4], ts[2:4])
        assert dev_calls(0) == dev_calls(1) == (0, 0, 0)
        for i in (-1, 2):
            assert dev_calls(i) == (RB_ERR_ARG,) * 3
        assert host_calls(0) == (RB_ERR_STATE,) * 3
        with pytest.raises(capi.RbError, match="-4"):
            pl.mirror(0)
        with pytest.raises(capi.RbError, match="-2"):
            pl.depth_image_dev(2)
        with pytest.raises(ValueError):
            pl.set_output_memory("pinned")
    finally:
        pl.close()
    seq = pu.euroc_sequence()
    pl = capi.Pipeline(capi.default_params(synth.EUROC), max_batch=2)
    try:
        pl.set_imu(synth.imu_samples(seq, 4))
        for where in (0, 1):
            assert pl.L.rb_pipeline_set_output_memory(pl.h_, where) == RB_ERR_ARG
    finally:
        pl.close()

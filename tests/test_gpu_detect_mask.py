"""Detection masks on the device.  Stage level: rb_map_detect_masked equals the masked restatement (tests/detect_mask.py) bit
for bit at R = 1..4 on every mask family, over a threshold chain with auto-gain on.  Pipeline: all-ones masks, and masks
that only zero pixels without a keyline, give the unmasked run's bytes; a fixed mask equals the same mask per frame, and a
fixed mask with per-frame masks their AND, in every input layout, with and without undistortion and at 1241x376;
masked_enqueue gives push_masked's bytes; IMU dataset and live mode; checkpoints; launch counts with the mask cleared;
argument errors."""
import ctypes as C

import numpy as np
import pytest

import front_states as fs
import pipeline_util as pu
from detect_mask import candidates, mask_families, port_detect_masked

pytestmark = pytest.mark.gpu

KITTI = dict(w=1241, h=376, zfx=718.856, zfy=718.856, ppx=607.1928, ppy=185.2157)
RB_ERR_ARG, RB_ERR_STATE = -2, -4
BATCH = 4
SIZES = [4, 4, 1, 3]          # 12 frames: the first push runs eagerly, the others replay captured batches
B = fs.BASE

_streams = {}


def stream(cam):
    from rebvo_b200 import synth
    key = cam["w"]
    if key not in _streams:
        _streams[key] = synth.Sequence(w=cam["w"], h=cam["h"], seed=21, zf=cam["zfx"]).frames(sum(SIZES))
    return _streams[key]


def fixed_mask(cam):
    """The bottom 20 % of the rows (a car's bonnet) and a 16-pixel frame (the housing), zero; the rest 255."""
    m = np.full((cam["h"], cam["w"]), 255, np.uint8)
    m[int(cam["h"] * 0.8):] = 0
    m[:16] = m[:, :16] = m[:, -16:] = 0
    return m


def blob_masks(cam, n, seed=0):
    """One mask per frame: a disc that moves from frame to frame (an object that moves on its own), zero; the rest 1."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:cam["h"], 0:cam["w"]]
    out = np.ones((n, cam["h"], cam["w"]), np.uint8)
    for i in range(n):
        cx, cy = rng.uniform(0.2, 0.8) * cam["w"], rng.uniform(0.2, 0.8) * cam["h"]
        out[i][(xx - cx) ** 2 + (yy - cy) ** 2 < (0.15 * cam["h"]) ** 2] = 0
    return out


def layout(frames, how):
    """Frames as `how` passes them: packed host, strided host or strided device (each frame in a buffer with padded rows)."""
    if how == "packed":
        return frames
    pad = np.zeros((len(frames), frames.shape[1], frames.shape[2] + 5) + frames.shape[3:], np.uint8)
    pad[:, :, 3:3 + frames.shape[2]] = frames
    if how == "host_strided":
        return [pad[i, :, 3:3 + frames.shape[2]] for i in range(len(frames))]
    import torch
    dev = torch.from_numpy(pad).cuda()
    return [dev[i, :, 3:3 + frames.shape[2]] for i in range(len(frames))]


def dev_masks(masks):
    """Per-frame masks in device memory, each in a buffer with padded rows (a step > w)."""
    import torch
    pad = torch.zeros((len(masks), masks.shape[1], masks.shape[2] + 7), dtype=torch.uint8, device="cuda")
    pad[:, :, 2:2 + masks.shape[2]] = torch.from_numpy(np.array(masks, np.uint8)).cuda()
    return [pad[i, :, 2:2 + masks.shape[2]] for i in range(len(masks))]


def new_pipeline(cam, kc=False, mirror=1, depth_image=0, imu=None, live=False):
    from rebvo_b200 import capi
    pl = capi.Pipeline(capi.default_params(cam), max_batch=BATCH)
    if kc:
        pl.set_undistort(pu.EUROC_KC)
    if imu is not None:
        ip = capi.default_imu_params(InitBias=1, InitBiasFrameNum=5)
        if live:
            pl.set_imu_live(ip, float(np.mean(np.diff(imu[:, 0]))), len(imu) + 8)
            pl.push_imu(imu)
        else:
            pl.set_imu(imu, ip)
    else:
        if mirror:
            pl.set_mirror(mirror)
        pl.set_depth(capi.depth_params())
        if depth_image:
            pl.set_depth_image(depth_image)
    pl.set_odometry(True)
    return pl


def outputs(pl, nav, mirror, depth_image, imu):
    out = [pu.raw(nav).tobytes(), pu.raw(pl.odometry()).tobytes()]
    for i in range(0 if imu is not None else len(nav)):
        out.append(pl.mirror(i).tobytes() if mirror else None)
        cells, md = pl.depth(i)
        out.append(tuple(np.ascontiguousarray(cells[k]).tobytes() for k in ("rho", "s_rho", "dist", "fixed")) +
                   (np.float64(md).tobytes(),))
        if depth_image:
            r, s = pl.depth_image(i)
            out.append(r.tobytes() + (b"" if s is None else s.tobytes()))
    return out


def run(cam, how="packed", kc=False, fixed=None, per_frame=None, mirror=1, depth_image=0, imu=None, live=False,
        sizes=SIZES, enqueue=0):
    """The stream through one pipeline in pushes of `sizes`: (outputs per push, launches per push, mirror records per
    frame).  fixed: the fixed mask (set before the first push); per_frame: [n, h, w] masks passed per frame."""
    import torch
    ts, fr = stream(cam)
    pl = new_pipeline(cam, kc, mirror, depth_image, imu, live)
    res, launches, mirrors = [], [], []
    try:
        if fixed is not None:
            pl.set_detect_mask(fixed)
        if enqueue:
            pl.set_async(enqueue)
        s, pending = 0, []
        for k, n in enumerate(sizes):
            f, t = layout(fr[s:s + n], how), ts[s:s + n]
            m = None if per_frame is None else dev_masks(per_frame[s:s + n])
            l0 = pl.launches()
            if enqueue:
                pending.append((pl.enqueue(f, t, masks=m), m))
                if len(pending) == enqueue or k == len(sizes) - 1:
                    for tk, _ in pending:
                        nav = pl.wait(tk)
                        res.append(outputs(pl, nav, mirror, depth_image, imu))
                    pending = []
            else:
                if m is not None:
                    nav = pl.push_masked(f, m, t)
                elif how == "packed":
                    nav = pl.push(f, t)
                else:
                    nav = pl.push_frames(f, t)
                torch.cuda.synchronize()
                launches.append(pl.launches() - l0)
                res.append(outputs(pl, nav, mirror, depth_image, imu))
                if mirror == 1 and imu is None:
                    mirrors += [pl.mirror(i).copy() for i in range(len(nav))]
            s += n
    finally:
        pl.close()
    return res, launches, mirrors


def assert_same(a, b, what):
    assert len(a) == len(b), what
    for k, (x, y) in enumerate(zip(a, b)):
        assert x == y, "%s: push %d differs" % (what, k)


def assert_off_zero_bytes(mirrors, keep_of_frame):
    for i, rec in enumerate(mirrors):
        keep = keep_of_frame(i).reshape(-1)
        assert np.all(keep[rec["p_inx"]] != 0), "frame %d has a keyline on a masked pixel" % i


# ---- stage level --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 2, 3, 4])
def test_stage_matches_restatement(built, R):
    from rebvo_b200 import capi
    from test_cpu_front_states import same_detect
    cam = fs.CAM
    ctx = capi.Ctx(cam, fs.SIGMA0, fs.KSIGMA, kl_capacity=50000)
    maps = []
    try:
        frames = []
        for seed in (3, 11, 17):
            m = ctx.new_map()
            maps.append(m)
            m.upload_gray(fs.edge_frame(cam["w"], cam["h"], seed))
            m.dog_build()
            frames.append((m, m.plane("img0"), m.plane("dog")))
        m0, img0, dog = frames[0]
        cand = candidates(img0, dog, R, B["per_hist"], B["dog_thresh"], B["tresh"])
        kl_max = len(cand) // 2
        fam = mask_families(cam["w"], cam["h"], R, cand, kl_max)
        prev = {}
        for name, keep in fam.items():
            # one frame at a fixed threshold, then a chain over the three frames with auto-gain on
            chain = [(0, 0.0)] + [(f, 2e-6) for f in (0, 1, 2, 1)]
            t, l = B["tresh"], 0
            pt, plk = B["tresh"], 0
            for step, (f, gain) in enumerate(chain):
                m, img0, dog = frames[f]
                det = capi.DetectParams(R, B["per_hist"], B["dog_thresh"], kl_max, B["kl_ref"], gain, B["tmax"],
                                        B["tmin"])
                kn, t, l = m.detect_masked(det, keep, t, l)
                d = dict(kn=kn, t=t, l=l, kl=m.keylines(), mask=m.mask(), reest=[])
                pkn, pt, plk, pkl, pmask = port_detect_masked(img0, dog, R, B["per_hist"], B["dog_thresh"], kl_max, pt,
                                                              plk, B["kl_ref"], gain, B["tmax"], B["tmin"], cam["ppx"],
                                                              cam["ppy"], keep, prev.get(f))
                prev[f] = pmask
                same_detect(d, dict(kn=pkn, t=pt, l=plk, kl=pkl, mask=pmask, reest=[]), "%s step %d" % (name, step))
                assert np.all(keep.reshape(-1)[d["kl"]["p_inx"]] != 0), name
        # a NULL mask or a step shorter than a row
        t, l, kn = C.c_double(B["tresh"]), C.c_int(0), C.c_int(0)
        keep = fam["ones"]
        for ptr, step in ((None, cam["w"]), (keep.ctypes.data_as(C.c_void_p), cam["w"] - 1)):
            assert m0.L.rb_map_detect_masked(m0.h_, m0.h_, C.byref(det), ptr, C.c_int64(step), C.byref(t), C.byref(l),
                                             C.byref(kn)) == RB_ERR_ARG
    finally:
        for m in maps:
            m.close()
        ctx.close()


# ---- pipeline ---------------------------------------------------------------------------------------------------------
def test_all_ones_and_complement(built):
    from rebvo_b200 import synth
    cam = synth.EUROC
    n = sum(SIZES)
    base, launches, mirrors = run(cam)
    ones = np.ones((n, cam["h"], cam["w"]), np.uint8)
    assert_same(run(cam, fixed=ones[0])[0], base, "all-ones fixed mask")
    assert_same(run(cam, per_frame=ones)[0], base, "all-ones per-frame masks")
    # zero on every pixel without a keyline in the unmasked run: non-candidates and candidates past the cut masked
    comp = np.zeros_like(ones)
    for i, rec in enumerate(mirrors):
        comp[i].reshape(-1)[rec["p_inx"]] = 1
    assert_same(run(cam, per_frame=comp)[0], base, "complement of the keylines")
    for mode, dimg in ((2, 2),):
        b2 = run(cam, mirror=mode, depth_image=dimg)[0]
        assert_same(run(cam, fixed=ones[0], mirror=mode, depth_image=dimg)[0], b2, "all-ones fixed, mirror 2")
        assert_same(run(cam, per_frame=ones, mirror=mode, depth_image=dimg)[0], b2, "all-ones per frame, mirror 2")


@pytest.mark.parametrize("cam_name,how,kc", [("euroc", "packed", False), ("euroc", "host_strided", False),
                                             ("euroc", "dev_strided", False), ("euroc", "packed", True),
                                             ("euroc", "dev_strided", True), ("kitti", "packed", False),
                                             ("kitti", "dev_strided", False)])
def test_fixed_equals_per_frame(built, cam_name, how, kc):
    from rebvo_b200 import synth
    cam = synth.EUROC if cam_name == "euroc" else KITTI
    n = sum(SIZES)
    F = fixed_mask(cam)
    M = blob_masks(cam, n)
    base = run(cam, how, kc)[0]
    a, _, ma = run(cam, how, kc, fixed=F)
    b, _, _ = run(cam, how, kc, per_frame=np.broadcast_to(F, M.shape))
    assert_same(a, b, "fixed mask vs the same mask per frame")
    assert a != base, "the fixed mask changed nothing"
    assert_off_zero_bytes(ma, lambda i: F)
    c, _, mc = run(cam, how, kc, fixed=F, per_frame=M)
    d, _, _ = run(cam, how, kc, per_frame=(F != 0) & (M != 0))
    assert_same(c, d, "fixed + per-frame masks vs their AND per frame")
    assert_off_zero_bytes(mc, lambda i: (F != 0) & (M[i] != 0))


def test_geometry_matches_restatement(built):
    """Partial per-frame masks over a tracked sequence: each frame's mirror geometry is the masked restatement on that
    frame's planes at the nav record's threshold, and no keyline lies on a zero byte."""
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = stream(cam)
    M = blob_masks(cam, len(ts), seed=3)
    p = capi.default_params(cam)
    pl = new_pipeline(cam)
    try:
        s = 0
        for n in SIZES:
            nav = pl.push_masked(fr[s:s + n], dev_masks(M[s:s + n]), ts[s:s + n])
            for i in range(n):
                img0, dog = pl.batch_plane(i, "img0"), pl.batch_plane(i, "dog")
                kl_max = max(1, min(p.det.kl_max, p.kl_capacity if p.kl_capacity > 0 else 50000))
                want = port_detect_masked(img0, dog, p.det.plane_fit_size, p.det.pos_neg_thresh, p.det.dog_thresh,
                                          kl_max, float(nav[i]["thresh"]), 0, 0, 0.0, 1.0, 0.0, cam["ppx"], cam["ppy"],
                                          M[s + i])
                got = pl.mirror(i)
                assert want[0] == nav[i]["kn"] == len(got), (s + i, want[0], nav[i]["kn"])
                for f in ("p_inx", "c_p", "m_m", "n_id", "p_id"):
                    assert np.array_equal(np.ascontiguousarray(got[f]).view(np.uint8),
                                          np.ascontiguousarray(want[3][f]).view(np.uint8)), (s + i, f)
                assert np.all(M[s + i].reshape(-1)[got["p_inx"]] != 0)
            s += n
    finally:
        pl.close()


@pytest.mark.parametrize("depth", [2, 4])
def test_enqueue_matches_push(built, depth):
    from rebvo_b200 import synth
    cam = synth.EUROC
    n = sum(SIZES)
    F, M = fixed_mask(cam), blob_masks(cam, n, seed=5)
    want = run(cam, "dev_strided", fixed=F, per_frame=M)[0]
    got = run(cam, "dev_strided", fixed=F, per_frame=M, enqueue=depth)[0]
    assert_same(got, want, "masked_enqueue vs push_masked")


@pytest.mark.parametrize("live", [False, True])
def test_imu(built, live):
    from rebvo_b200 import synth
    cam = synth.EUROC
    n = sum(SIZES)
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=21, zf=cam["zfx"])
    imu = synth.imu_samples(seq, n + 2)
    F = fixed_mask(cam)
    a = run(cam, fixed=F, imu=imu, live=live, mirror=0)[0]
    b = run(cam, per_frame=np.broadcast_to(F, (n,) + F.shape), imu=imu, live=live, mirror=0)[0]
    base = run(cam, imu=imu, live=live, mirror=0)[0]
    assert_same(a, b, "IMU mode: fixed vs per frame")
    assert a != base


def test_checkpoint_keeps_the_mask_out(built):
    """save_state -> load_state into a pipeline with the same fixed mask resumes with the uninterrupted run's bytes."""
    from rebvo_b200 import synth
    cam = synth.EUROC
    F = fixed_mask(cam)
    ts, fr = stream(cam)
    whole = run(cam, fixed=F)[0]
    pl = new_pipeline(cam)
    pl.set_detect_mask(F)
    for s, n in ((0, 4), (4, 4)):
        pl.push(fr[s:s + n], ts[s:s + n])
    blob = pl.save_state()
    pl.close()
    pl = new_pipeline(cam)
    try:
        pl.set_detect_mask(F)
        pl.load_state(blob)
        got = []
        for s, n in ((8, 1), (9, 3)):
            got.append(outputs(pl, pl.push(fr[s:s + n], ts[s:s + n]), 1, 0, None))
        assert_same(got, whole[2:], "resumed run")
    finally:
        pl.close()


def test_cleared_mask_launches_and_bytes(built):
    from rebvo_b200 import synth
    cam = synth.EUROC
    F = fixed_mask(cam)
    base, lb, _ = run(cam)
    # set and cleared before the first push: the pipeline of one that never had a mask
    ts, fr = stream(cam)
    res, launches = [], []
    pl = new_pipeline(cam)
    try:
        pl.set_detect_mask(F)
        pl.set_detect_mask(None)
        s = 0
        for n in SIZES:
            l0 = pl.launches()
            nav = pl.push(fr[s:s + n], ts[s:s + n])
            launches.append(pl.launches() - l0)
            res.append(outputs(pl, nav, 1, 0, None))
            s += n
    finally:
        pl.close()
    assert_same(res, base, "mask set and cleared")
    assert launches == lb
    # a masked push and a cleared one launch what an unmasked push of the same size launches
    _, lm, _ = run(cam, fixed=F)
    assert lm == lb


def test_argument_errors(built):
    import torch
    from rebvo_b200 import capi, synth
    cam = synth.EUROC
    ts, fr = stream(cam)
    want = run(cam, sizes=[4, 4])[0]
    pl = new_pipeline(cam)
    L = pl.L
    try:
        nav = np.zeros(4, capi.NAV)
        t = np.ascontiguousarray(ts[:4])
        frames = np.array([(fr[i].ctypes.data, cam["w"] * 3) for i in range(4)], capi.FRAME)
        mk = torch.ones((4, cam["h"], cam["w"]), dtype=torch.uint8, device="cuda")
        good = np.array([(mk[i].data_ptr(), cam["w"]) for i in range(4)], capi.FRAME)
        bad_null = good.copy()
        bad_null[2]["data"] = 0
        bad_step = good.copy()
        bad_step[1]["step"] = cam["w"] - 1
        fp = frames.ctypes.data_as(C.c_void_p)
        for masks in (None, bad_null.ctypes.data_as(C.c_void_p), bad_step.ctypes.data_as(C.c_void_p)):
            assert L.rb_pipeline_push_masked(pl.h_, 0, 0, fp, masks, t.ctypes.data_as(C.c_void_p), 4,
                                             nav.ctypes.data_as(C.c_void_p)) == RB_ERR_ARG
        assert L.rb_pipeline_set_detect_mask(pl.h_, C.c_void_p(mk.data_ptr()), C.c_int64(cam["w"] - 1), 1) == RB_ERR_ARG
        tk = C.c_int64(-1)
        assert L.rb_pipeline_masked_enqueue(pl.h_, 0, 0, fp, good.ctypes.data_as(C.c_void_p),
                                            t.ctypes.data_as(C.c_void_p), 4, C.byref(tk)) == RB_ERR_ARG   # async off
        got = [outputs(pl, pl.push(fr[0:4], ts[0:4]), 1, 0, None)]
        pl.set_async(2)
        k = pl.enqueue(fr[4:8], ts[4:8])
        assert L.rb_pipeline_set_detect_mask(pl.h_, None, C.c_int64(0), 0) == RB_ERR_STATE
        got.append(outputs(pl, pl.wait(k), 1, 0, None))
        assert_same(got, want, "pushes after refused calls")
    finally:
        pl.close()
    imu_pl = new_pipeline(cam, imu=synth.imu_samples(synth.Sequence(w=cam["w"], h=cam["h"], seed=21, zf=cam["zfx"]), 4))
    try:
        tk = C.c_int64(-1)
        assert imu_pl.L.rb_pipeline_masked_enqueue(imu_pl.h_, 0, 0, frames.ctypes.data_as(C.c_void_p),
                                                   good.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p), 4,
                                                   C.byref(tk)) == RB_ERR_ARG
    finally:
        imu_pl.close()

"""States of the front of the frame: the undistortion maps, frames and expected planes that the ingress tests
(tests/test_cpu_ingress_states.py, tests/test_gpu_ingress.py) run on.

- undistort_map restates image_undistort's map (rb_undistort_create) in NumPy, with the reference's float / double mix and
  its `(unsigned)(long long)` bound test; apply_map applies it in integer arithmetic as biInterp does.
- MAPS are the (camera, kc) cases, each with the minimum reach (reach()) it is built for.
- frame() makes the seeded frames: random bytes, frames with edges, and an all-255 frame.
- expected() is the reference's undistort_rgb -> rgb2bw -> sspace::build planes of one (camera, kc, sigma0, frame), cached for
  the process.  A mono frame stands for the replicated RGB24 frame, so its planes are those of that frame.
- INSTANCES mirrors rb_gray_enqueue's dispatch (gray.cu): which kernel instance a push runs.

Nothing here needs a GPU; the reference is imported only by expected() and ref_undistort()."""
import functools

import numpy as np

EUROC = dict(w=752, h=480, zfx=458.654, zfy=457.296, ppx=367.215, ppy=248.375)
# EuRoC cam0 (GlobalConfig_EuRoC_2.txt:64-68) and the mild rad-tan model test_gpu_frames.py uses for the KITTI sizes
EUROC_KC = (-0.28340811, 0.07395907, 0.0, 0.00019359, 1.76187114e-05)
KC = (-0.12, 0.03, 0.0, 1e-4, 2e-5)
SIGMAS = (1.7818, 3.56359)   # the two box plans: 3/3/5 + 3/5/5 and 7/7/7 + 9/9/9
KSIGMA = 1.2599


def kitti(w, h):
    return dict(w=w, h=h, zfx=718.856, zfy=718.856, ppx=w / 2.0 - 13.3, ppy=h / 2.0 - 2.8)


CAMS = {
    "752x480": EUROC,
    "1241x376": kitti(1241, 376),
    "1226x370": kitti(1226, 370),
    "1239x375": kitti(1239, 375),   # w % 4 == 3, N odd: every frame after the first starts at an odd byte
    "640x480": dict(w=640, h=480, zfx=525.0, zfy=525.0, ppx=320.0, ppy=240.0),
    "1280x960": dict(w=1280, h=960, zfx=1100.0, zfy=1098.5, ppx=652.25, ppy=471.75),
}


def cam_variant(name, **over):
    c = dict(CAMS[name])
    c.update(over)
    return c


# (camera, kc, reach): reach names a minimum count of reach() that the case is built to meet.  kc = 0 turns the pipeline's
# undistortion off, so the kc = 0 cases run on the standalone rb_undistort only (pipeline=False).
MAPS = {
    # the cameras' own barrel models: every source inside the frame, 4 taps, a pair everywhere
    "euroc": dict(cam=CAMS["752x480"], kc=EUROC_KC, reach=dict(taps4=360960, zero_weight=100)),
    "kitti1241": dict(cam=CAMS["1241x376"], kc=KC, reach=dict(taps4=466616, zero_weight=1000, exact_one=10)),
    "kitti1226": dict(cam=CAMS["1226x370"], kc=KC, reach=dict(taps4=453620, zero_weight=1000, exact_one=10)),
    "kitti1239": dict(cam=CAMS["1239x375"], kc=KC, reach=dict(taps4=464625, zero_weight=1000, exact_one=10)),
    # a strong pincushion: the corners' sources fall outside the frame (0 taps), the borders' on the last row / column
    "pincushion640": dict(cam=CAMS["640x480"], kc=(0.35, 0.25, 0.0, 1e-3, -1e-3),
                          reach=dict(taps0=5000, taps1=1, taps2=100, taps4=200000, last_rows=100, rgb_clamp=1)),
    # the principal point far off centre: one side's sources fall outside the frame
    "offcentre1280": dict(cam=cam_variant("1280x960", ppx=300.0, ppy=800.0), kc=(0.06, 0.02, 0.0, 2e-4, -1e-4),
                          reach=dict(taps0=5000, taps1=1, taps2=100, taps4=500000)),
    "hd1280": dict(cam=CAMS["1280x960"], kc=(0.08, -0.01, 0.0, -1e-4, 1e-4),
                   reach=dict(taps4=1000000, taps2=100, last_rows=100)),
    # principal point on integers and on x.5, a weak distortion whose sources sweep the last rows and the corners
    "pp_int": dict(cam=cam_variant("640x480", ppx=320.0, ppy=240.0), kc=(2e-3, 0.0, 0.0, 0.0, 0.0),
                   reach=dict(taps4=250000, last_rows=100, rgb_clamp=1, tap0=1, tapN=1)),
    "pp_half": dict(cam=cam_variant("640x480", ppx=319.5, ppy=239.5), kc=(2e-3, 0.0, 0.0, 0.0, 0.0),
                    reach=dict(taps4=250000, last_rows=100, rgb_clamp=1, tap0=1, tapN=1)),
    "pp_int1239": dict(cam=cam_variant("1239x375", ppx=619.0, ppy=187.0), kc=(1e-3, 0.0, 0.0, 0.0, 0.0),
                       reach=dict(taps4=400000, last_rows=100, rgb_clamp=1, tap0=1, tapN=1)),
    # kc = 0: the identity (x - ppx + ppx == x in float, also at x.5), so the weights are exactly (1, 0, 0, 0) and the
    # zero-weight taps still count
    "kc0_int": dict(cam=cam_variant("640x480", ppx=320.0, ppy=240.0), kc=(0.0,) * 5, pipeline=False,
                    reach=dict(exact_one=300000, zero_weight=900000, last_rows=100, rgb_clamp=1, tap0=1, tapN=1, taps1=1)),
    "kc0_half": dict(cam=cam_variant("640x480", ppx=319.5, ppy=239.5), kc=(0.0,) * 5, pipeline=False,
                     reach=dict(exact_one=300000, zero_weight=900000, last_rows=100, rgb_clamp=1, tap0=1, tapN=1, taps1=1)),
}


def undistort_map(cam, kc):
    """image_undistort::image_undistort (image_undistort.cpp:29-94) on (cam, kc): per pixel o = y*w + x the tap count num,
    the source indices inx[4] and the 16.16 weights iw[4] of its valid taps in the order p00, p01, p10, p11, the unused
    ones 0 (as rb_undistort_create lays them out)."""
    f32, f64 = np.float32, np.float64
    w, h = int(cam["w"]), int(cam["h"])
    ppx, ppy, zfx, zfy = f32(cam["ppx"]), f32(cam["ppy"]), f32(cam["zfx"]), f32(cam["zfy"])
    zfm = f64(f32(zfx + zfy) / f32(2))   # cam_model: zfm((focal_dist.x + focal_dist.y) / 2), float arithmetic
    Kc2, Kc4, Kc6, P1, P2 = (f64(k) for k in kc)
    y, x = np.mgrid[0:h, 0:w]
    qx = x.astype(f32) - ppx                  # Img2Hom in float
    qy = y.astype(f32) - ppy
    xp, yp = qx.astype(f64) / zfm, qy.astype(f64) / zfm   # distortHom2Hom in double
    r2 = xp * xp + yp * yp
    xpp = xp * (1 + r2 * (Kc2 + r2 * (Kc4 + r2 * Kc6))) + 2 * P1 * xp * yp + P2 * (r2 + 2 * xp * xp)
    ypp = yp * (1 + r2 * (Kc2 + r2 * (Kc4 + r2 * Kc6))) + P1 * (r2 + 2 * yp * yp) + 2 * P2 * xp * yp
    idx = (xpp * f64(zfx)).astype(f32) + ppx  # back into the float point, Hom2Img in float
    idy = (ypp * f64(zfy)).astype(f32) + ppy
    assert np.all(np.abs(idx) < 2 ** 31) and np.all(np.abs(idy) < 2 ** 31), "sources beyond the int range"
    p00x, p00y = np.floor(idx), np.floor(idy)
    p11x, p11y = p00x + f32(1), p00y + f32(1)

    def valid(fx, fy):   # Image::isInxValid(const uint &, const uint &) of a float: through a 64-bit truncation
        ux = fx.astype(np.int64) & 0xffffffff
        uy = fy.astype(np.int64) & 0xffffffff
        return (ux < w) & (uy < h)

    taps = [(p00x, p00y, (p11x - idx) * (p11y - idy)), (p11x, p00y, (idx - p00x) * (p11y - idy)),
            (p00x, p11y, (p11x - idx) * (idy - p00y)), (p11x, p11y, (idx - p00x) * (idy - p00y))]
    ok = np.stack([valid(tx, ty) for tx, ty, _ in taps], -1).reshape(-1, 4)
    ind = np.stack([np.round(ty).astype(np.int64) * w + np.round(tx).astype(np.int64) for tx, ty, _ in taps], -1)
    ind = ind.reshape(-1, 4)
    wgt = np.stack([t[2] for t in taps], -1).reshape(-1, 4).astype(f32)
    sum_w = np.zeros(len(wgt), f32)
    for k in range(4):
        sum_w = np.where(ok[:, k], sum_w + wgt[:, k], sum_w).astype(f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        iw_all = ((wgt / sum_w[:, None]).astype(f32) * f32(1 << 16)).astype(f32)
    iw_all = np.where(ok, np.trunc(np.nan_to_num(iw_all)), 0).astype(np.int64)
    assert np.all(ind[ok] >= 0) and np.all(ind[ok] < w * h)
    order = np.argsort(~ok, axis=1, kind="stable")   # the valid taps first, in their order
    num = ok.sum(1)
    inx = np.take_along_axis(np.where(ok, ind, 0), order, 1)
    iw = np.take_along_axis(iw_all, order, 1)
    return num.astype(np.int32), inx.astype(np.int64), iw.astype(np.int64)


def apply_map(m, rgb):
    """biInterp(Image<RGB24Pixel>&) (image_undistort.h:63-78) of every pixel: the integer sums >> 16, as u8."""
    num, inx, iw = m
    h, w = rgb.shape[:2]
    src = rgb.reshape(-1, 3).astype(np.int64)
    acc = np.zeros((len(num), 3), np.int64)
    for k in range(4):
        acc += iw[:, k:k + 1] * src[inx[:, k]]
    return ((acc >> 16) & 0xff).astype(np.uint8).reshape(h, w, 3)


def reach(m, cam):
    """What a map reaches, as counts of output pixels (tap phases: of both rows of a pair)."""
    num, inx, iw = m
    w, h = cam["w"], cam["h"]
    N = w * h
    pair = (inx[:, 1] == inx[:, 0] + 1) & (inx[:, 3] == inx[:, 2] + 1)
    both = np.concatenate([inx[pair, 0], inx[pair, 2]])
    last_word = (3 * N - 1) >> 2
    validtap = np.arange(4)[None, :] < num[:, None]
    out = {"taps%d" % k: int((num == k).sum()) for k in range(5)}
    out.update(
        pair=int(pair.sum()), nonpair=int((~pair).sum()),
        last_rows=int((pair & (inx[:, 2] >= N - w)).sum()),                        # the bottom run on row h-1
        rgb_clamp=int((pair & (((3 * inx[:, 2]) >> 2) + 2 > last_word)).sum()),  # ug_pixel's last_word clamp taken
        tap0=int((validtap & (inx == 0)).any(1).sum()), tapN=int((validtap & (inx == N - 1)).any(1).sum()),
        zero_weight=int((validtap & (iw == 0)).sum()),
        exact_one=int(((num == 4) & (iw[:, 0] == 1 << 16) & (iw[:, 1:] == 0).all(1)).sum()),
        **{"rgb_phase%d" % k: int(((3 * both) % 4 == k).sum()) for k in range(4)},
        **{"mono_phase%d" % k: int((both % 4 == k).sum()) for k in range(4)})
    return out


@functools.lru_cache(maxsize=None)
def map_of(name):
    c = MAPS[name]
    return undistort_map(c["cam"], c["kc"])


def ref_undistort(cam, kc, rgb):
    from oracle import refapi
    return refapi.undistort_rgb(cam, kc, rgb)


# ---- frames -----------------------------------------------------------------------------------------------------------
def frame(cam, key):
    """An RGB24 frame (h, w, 3) of `cam`.  key: ("rand", seed) random bytes, ("edge", seed) random bytes darkened off a
    corner (an edge, so that the planes are not just noise, as test_gpu_scalespace_edges.py), ("mono", seed) random gray
    bytes replicated into three channels, ("white",) every byte 255 (the integral reaches 765 N)."""
    w, h = cam["w"], cam["h"]
    if key[0] == "white":
        return np.full((h, w, 3), 255, np.uint8)
    rng = np.random.default_rng(1000 + key[1])
    if key[0] == "mono":
        return np.repeat(rng.integers(0, 256, (h, w, 1), dtype=np.uint8), 3, axis=2)
    rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if key[0] == "edge":
        rgb[h // 3:, w // 4:] //= 3
    return rgb


def frames(cam, keys, mono=False):
    """The frames of `keys` stacked: RGB24 (n, h, w, 3), or mono (n, h, w) -- first channel of a ("mono", seed) frame."""
    out = np.stack([frame(cam, k) for k in keys])
    return out[..., 0].copy() if mono else out


def _ck(cam):
    return tuple(sorted((k, float(v)) for k, v in cam.items()))


@functools.lru_cache(maxsize=None)
def _expected(cam_key, kc, sigma0, key):
    from oracle import refapi
    cam = dict(cam_key)
    cam["w"], cam["h"] = int(cam["w"]), int(cam["h"])
    rgb = frame(cam, key)
    if kc is not None:
        rgb = refapi.undistort_rgb(cam, kc, rgb)
    r = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], sigma0, KSIGMA)
    r.rgb2bw(rgb)
    r.build()
    return {p: r.plane(p).copy() for p in ("gray", "img0", "dog")}


def expected(cam, kc, sigma0, key):
    """The reference's planes of frame(cam, key): image_undistort (kc not None) -> rgb2bw -> sspace::build (cached)."""
    return _expected(_ck(cam), None if kc is None else tuple(float(k) for k in kc), float(sigma0), tuple(key))


# ---- rb_gray_enqueue's dispatch ---------------------------------------------------------------------------------------
def instance(w, und, mono, strided, nimg):
    """The kernel instance rb_gray_enqueue (gray.cu) runs for a batch: ("k_gray", MONO, L) or ("k_undistort_gray", IMGS,
    MONO, L), L one of ALIGNED, ANYW, STRIDED."""
    layout = "STRIDED" if strided else ("ALIGNED" if w % 4 == 0 else "ANYW")
    if not und:
        return ("k_gray", bool(mono), layout)
    return ("k_undistort_gray", 4 if nimg >= 4 else 1, bool(mono), layout)


INSTANCES = {("k_gray", m, l) for m in (False, True) for l in ("ALIGNED", "ANYW", "STRIDED")} | \
            {("k_undistort_gray", i, m, l) for i in (1, 4) for m in (False, True) for l in ("ALIGNED", "ANYW", "STRIDED")}


# ---- the pipeline cases of tests/test_gpu_ingress.py ------------------------------------------------------------------
# how: "host" packed host frames (rb_pipeline_push / _mono), "dev" packed device frames at byte offset offsets[k % len] of
# an aligned allocation (push_dev / push_mono_dev), "shost" / "sdev" strided host / device frames, one buffer per frame at
# byte offset i % 4 with the row steps of test_gpu_frames.py.  m: "rgb" or "mono".  und: a MAPS name or None.  sizes: the
# pushes, in order (the first push runs eagerly, the next ones of a size capture and replay the batch's graph).  B: max_batch.
# sub: REBVO_B200_SUB (host pushes of n >= 3 sub frames are cut into a head of sub frames and the rest; default 8).
def _case(id, cam, how, sizes, B=64, m="rgb", und=None, offsets=(0,), sub=None, sigma=3.56359, imu=False, white=False):
    return dict(id=id, cam=cam, how=how, sizes=tuple(sizes), B=B, m=m, und=und, offsets=tuple(offsets), sub=sub,
                sigma=sigma, imu=imu, white=white)


CASES = [
    # the gray pass without undistortion: k_gray<MONO, L>
    _case("gray_rgb_aligned_host", "752x480", "host", (1, 2, 3, 3, 2)),
    _case("gray_rgb_aligned_dev_unaligned", "752x480", "dev", (4, 4, 4, 4, 5, 5), offsets=(0, 1, 2, 3, 1, 3)),
    _case("gray_rgb_aligned_dev_640", "640x480", "dev", (3, 3, 3), B=3, offsets=(3, 1, 2)),
    _case("gray_rgb_aligned_dev_1280", "1280x960", "dev", (2, 2), offsets=(2, 1)),
    _case("gray_mono_aligned_host", "752x480", "host", (5, 7, 8, 8), B=8, m="mono"),
    _case("gray_mono_aligned_dev", "1280x960", "dev", (2, 2), m="mono"),
    _case("gray_rgb_anyw_host_sub", "1239x375", "host", (17, 17, 31), sub=5),
    _case("gray_mono_anyw_host_sub", "1239x375", "host", (16, 16), B=16, m="mono", sub=5),
    _case("gray_rgb_anyw_dev", "1241x376", "dev", (3, 3, 3, 3, 31), offsets=(0, 1, 2, 3, 1)),
    _case("gray_mono_anyw_dev", "1226x370", "dev", (7, 7), B=7, m="mono"),
    _case("gray_rgb_strided_dev", "1226x370", "sdev", (5, 5, 2)),
    _case("gray_mono_strided_dev", "752x480", "sdev", (1, 8, 8), m="mono"),
    _case("gray_rgb_strided_host", "1241x376", "shost", (4, 4)),
    # the fused undistortion: k_undistort_gray<IMGS, MONO, L>
    _case("und_rgb_aligned_host", "752x480", "host", (1, 3, 4, 5, 5), und="euroc"),
    _case("und_rgb_aligned_dev", "640x480", "dev", (2, 7, 7, 8, 8), B=8, und="pincushion640", offsets=(0, 1, 2, 3, 2)),
    _case("und_mono_aligned_host", "1280x960", "host", (2, 2, 4, 8), m="mono", und="hd1280"),
    _case("und_mono_aligned_dev", "640x480", "dev", (3, 5, 5), B=5, m="mono", und="pp_half"),
    _case("und_rgb_anyw_host_sub", "1239x375", "host", (2, 17, 17), und="kitti1239", sub=5),
    _case("und_rgb_anyw_dev", "1239x375", "dev", (3, 3, 4, 4), und="pp_int1239", offsets=(1, 2, 3, 0)),
    _case("und_mono_anyw_host", "1241x376", "host", (1, 2, 7, 7), m="mono", und="kitti1241"),
    _case("und_mono_anyw_dev", "1226x370", "dev", (3, 4, 4), B=4, m="mono", und="kitti1226"),
    _case("und_rgb_strided_dev", "1226x370", "sdev", (2, 5, 5), und="kitti1226"),
    _case("und_mono_strided_dev", "1280x960", "sdev", (1, 4, 4), m="mono", und="offcentre1280"),
    _case("und_rgb_strided_host", "752x480", "shost", (3, 8), und="euroc"),
    _case("und_rgb_640_int", "640x480", "dev", (2, 2), und="pp_int", offsets=(1, 3)),
    # IMU mode (imu_flow.cuh's gray call), a device buffer at an odd byte, w % 4 == 0, without undistortion
    _case("imu_rgb_dev_unaligned", "752x480", "dev", (4, 4), B=8, offsets=(1, 3), imu=True),
] + [
    # the batched scale space at m = 1, 2, 5, 64 in a 64-frame workspace (device pushes: one sub-batch), both box plans;
    # the all-255 frame at the last slot of the 64-frame batch
    _case("sspace_%s_s%.2f" % (cam, s), cam, "dev", (1, 2, 5, 64), sigma=s, white=True)
    for cam in ("752x480", "1241x376", "1239x375", "1280x960") for s in SIGMAS
]

POOL = 5   # frame i of a case is pool frame i % POOL: neighbours in a batch always differ


def case_keys(case, first, n):
    """The frame keys of frames first .. first+n-1 of a case; with `white`, the last frame of a 64-frame push is all 255."""
    keys = []
    for i in range(first, first + n):
        if case["m"] == "mono":
            keys.append(("mono", i % POOL))
        else:
            keys.append(("rand", i % POOL) if i % POOL < 3 else ("edge", i % POOL))
    if case["white"] and n == 64:
        keys[-1] = ("white",)
    return keys


def sub_batches(case, n):
    """The scale-space batches of one push of n frames (push_impl): a host push of n >= 3 sub frames is a head of sub
    frames and the rest; every other push is one batch."""
    sub = case["sub"] or 8
    if case["how"] in ("host", "shost") and not case["imu"] and n >= 3 * sub:
        return [sub, n - sub]
    return [n]


def case_instances(case):
    """The kernel instances the case's pushes run (rb_gray_enqueue's dispatch)."""
    w = CAMS[case["cam"]]["w"]
    out = set()
    for n in case["sizes"]:
        for nb in sub_batches(case, n):
            out.add(instance(w, case["und"] is not None, case["m"] == "mono", case["how"] == "sdev", nb))
    return out


def case_cam(case):
    """The camera of a case: its undistortion map's (same size, that map's principal point), or CAMS[cam]."""
    if case["und"] is None:
        return CAMS[case["cam"]]
    c = MAPS[case["und"]]["cam"]
    assert (c["w"], c["h"]) == (CAMS[case["cam"]]["w"], CAMS[case["cam"]]["h"])
    return c


def case_kc(case):
    return None if case["und"] is None else MAPS[case["und"]]["kc"]

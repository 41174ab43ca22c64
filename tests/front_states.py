"""The front end of every frame on crafted states: the detector (UpdateThresh + build_mask + join_edges,
edge_finder.cpp:67-365), reEstimateThresh (:373-405) and build_field (global_tracker.cpp:61-105).

The states are deterministic: gray frames from seeded generators (step edges and thin lines at 0, 45, 90, 135 degrees and
at arbitrary angles, rings), and thresholds picked from the reference's own Img(0) / DoG planes so that pixels sit exactly
on each of build_mask's four comparisons.  Every state is a job that three executors run the same way:
  - the reference (oracle/refapi.py) in this process for R = 2, or in a child process for the other window sizes
    (build_mask caches its pseudo inverse per process, edge_finder.cpp:83-84): `python tests/front_states.py in out`;
  - the NumPy restatement (plane_fit.port_detect, port_reestimate and port_field below);
  - the device (rebvo_b200.capi).
`reach` counts, on the restatement's intermediates, what each state reaches: pixels exactly on each comparison, keylines
per NextPoint quadrant and probe, p_id collisions, where the kl_max cut falls, controller clamps and field ties."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (HERE, ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)
from plane_fit import (MAX_IMG_VALUE, detect_terms, detect_tests, keyline_dtype, port_detect, ref_child,  # noqa: E402
                       run_ref_job)

SIGMA0, KSIGMA = 1.7818, 1.2599
# 331 = 10 * 32 + 11: every row ends in a partial 32-pixel chunk; 11 segments a row, 2200 in all, so each k_seg_scan
# thread scans per = 3 segments
CAM = dict(w=331, h=200, zfx=260.0, zfy=258.0, ppx=165.3, ppy=99.75)
# the KITTI width: 39 chunks a row, the last one 25 pixels wide; per = 15
CAM_K = dict(w=1241, h=376, zfx=718.856, zfy=718.856, ppx=607.1928, ppy=185.2157)
BASE = dict(per_hist=0.4, dog_thresh=0.095259868922420, tresh=0.01, kl_ref=1500, gain=0.0, tmax=0.5, tmin=0.005)


# ---- frames ----------------------------------------------------------------------------------------------------------
def edge_frame(w, h, seed, contrast=1.0, tile=36):
    """Gray float32 [h, w]: one feature per tile -- a step edge, a thin line or a ring -- at 0, 45, 90, 135 degrees or a
    seeded angle, with a seeded sub-pixel offset, width and contrast.  Axis-aligned features have exactly constant rows
    or columns, so their DoG gradient has an exactly zero component."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    g = np.full((h, w), 128.0)
    for ty in range(0, h, tile):
        for tx in range(0, w, tile):
            sl = (slice(ty, min(ty + tile, h)), slice(tx, min(tx + tile, w)))
            kind = int(rng.integers(3))
            a = [0.0, 45.0, 90.0, 135.0, float(rng.uniform(0, 180))][int(rng.integers(5))]
            n = {0.0: (1.0, 0.0), 90.0: (0.0, 1.0)}.get(a, (np.cos(np.radians(a)), np.sin(np.radians(a))))
            cx = tx + tile / 2 + float(rng.integers(-6, 7)) * 0.5 + (0.0 if rng.random() < 0.5 else rng.uniform(0, 1))
            cy = ty + tile / 2 + float(rng.integers(-6, 7)) * 0.5 + (0.0 if rng.random() < 0.5 else rng.uniform(0, 1))
            s = float(rng.uniform(0.6, 2.5))
            amp = float(rng.uniform(30, 110)) * contrast * (1 if rng.random() < 0.5 else -1)
            X, Y = xx[sl] - cx, yy[sl] - cy
            if kind == 0:
                v = np.tanh((n[0] * X + n[1] * Y) / s)
            elif kind == 1:
                v = 2.0 * np.exp(-((n[0] * X + n[1] * Y) / s) ** 2) - 1.0
            else:
                v = np.tanh((np.hypot(X, Y) - rng.uniform(5, tile / 2 - 2)) / s)
            g[sl] = 128.0 + amp * v
    return g.astype(np.float32)


def ref_planes(cam, gray):
    """(img0, dog) of the reference's scale space on a gray plane (independent of the window size)."""
    from oracle import refapi
    m = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], SIGMA0, KSIGMA)
    m.set_gray(gray)
    m.build()
    return m.plane("img0"), m.plane("dog")


# ---- thresholds on a comparison ---------------------------------------------------------------------------------------
def _f32(x):
    return np.float32(x)


def _near(x, k=4):
    x = _f32(x)
    out = [x]
    up = dn = x
    for _ in range(k):
        up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(-np.inf))
        out += [up, dn]
    return out


def solve_square(v, a):
    """A float32 x with fl(fl(x * a)^2) == v (a, v float32), or None: the threshold whose squared bound is exactly v."""
    v, a = _f32(v), _f32(a)
    for t in _near(np.sqrt(np.float64(v))):
        if t * t != v:
            continue
        for x in _near(np.float64(t) / np.float64(a)):
            if x * a == t:
                return x
    return None


def _next_bound(v, solve, d):
    """The threshold of the bound nearest to v on side d (-inf / +inf) that a float32 threshold can reach: one ulp from v
    where the squares allow it, a few ulps otherwise."""
    for _ in range(8):
        v = np.nextafter(v, np.float32(d))
        x = solve(v)
        if x is not None:
            return x
    raise AssertionError("no float32 bound near %r" % v)


def _ulp_states(values, decisive, solve):
    """The value v among `values` with the most decisive pixels that a bound can be placed on, and the bounds next to it:
    {"at": x, "below": x, "above": x} (bound == v, just below v, just above v)."""
    vals, counts = np.unique(values[decisive], return_counts=True)
    for i in np.argsort(-counts, kind="stable")[:400]:
        v = vals[i]
        x = solve(v)
        if x is not None:
            return dict(at=x, below=_next_bound(v, solve, -np.inf), above=_next_bound(v, solve, np.inf)), int(counts[i])
    raise AssertionError("no value can be placed on a float32 bound")


def pick_grad(T, R, base):
    """DetectorThresh values whose (t1)^2 = (DetectorThresh * 765)^2 equals, is 1 ulp below and 1 ulp above the n2gI of
    pixels that pass the other three tests."""
    P = detect_tests(T, R, base["per_hist"], 0.02, base["tresh"])
    ok = P["pn"] & P["sub"] & P["dog"] & (T["n2gI"] > _f32(2e3)) & (T["n2gI"] < _f32(1e5))
    xs, _ = _ulp_states(T["n2gI"], ok, lambda v: solve_square(v, MAX_IMG_VALUE))
    return {k: float(x) for k, x in xs.items()}


def pick_dog(T, R, base):
    """dog_thresh values whose (t1 * dog_thresh)^2 equals, is 1 ulp below and 1 ulp above the n2_m of pixels that pass
    the other three tests."""
    P = detect_tests(T, R, base["per_hist"], base["dog_thresh"], base["tresh"])
    t1 = _f32(base["tresh"]) * MAX_IMG_VALUE
    xs, _ = _ulp_states(T["n2_m"], P["grad"] & P["pn"] & P["sub"], lambda v: solve_square(v, t1))
    return {k: float(x) for k, x in xs.items()}


def pick_pos_neg(T, R, base):
    """per_hist = k / (2R+1)^2 with float((2R+1)^2) * per_hist == k exactly, for the k with the most pixels at |pn| = k
    that pass the other tests."""
    n2 = (2 * R + 1) ** 2
    P = detect_tests(T, R, base["per_hist"], base["dog_thresh"], base["tresh"])
    ok = P["grad"] & P["sub"] & P["dog"]
    best = None
    for k in range(1, n2, 2):
        for ph in _near(k / n2, 2):
            if _f32(n2) * ph == _f32(k):
                c = int((ok & (np.abs(T["pn"]) == k)).sum())
                if best is None or c > best[0]:
                    best = (c, float(ph))
                break
    return best[1]


# ---- what the restatement reaches -------------------------------------------------------------------------------------
def boundary_counts(T, R, st):
    """Pixels exactly on each comparison that pass the other three tests, i.e. whose candidacy the comparison decides."""
    P = detect_tests(T, R, st["per_hist"], st["dog_thresh"], st["tresh"])
    on = dict(grad=T["n2gI"] == P["t1sq"], pn=np.abs(T["pn"]).astype(np.float64) == np.float64(P["lim"]),
              sub=(np.abs(T["xsub"]) == 0.5) | (np.abs(T["ysub"]) == 0.5), dog=T["n2_m"] == P["t5sq"])
    out = {}
    for k in on:
        others = np.ones(len(T["pn"]), bool)
        for j in on:
            if j != k:
                others &= P[j]
        out[k + "_on"] = int((on[k] & others).sum())
    # pixels within 8 float ulps of the squared bounds (the states with the bound just below / above a value)
    for k, v, b in (("grad", T["n2gI"], P["t1sq"]), ("dog", T["n2_m"], P["t5sq"])):
        others = np.ones(len(T["pn"]), bool)
        for j in on:
            if j != k:
                others &= P[j]
        d = np.abs(v.view(np.int32).astype(np.int64) - int(np.float32(b).view(np.int32)))
        out[k + "_near"] = int(((d >= 1) & (d <= 8) & others).sum())
    out["xs_nan"] = int((np.isnan(T["xsub"]) | np.isnan(T["ysub"])).sum())
    return out


def join_counts(kl, mask):
    """Keylines per NextPoint quadrant and first successful probe, zero tangent components, x.5 positions and p_id
    collisions (join_edges, edge_finder.cpp:221-320)."""
    h, w = mask.shape
    out = {}
    if len(kl) == 0:
        return out
    m = kl["m_m"]
    tx, ty = -m[:, 1], m[:, 0]
    q = np.where(ty > 0, np.where(tx > 0, 0, 1), np.where(tx < 0, 2, 3))
    x = (kl["c_p"][:, 0].astype(np.float64) + 0.5).astype(np.int64)
    y = (kl["c_p"][:, 1].astype(np.float64) + 0.5).astype(np.int64)
    sx = np.where(ty > 0, np.where(tx > 0, 1, -1), np.where(tx < 0, -1, 1))
    sy = np.where(ty > 0, 1, -1)
    flat = mask.reshape(-1)
    probe = np.full(len(kl), 3)
    for k, (px, py) in enumerate(((x + sx, y), (x, y + sy), (x + sx, y + sy))):
        pi = py * w + px
        inside = (pi >= 0) & (pi < h * w)
        v = np.where(inside, flat[np.where(inside, pi, 0)], -1)
        probe = np.where((probe == 3) & (v >= 0), k, probe)
    for a in range(4):
        for b in range(4):
            out["q%d_p%d" % (a, b)] = int(((q == a) & (probe == b)).sum())
    out["tx_zero"] = int((tx == 0).sum())
    out["ty_zero"] = int((ty == 0).sum())
    out["neg_zero"] = int(((tx == 0) & np.signbit(tx)).sum() + ((ty == 0) & np.signbit(ty)).sum())
    out["c_p_half"] = int((np.modf(kl["c_p"])[0] == 0.5).sum())
    nid = kl["n_id"][kl["n_id"] >= 0]
    out["p_id_collisions"] = int((np.bincount(nid, minlength=len(kl)) >= 2).sum())
    return out


def cut_position(cam, R, cand_idx, kl_max):
    """(lane, segment, scan thread, first / last segment of that thread's range, last chunk of the row) of the last
    keyline the cut keeps, or None when nothing is cut."""
    w, h = cam["w"], cam["h"]
    kl_max = max(kl_max, 1)
    if len(cand_idx) < kl_max:
        return None
    p = int(cand_idx[kl_max - 1])
    x, y = p % w, p // w
    nchunk = (w + 31) // 32
    per = (h * nchunk + 1023) // 1024
    seg = y * nchunk + x // 32
    return dict(lane=x % 32, seg=seg, thread=seg // per, thread_first=seg % per == 0,
                thread_last=seg % per == per - 1, last_chunk=x // 32 == nchunk - 1)


# ---- jobs -------------------------------------------------------------------------------------------------------------
def _step(**kw):
    s = dict(BASE, kl_max=40000, prior=None, reest=[])
    s.update(kw)
    return s


def _cand(T, R, st):
    P = detect_tests(T, R, st["per_hist"], st["dog_thresh"], st["tresh"])
    return np.nonzero(P["grad"] & P["pn"] & P["sub"] & P["dog"])[0]


def detect_jobs(R):
    """Every detect state at window size R: a list of jobs {name, cam, kcap, grays, planes, steps, want}.  A job runs its
    steps in order with the threshold chained (tresh, l_kl_num); step `f` names the frame (one edge map per frame, reused
    by later steps on it); `prior` = (keylines, mask) loaded before the detect; `reest` = (knum, nbins) calls after it;
    `want` = minimum reach counts."""
    jobs = []
    g0 = edge_frame(CAM["w"], CAM["h"], 100 + R)
    g1 = edge_frame(CAM["w"], CAM["h"], 200 + R, tile=24)
    gflat = edge_frame(CAM["w"], CAM["h"], 300 + R, contrast=0.04)
    pl0, pl1, plf = ref_planes(CAM, g0), ref_planes(CAM, g1), ref_planes(CAM, gflat)
    T0 = detect_terms(*pl0, R)

    def job(name, steps, want, grays=(g0,), planes=(pl0,), cam=CAM, kcap=50000, fixed=None):
        assert want, name   # every state names what it must reach
        jobs.append(dict(name="R%d_%s" % (R, name), R=R, cam=cam, sigma0=SIGMA0, ksigma=KSIGMA, kcap=kcap,
                         grays=list(grays), planes=list(planes), steps=steps, want=want, fixed=fixed or {},
                         t0=steps[0]["tresh"]))

    # the four comparisons: on the bound, and the bound one float ulp to either side
    for k, tr in pick_grad(T0, R, BASE).items():
        job("grad_" + k, [_step(tresh=tr, dog_thresh=0.02)], {"grad_on": 1} if k == "at" else {"grad_near": 1})
    for k, dt in pick_dog(T0, R, BASE).items():
        job("dog_" + k, [_step(dog_thresh=dt)], {"dog_on": 1} if k == "at" else {"dog_near": 1})
    ph = pick_pos_neg(T0, R, BASE)
    job("pos_neg_on", [_step(per_hist=ph)], {"pn_on": 5})
    job("pos_neg_zero", [_step(per_hist=0.0)], {"empty": 1})
    # a black corner: there the DoG window is exactly 0, theta0 = theta1 = 0 and xs = NaN passes the sub-pixel test;
    # the gradient test rejects those pixels
    gz = g0.copy()
    gz[:70, :70] = 0.0
    plz = ref_planes(CAM, gz)
    job("dog_zero_window", [_step()], {"xs_nan": 100}, grays=(gz,), planes=(plz,))
    job("pos_neg_one", [_step(per_hist=1.0)], {"q0_p0": 1, "q1_p0": 1, "q2_p0": 1, "q3_p0": 1})
    # the kl_max cut
    cand = _cand(T0, R, BASE)
    T = len(cand)
    ys, xs = T0["ys"][cand], T0["xs"][cand]
    idx = ys * CAM["w"] + xs
    for km in (0, -7):
        job("cut_kl_max%d" % km, [_step(kl_max=km)], {"kl_max_nonpositive_one": 1})
    for km in (1, 2):
        job("cut_kl_max%d" % km, [_step(kl_max=km)], {"cut": 1})
    for km in (T - 1, T):
        job("cut_total%+d" % (km - T), [_step(kl_max=int(km))], {"cut": 1})
    job("cut_total+1", [_step(kl_max=T + 1)], {"no_cut": 1})
    nchunk = (CAM["w"] + 31) // 32
    per = (CAM["h"] * nchunk + 1023) // 1024
    seg = ys * nchunk + xs // 32
    picks = dict(lane0=np.nonzero(xs % 32 == 0)[0], lane31=np.nonzero(xs % 32 == 31)[0],
                 last_chunk=np.nonzero(xs // 32 == nchunk - 1)[0], thread_first=np.nonzero(seg % per == 0)[0],
                 thread_last=np.nonzero(seg % per == per - 1)[0])
    for k, ii in picks.items():
        ii = ii[(ii > 10) & (ii < T - 10)]
        i = int(ii[len(ii) // 2])
        job("cut_keep_" + k, [_step(kl_max=i + 1)], {"cut_" + k: 1})     # the last kept keyline on it
        job("cut_drop_" + k, [_step(kl_max=i)], {"drop_" + k: 1})       # the first dropped one on it
    job("kcap_small", [_step(kl_max=40000)], {"cut": 1}, kcap=T // 2)
    job("kcap_eq_kl_max", [_step(kl_max=T // 3)], {"cut": 1}, kcap=T // 3)
    # the cut on a 1241-pixel row (per = 15 segments a scan thread)
    gk = edge_frame(CAM_K["w"], CAM_K["h"], 400 + R)
    plk = ref_planes(CAM_K, gk)
    Tk = detect_terms(*plk, R)
    ck = _cand(Tk, R, BASE)
    xk = Tk["xs"][ck]
    i = int(np.nonzero(xk // 32 == (CAM_K["w"] + 31) // 32 - 1)[0][len(ck) // 1000])
    job("kitti_cut_last_chunk", [_step(kl_max=i + 1)], {"cut_last_chunk": 1}, grays=(gk,), planes=(plk,), cam=CAM_K)
    # the whole 1241x376 frame also holds keylines on x.5 positions, and at R = 1 a pixel exactly on the sub-pixel test
    # (|xs| = 0.5 in float32): the seeds are chosen for it, no construction forces it
    job("kitti_full", [_step()], dict({"p_id_collisions": 100, "c_p_half": 1}, **({"sub_on": 1} if R == 1 else {})),
        grays=(gk,), planes=(plk,), cam=CAM_K)
    # a map that already holds a mask: ids on border pixels (loaded) survive a detect unless the cut clears past them
    kn1, _, _, kl1, mask1 = port_detect(*pl1, R, BASE["per_hist"], BASE["dog_thresh"], 40000, BASE["tresh"], 0, 0, 0.0,
                                        1.0, 0.0, CAM["ppx"], CAM["ppy"])
    rng = np.random.default_rng(R)
    prior = mask1.copy()
    border = np.ones_like(prior, bool)
    border[R:-R, R:-R] = False
    prior[border] = np.where(rng.random(int(border.sum())) < 0.5, rng.integers(0, kn1, int(border.sum())), -1)
    job("prior_border_ids", [_step(prior=(kl1, prior))], {"border_ids_out": 50})
    job("prior_border_ids_cut", [_step(prior=(kl1, prior), kl_max=T // 2)], {"border_ids_out": 10,
                                                                           "border_ids_cleared": 10})
    job("prior_border_ids_kl_max0", [_step(prior=(kl1, prior), kl_max=0)], {"border_ids_cleared": 50})
    # a map whose mask comes from a detect with another window size (on the device: that detect on the same map; on the
    # reference, which cannot change window size within a process: that detect's mask loaded).  A narrower window
    # rewrites the whole old interior.  A wider one leaves the ring between the two margins alone in the reference's
    # loop; the library clears it (k_mask_margin), so that a map gives the same result whatever window detected on it
    # last, and the reference is given the mask with that ring cleared.
    other = {1: 4, 4: 1}.get(R)
    if other:
        kno, _, _, klo, masko = port_detect(*pl0, other, BASE["per_hist"], BASE["dog_thresh"], 40000, BASE["tresh"], 0,
                                            0, 0.0, 1.0, 0.0, CAM["ppx"], CAM["ppy"])
        yy, xx = np.mgrid[0:CAM["h"], 0:CAM["w"]]
        d = np.minimum(np.minimum(xx, CAM["w"] - 1 - xx), np.minimum(yy, CAM["h"] - 1 - yy))
        ring = (d >= other) & (d < R)
        fixed = {"ring_ids": int((masko[ring] >= 0).sum()), "prior_ids": int((masko >= 0).sum())}
        masko = np.where(ring, -1, masko).astype(np.int32)
        name = "switch_%d_to_%d" % (other, R)
        want = {"ring_ids": 10} if other < R else {"prior_ids": 1000}
        job(name, [_step(prior=(klo, masko), pre_detect=other)], want, fixed=fixed)
        job(name + "_cut", [_step(prior=(klo, masko), pre_detect=other, kl_max=T // 2)], dict(want, cut=1),
            fixed=fixed)
    # the P-controller over 24 detects, dense and near-flat frames alternating
    seq = [0, 1, 2, 2, 0, 2, 1, 2, 0, 0, 2, 1, 2, 0, 2, 2, 1, 0, 2, 1, 0, 2, 2, 1]
    three = dict(grays=(g0, g1, gflat), planes=(pl0, pl1, plf))
    ctl = dict(kl_ref=1200, reest=[(1000, 100)])
    job("ctl_clamps", [_step(f=f, gain=2e-4, tmax=0.06, tmin=0.004, **ctl) for f in seq],
        {"clamp_max": 3, "clamp_min": 3, "err_pos": 3, "err_neg": 3}, **three)
    job("ctl_unclamped", [_step(f=f, gain=3e-6, tmax=0.5, tmin=0.0005, **ctl) for f in seq],
        {"err_pos": 3, "err_neg": 3}, **three)
    job("ctl_gain0", [_step(f=f, gain=0.0, **ctl) for f in seq], {"gain0_steps": len(seq)}, **three)
    job("ctl_tmin_gt_tmax", [_step(f=f, gain=1e-5, tmax=0.008, tmin=0.02, **ctl) for f in seq],
        {"clamp_max": 3, "clamp_min": 3}, **three)
    # reEstimateThresh after a detect, every knum / nbins edge; then an empty detect on the same map
    kn_full = T
    re = [(kn, nb) for kn in (-3, 0, 1, kn_full - 1, kn_full, kn_full + 9) for nb in (1, 2, 100, 4096)]
    job("reest_after_detect", [_step(reest=re)], {"reest_knum_le0": 8, "reest_knum_gt_kn": 4})
    job("empty_after_detect", [_step(), _step(per_hist=0.0, reest=[(10, 100)])], {"empty": 1, "reest_stale": 1})
    return jobs


def steps_of(job, results):
    """Over the steps: the controller's error signs and clamps, steps with gain 0, empty detects and reEstimateThresh
    calls past each end of knum."""
    out = dict(clamp_max=0, clamp_min=0, err_pos=0, err_neg=0, gain0_steps=0, empty=0, reest_knum_le0=0,
               reest_knum_gt_kn=0, reest_stale=0)
    l = 0
    for st, r in zip(job["steps"], results):
        out["gain0_steps"] += st["gain"] == 0
        out["empty"] += r["kn"] == 0
        out["reest_knum_le0"] += sum(k <= 0 for k, _ in st["reest"])
        out["reest_knum_gt_kn"] += sum(k > r["kn"] for k, _ in st["reest"])
        out["reest_stale"] += len(st["reest"]) if r["kn"] == 0 else 0
        if st["gain"] > 0:
            e = st["kl_ref"] - l
            out["err_pos"] += e > 0
            out["err_neg"] += e < 0
            out["clamp_max"] += r["t"] == st["tmax"]
            out["clamp_min"] += r["t"] == st["tmin"]
        l = r["l"]
    return {k: int(v) for k, v in out.items()}


def reach(job, results):
    """Reach counts of a detect job on the restatement's results."""
    c = steps_of(job, results)
    c.update(job["fixed"])
    R = job["R"]
    h, w = job["planes"][0][0].shape
    border = np.ones((h, w), bool)
    border[R:h - R, R:w - R] = False

    def add(k, v):
        c[k] = c.get(k, 0) + int(v)

    for st, r in zip(job["steps"], results):
        if st["prior"] is not None:
            pm = st["prior"][1]
            add("border_ids_cleared", ((pm >= 0) & (r["mask"] < 0) & border).sum())
        add("border_ids_out", ((r["mask"] >= 0) & border).sum())
        add("kl_max_nonpositive_one", st["kl_max"] <= 0 and r["kn"] == 1)
        T = detect_terms(*job["planes"][st.get("f", 0)], R)
        tr = dict(st, tresh=r["t"])
        for k, v in boundary_counts(T, R, tr).items():
            c[k] = c.get(k, 0) + v
        for k, v in join_counts(r["kl"], r["mask"]).items():
            c[k] = c.get(k, 0) + v
        cand = _cand(T, R, tr)
        kl_max = min(st["kl_max"], job["kcap"])
        ci = T["ys"][cand] * job["cam"]["w"] + T["xs"][cand]
        pos = cut_position(job["cam"], R, ci, kl_max)
        add("cut", pos is not None)
        add("no_cut", pos is None and len(cand) > 0)
        drop = cut_position(job["cam"], R, ci, max(kl_max, 1) + 1)     # the first keyline the cut drops
        for tag, q in (("cut_", pos), ("drop_", drop)):
            if q:
                add(tag + "lane0", q["lane"] == 0)
                add(tag + "lane31", q["lane"] == 31)
                for k in ("thread_first", "thread_last", "last_chunk"):
                    add(tag + k, q[k])
    return c


# ---- executors --------------------------------------------------------------------------------------------------------
def _kl_max(job, st):
    return min(st["kl_max"], job["kcap"])


def run_port(job):
    h, w = job["planes"][0][0].shape
    masks, n_m0, out = {}, {}, []
    t, l = job["t0"], 0
    for st in job["steps"]:
        f = st.get("f", 0)
        if st["prior"] is not None:
            masks[f] = st["prior"][1]
            if len(st["prior"][0]):
                n_m0[f] = st["prior"][0]["n_m"][0]
        kn, t, l, kl, mask = port_detect(*job["planes"][f], job["R"], st["per_hist"], st["dog_thresh"],
                                         _kl_max(job, st), t, l, st["kl_ref"], st["gain"], st["tmax"], st["tmin"],
                                         job["cam"]["ppx"], job["cam"]["ppy"], masks.get(f))
        masks[f] = mask
        if kn:
            n_m0[f] = kl["n_m"][0]
        out.append(dict(kn=kn, t=t, l=l, kl=kl, mask=mask,
                        reest=[port_reestimate(kl["n_m"], k, n, n_m0.get(f)) for k, n in st["reest"]]))
    return out


def run_dev(job, ctxs):
    """ctxs: {(cam w, h, kcap): capi.Ctx}, filled on demand."""
    from rebvo_b200 import capi
    cam = job["cam"]
    key = (cam["w"], cam["h"], job["kcap"])
    if key not in ctxs:
        ctxs[key] = capi.Ctx(cam, SIGMA0, KSIGMA, kl_capacity=job["kcap"])
    ctx = ctxs[key]
    maps, out = {}, []
    t, l = job["t0"], 0
    try:
        for st in job["steps"]:
            f = st.get("f", 0)
            if f not in maps:
                m = ctx.new_map()
                m.upload_gray(job["grays"][f])
                m.dog_build()
                maps[f] = m
            m = maps[f]
            if st.get("pre_detect"):
                pre = capi.DetectParams(st["pre_detect"], BASE["per_hist"], BASE["dog_thresh"], 40000, BASE["kl_ref"],
                                        0.0, 1.0, 0.0)
                m.detect(pre, BASE["tresh"], 0)
            elif st["prior"] is not None:
                m.load_keylines(st["prior"][0], st["prior"][1])
            det = capi.DetectParams(job["R"], st["per_hist"], st["dog_thresh"], st["kl_max"], st["kl_ref"], st["gain"],
                                    st["tmax"], st["tmin"])
            kn, t, l = m.detect(det, t, l)
            out.append(dict(kn=kn, t=t, l=l, kl=m.keylines(), mask=m.mask(),
                            reest=[np.float32(m.reestimate(k, n)) for k, n in st["reest"]]))
    finally:
        for m in maps.values():
            m.close()
    return out


def ref_results(tmp_dir, R, jobs):
    """The reference on jobs of window size R: in this process for R = 2, in one child process otherwise."""
    return [run_ref_job(j) for j in jobs] if R == 2 else ref_child(tmp_dir, R, jobs)


# ---- reEstimateThresh -------------------------------------------------------------------------------------------------
def _x86_int(a):
    """float -> int as x86-64 cvttss2si: NaN and out-of-range values give INT_MIN."""
    a = np.asarray(a, np.float64)
    bad = ~np.isfinite(a) | (a >= 2.0 ** 31) | (a < -2.0 ** 31)
    return np.where(bad, -2 ** 31, np.trunc(np.where(bad, 0, a))).astype(np.int64)


def port_reestimate(n_m, knum, n, stale=None):
    """edge_finder::reEstimateThresh (:373-405) in float32 on the keylines' n_m.  The search loop skips bin 0 and ends on
    i < n whatever it would read at histo[n].  With kn = 0 the reference returns kl[0].n_m, whatever an earlier detect or
    load left there (`stale`); the device returns 0 (DESIGN.md section 3)."""
    n_m = np.asarray(n_m, np.float32)
    if len(n_m) == 0:
        return np.float32(stale)
    mx, mn = n_m.max(), n_m.min()
    rng = np.float32(mx - mn)
    with np.errstate(divide="ignore", invalid="ignore"):
        b = _x86_int(np.float32(n) * (mx - n_m) / rng)
    b = np.clip(np.minimum(b, n - 1), 0, None)
    histo = np.bincount(b, minlength=n)
    i, a = 0, 0
    while i < n and a < knum:
        i += 1
        a += histo[i] if i < n else 0
    return np.float32(mx - np.float32(np.float32(i) * rng) / np.float32(n))


def reest_sets():
    """(name, n_m) keyline sets for reEstimateThresh, each loaded on both sides."""
    rng = np.random.default_rng(3)
    f = np.float32
    return [
        ("one", np.array([37.25], f)),
        ("all_equal", np.full(10, 12.5, f)),
        ("two_values", np.array([3.0, 9.0, 3.0, 9.0, 9.0], f)),
        ("exact_bins", np.arange(0, 101, dtype=f)),                     # 100 * (100 - v) / 100 is an integer
        ("exact_bins_4096", (np.arange(0, 4097, dtype=np.float64) / 16.0).astype(f)),
        ("random", rng.uniform(5, 900, 3000).astype(f)),
        ("one_bin_50000", np.concatenate([np.full(49990, 250.0, f), rng.uniform(0, 1000, 10).astype(f)])),
    ]


def reest_calls(kn):
    return [(k, n) for k in sorted({-1, 0, 1, max(kn - 1, 0), kn, kn + 3}) for n in (1, 2, 100, 4096)]


def keylines_with(n_m, c_p=None, u_m=None):
    KL = keyline_dtype()
    kl = np.zeros(len(n_m), KL)
    kl["n_m"] = n_m
    kl["c_p"] = c_p if c_p is not None else 0
    kl["u_m"] = u_m if u_m is not None else 0
    for k in ("n_id", "p_id", "m_id", "m_id_f", "m_id_kf", "net_id", "stereo_m_id"):
        kl[k] = -1
    return kl


# ---- build_field ------------------------------------------------------------------------------------------------------
def _round_half_away(x):
    """roundf: half-way cases away from zero, exact in float64 for float32 inputs."""
    x = np.asarray(x, np.float64)
    return np.sign(x) * np.floor(np.abs(x) + 0.5)


def port_field(kl, radius, min_mod, w, h):
    """global_tracker::build_field (:61-105): per pixel the keyline with the smallest |t|, the later one on a tie; {dist,
    ikl} int32 [h, w, 2] with dist 0 and ikl -1 on empty pixels."""
    kn = len(kl)
    out = np.zeros((h, w, 2), np.int32)
    out[:, :, 1] = -1
    keep = np.nonzero(~((np.float32(min_mod) > 0) & (kl["n_m"] < np.float32(min_mod))))[0]
    if len(keep) == 0:
        return out
    t = np.arange(-radius, radius, dtype=np.int64)
    ikl = np.repeat(keep, len(t))
    tt = np.tile(t, len(keep))
    u, c = kl["u_m"][ikl], kl["c_p"][ikl]
    tf = tt.astype(np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        fx = u[:, 0] * tf + c[:, 0]                      # float32 product, then sum (no contraction)
        fy = u[:, 1] * tf + c[:, 1]
    xi, yi = _round_half_away(fx), _round_half_away(fy)
    ok = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
    pix = (yi[ok] * w + xi[ok]).astype(np.int64)
    at, who = np.abs(tt[ok]), ikl[ok]
    o = np.lexsort((-who, at, pix))
    pix, at, who = pix[o], at[o], who[o]
    first = np.ones(len(pix), bool)
    first[1:] = pix[1:] != pix[:-1]
    flat = out.reshape(-1, 2)
    flat[pix[first], 0] = at[first]
    flat[pix[first], 1] = who[first]
    return out


def field_ties(kl, radius, min_mod, w, h):
    """Pixels where two or more keylines reach the winning |t|."""
    fld = port_field(kl, radius, min_mod, w, h)
    t = np.arange(-radius, radius)
    keep = np.nonzero(~((np.float32(min_mod) > 0) & (kl["n_m"] < np.float32(min_mod))))[0]
    cnt = np.zeros(w * h, np.int64)
    for i in keep:
        tf = t.astype(np.float32)
        with np.errstate(over="ignore", invalid="ignore"):
            xi = _round_half_away(kl["u_m"][i, 0] * tf + kl["c_p"][i, 0])
            yi = _round_half_away(kl["u_m"][i, 1] * tf + kl["c_p"][i, 1])
        ok = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
        pix = (yi[ok] * w + xi[ok]).astype(np.int64)
        win = fld.reshape(-1, 2)[pix, 0] == np.abs(t[ok])
        cnt[np.unique(pix[win])] += 1
    return int((cnt >= 2).sum())


def field_sets(w, h, kcap):
    """(name, keylines, [(radius, min_mod), ...], minimum ties) for build_field."""
    f = np.float32
    rng = np.random.default_rng(11)
    sets = []
    P = np.array([150.0, 90.0])

    def through(n, t0, same):
        a = rng.uniform(0, 2 * np.pi, n)
        u = np.stack([np.cos(a), np.sin(a)], 1).astype(f)
        t = np.full(n, t0) if same else rng.integers(1, 30, n)
        c = (P[None] - u.astype(np.float64) * t[:, None]).astype(f)
        return keylines_with(rng.uniform(1, 50, n).astype(f), c, u)

    for n in (2, 32, 1000):
        sets.append(("ties_%d" % n, through(n, 7, True), [(40, 0.0), (8, 0.0)], 1))
        sets.append(("crossing_%d" % n, through(n, 0, False), [(40, 0.0)], 0))
    # axis-aligned segments on x.5 / y.5: roundf sends x.5 away from zero, -0.5 to -1 (outside)
    c = np.array([[0.5, 10.0], [10.0, 0.5], [w - 1.5, 20.0], [30.0, h - 1.5], [-0.5, 50.0], [60.0, -0.5],
                  [100.5, 100.5], [-0.5, -0.5]], f)
    u = np.array([[1, 0], [0, 1], [-1, 0], [0, -1], [0, 1], [1, 0], [-1, 0], [1, 0]], f)
    sets.append(("half_pixels", keylines_with(np.full(len(c), 10.0, f), c, u), [(1, 0.0), (40, 0.0), (100, 0.0)], 0))
    # segments leaving each border and corner; u_m far outside int range
    c = np.array([[2, 2], [w - 3, 2], [2, h - 3], [w - 3, h - 3], [w / 2, 1], [1, h / 2], [w - 2, h / 2], [w / 2, h - 2],
                  [50, 50], [60, 60]], f)
    a = np.radians(np.array([225, 315, 135, 45, 270, 180, 0, 90, 0, 30]))
    u = np.stack([np.cos(a), np.sin(a)], 1).astype(f)
    u[8] = (3e9, 0.0)
    u[9] = (-4e9, 2e9)
    sets.append(("borders_big_u", keylines_with(np.full(len(c), 5.0, f), c, u), [(1, 0.0), (40, 0.0), (100, 0.0)], 0))
    # n_m at min_mod and 1 ulp below it; min_mod <= 0 keeps all
    mm = f(20.0)
    nm = np.array([mm, np.nextafter(mm, f(0)), mm, np.nextafter(mm, f(0)), 30.0, 5.0], f)
    c = rng.uniform(20, min(w, h) - 20, (len(nm), 2)).astype(f)
    a = rng.uniform(0, 2 * np.pi, len(nm))
    u = np.stack([np.cos(a), np.sin(a)], 1).astype(f)
    sets.append(("min_mod", keylines_with(nm, c, u), [(40, float(mm)), (40, 0.0), (40, -1.0)], 0))
    # kn = kcap random keylines
    n = kcap
    c = np.stack([rng.uniform(-5, w + 5, n), rng.uniform(-5, h + 5, n)], 1).astype(f)
    a = rng.uniform(0, 2 * np.pi, n)
    a[: n // 4] = rng.integers(0, 8, n // 4) * (np.pi / 4)
    u = np.stack([np.cos(a), np.sin(a)], 1).astype(f)
    sets.append(("kcap", keylines_with(rng.uniform(0, 100, n).astype(f), c, u), [(40, 50.0), (100, 0.0)], 20))
    sets.append(("kn0", keylines_with(np.zeros(0, f)), [(40, 0.0)], 0))
    return sets


# ---- a stream for the fused pipeline ----------------------------------------------------------------------------------
PIPE_SEQ = [0, 1, 2, 2, 0, 2, 1, 2, 0, 0, 2, 1, 2, 0, 2, 2, 1, 0, 2, 1, 0, 2, 2, 1]
PIPE_DET = dict(plane_fit_size=2, pos_neg_thresh=0.4, dog_thresh=0.095259868922420, kl_max=40000, kl_ref=1000, gain=2e-4,
                thresh_max=0.06, thresh_min=0.004)


def pipe_stream():
    """(ts, mono uint8 [24, h, w]): dense and near-flat frames of CAM alternating, so that PIPE_DET's controller clamps at
    both ends."""
    fr = [np.clip(np.rint(edge_frame(CAM["w"], CAM["h"], s, contrast=c)), 0, 255).astype(np.uint8)
          for s, c in ((500, 1.0), (501, 1.0), (502, 0.04))]
    return np.arange(len(PIPE_SEQ)) / 20.0, np.stack([fr[i] for i in PIPE_SEQ])

"""DetectorPlaneFitSize R = 1..4: a NumPy restatement of the reference's detector for any window size, and the reference
itself run in a child process.

edge_finder::build_mask caches its pseudo inverse in a function-static sized by the first call of the process
(edge_finder.cpp:83-84); a later call with another win_s aborts in TooN's size check.  The in-process reference
(oracle/refapi.py) is used with R = 2 elsewhere, so every reference result for another R comes from a fresh process:
`python tests/plane_fit.py in.npz out.npz` (ref_detect_child below).

The restatement follows build_mask + join_edges (edge_finder.cpp:67-214, 304-320) with UpdateThresh (:330-335): float32
where the reference computes in float, float64 sums in its k order with no contraction, pixels vectorised, the kl_max
cut in raster order."""
import os
import pickle
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAX_IMG_VALUE = np.float32(765)
RHO_INIT, RHO_MAX = 1.0, 20.0


def keyline_dtype():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from rebvo_b200.capi import KEYLINE
    return KEYLINE


def plane_fit_pinv(ws):
    """PInv = Matrix3x3Inv(Phi^T Phi) * Phi^T (edge_finder.cpp:83-100, toon_util.h:32-41): [3, (2 ws + 1)^2]."""
    phi = [(float(j), float(i), 1.0) for i in range(-ws, ws + 1) for j in range(-ws, ws + 1)]
    n = len(phi)
    A = [[0.0] * 3 for _ in range(3)]
    for r in range(3):
        for c in range(3):
            s = 0.0
            for k in range(n):
                s += phi[k][r] * phi[k][c]
            A[r][c] = s
    B = [[A[2][2] * A[1][1] - A[2][1] * A[1][2], -(A[2][2] * A[0][1] - A[2][1] * A[0][2]),
          A[1][2] * A[0][1] - A[1][1] * A[0][2]],
         [-(A[2][2] * A[1][0] - A[2][0] * A[1][2]), A[2][2] * A[0][0] - A[2][0] * A[0][2],
          -(A[1][2] * A[0][0] - A[1][0] * A[0][2])],
         [A[2][1] * A[1][0] - A[2][0] * A[1][1], -(A[2][1] * A[0][0] - A[2][0] * A[0][1]),
          A[1][1] * A[0][0] - A[1][0] * A[0][1]]]
    det = (A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) - A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0]) +
           A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]))
    B = [[B[r][c] / det for c in range(3)] for r in range(3)]
    out = np.zeros((3, n))
    for r in range(3):
        for k in range(n):
            s = 0.0
            for c in range(3):
                s += B[r][c] * phi[k][c]
            out[r, k] = s
    return out


def update_thresh(tresh, l_kl_num, kl_ref, gain, tmax, tmin):
    if gain > 0:
        tresh -= gain * float(kl_ref - l_kl_num)
        tresh = tmax if tresh > tmax else (tmin if tresh < tmin else tresh)
    return tresh


def detect_terms(img0, dog, R):
    """The per-pixel quantities build_mask tests, over the interior pixels in raster order (they do not depend on the
    thresholds): ys, xs, n2gI (:117), pn (:122-133), xsub / ysub (:146-147), mx / my (:154), n2_m (:157)."""
    h, w = dog.shape
    ys, xs = np.mgrid[R:h - R, R:w - R]
    ys, xs = ys.ravel(), xs.ravel()
    gx = img0[ys, xs + 1] - img0[ys, xs - 1]                     # sspace::calc_gradient (float32)
    gy = img0[ys + 1, xs] - img0[ys - 1, xs]
    pn = np.zeros(len(xs), np.int64)
    for i in range(-R, R + 1):
        for j in range(-R, R + 1):
            pn += np.where(dog[ys + i, xs + j] > 0, 1, -1)
    pinv = plane_fit_pinv(R)
    th = np.zeros((3, len(xs)))
    k = 0
    for i in range(-R, R + 1):
        for j in range(-R, R + 1):
            yv = dog[ys + i, xs + j].astype(np.float64)
            for r in range(3):
                th[r] = th[r] + pinv[r, k] * yv
            k += 1
    with np.errstate(divide="ignore", invalid="ignore"):
        den = th[0] * th[0] + th[1] * th[1]
        xsub = (-th[0] * th[2] / den).astype(np.float32)
        ysub = (-th[1] * th[2] / den).astype(np.float32)
    mx, my = th[0].astype(np.float32), th[1].astype(np.float32)
    return dict(ys=ys, xs=xs, n2gI=gx * gx + gy * gy, pn=pn, xsub=xsub, ysub=ysub, mx=mx, my=my, n2_m=mx * mx + my * my)


def detect_tests(T, R, pos_neg, dog_thresh, tresh):
    """The four tests of build_mask on detect_terms T with the detector's float32 thresholds: the boolean pass arrays
    (grad :119, pn :137, sub :150, dog :159) and the two squared bounds."""
    grad_thesh, per_hist, dog_thesh = np.float32(tresh), np.float32(pos_neg), np.float32(dog_thresh)
    t1 = grad_thesh * MAX_IMG_VALUE
    lim = np.float32((2.0 * R + 1.0) * (2.0 * R + 1.0)) * per_hist
    t5 = grad_thesh * MAX_IMG_VALUE * dog_thesh
    with np.errstate(invalid="ignore"):
        grad = ~(T["n2gI"] < t1 * t1)
        pn = ~(np.abs(T["pn"]).astype(np.float64) > np.float64(lim))
        sub = ~((np.abs(T["xsub"]) > 0.5) | (np.abs(T["ysub"]) > 0.5))
        dog = ~(T["n2_m"] < t5 * t5)
    return dict(grad=grad, pn=pn, sub=sub, dog=dog, t1sq=t1 * t1, lim=lim, t5sq=t5 * t5)


def port_detect(img0, dog, R, pos_neg, dog_thresh, kl_max, tresh, l_kl_num, kl_ref, gain, tmax, tmin, ppx, ppy,
                mask=None):
    """edge_finder::detect with win_s = R on the planes Img(0) and DoG (float32 [h, w]).  mask: the map's id mask before
    the call (default all -1), updated like the reference's img_mask_kl.  Returns (kn, tresh, l_kl_num, keylines, mask)."""
    h, w = dog.shape
    tresh = update_thresh(tresh, l_kl_num, kl_ref, gain, tmax, tmin)
    mask = np.full((h, w), -1, np.int32) if mask is None else np.array(mask, np.int32)
    T = detect_terms(img0, dog, R)
    P = detect_tests(T, R, pos_neg, dog_thresh, tresh)
    ys, xs, xsub, ysub, mx, my, n2_m = (T[k] for k in ("ys", "xs", "xsub", "ysub", "mx", "my", "n2_m"))
    ok = P["grad"] & P["pn"] & P["sub"] & P["dog"]
    mask[R:h - R, R:w - R] = -1
    cand = np.nonzero(ok)[0]
    kl_max = max(kl_max, 1)         # build_mask appends a keyline before it tests ++kn >= kl_max (:203)
    kn = min(len(cand), kl_max)
    sel = cand[:kn]
    KL = keyline_dtype()
    kl = np.zeros(kn, KL)
    idx = (ys[sel] * w + xs[sel]).astype(np.int32)
    n_m = np.sqrt(n2_m[sel])
    cx = xs[sel].astype(np.float32) + xsub[sel]
    cy = ys[sel].astype(np.float32) + ysub[sel]
    kl["p_inx"] = idx
    kl["m_m"] = np.stack([mx[sel], my[sel]], 1)
    kl["n_m"] = n_m
    kl["u_m"] = np.stack([mx[sel] / n_m, my[sel] / n_m], 1)
    kl["c_p"] = np.stack([cx, cy], 1)
    pm = np.stack([cx - np.float32(ppx), cy - np.float32(ppy)], 1)
    kl["p_m"] = pm
    kl["p_m_0"] = pm
    for f in ("rho", "rho0", "rho_nr", "stereo_rho"):
        kl[f] = RHO_INIT
    for f in ("s_rho", "s_rho0", "s_rho_nr", "stereo_s_rho"):
        kl[f] = RHO_MAX
    for f in ("n_id", "p_id", "net_id", "m_id", "m_id_f", "m_id_kf", "stereo_m_id"):
        kl[f] = -1
    flat = mask.reshape(-1)
    flat[idx] = np.arange(kn, dtype=np.int32)
    if kn >= kl_max and kn > 0:                                  # the cut clears the rest of the image (:203-207)
        flat[idx[-1] + 1:] = -1
    # join_edges: NextPoint from the rounded position; the last writer of p_id (the largest i) wins.  A probe past the
    # end of the mask (R = 1: a keyline on row h-2 whose c_p rounds to row h-1) counts as no keyline, as on the device;
    # the reference reads past its buffer there.
    if kn:
        x = (cx.astype(np.float64) + 0.5).astype(np.int64)
        y = (cy.astype(np.float64) + 0.5).astype(np.int64)
        tx, ty = -my[sel], mx[sel]
        sx = np.where(ty > 0, np.where(tx > 0, 1, -1), np.where(tx < 0, -1, 1))
        sy = np.where(ty > 0, 1, -1)
        nxt = np.full(kn, -1, np.int64)
        for px, py in ((x + sx, y), (x, y + sy), (x + sx, y + sy)):
            pi = py * w + px
            inside = (pi >= 0) & (pi < h * w)
            v = np.where(inside, flat[np.where(inside, pi, 0)], -1)
            nxt = np.where((nxt < 0) & (v >= 0), v, nxt)
        has = nxt >= 0
        kl["n_id"][has] = nxt[has]
        # an id loaded on a border pixel may be >= kn: its p_id lies past the keylines, as in the reference's array
        p_id = np.full(max(kn, int(nxt.max()) + 1), -1, np.int64)
        np.maximum.at(p_id, nxt[has], np.nonzero(has)[0])
        kl["p_id"] = p_id[:kn]
    return kn, tresh, kn, kl, mask


# ---- the reference in a child process ------------------------------------------------------------------------------
def run_ref_job(job):
    """The reference on one detect job (tests/front_states.py, detect_jobs): window size job["R"], one edge map per frame
    (job["grays"] through set_gray, or job["rgbs"] through rgb2bw), the steps in order with the threshold chained from
    job["t0"]; a step's `prior` = (keylines, mask) is loaded before its detect, its `reest` = [(knum, nbins)] run after
    it.  Returns per step {kn, t, l, kl, mask, reest}."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import refapi
    cam = job["cam"]
    maps, out = {}, []
    t, l = job["t0"], 0
    for st in job["steps"]:
        f = st.get("f", 0)
        if f not in maps:
            m = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], job["sigma0"],
                              job["ksigma"])
            if "rgbs" in job:
                m.rgb2bw(job["rgbs"][f])
            else:
                m.set_gray(job["grays"][f])
            m.build()
            maps[f] = m
        m = maps[f]
        if st.get("prior") is not None:
            m.set_keylines(st["prior"][0])
            m.set_mask(st["prior"][1], len(st["prior"][0]))
        kn, t, l = m.detect(job["R"], st["per_hist"], st["dog_thresh"], min(st["kl_max"], job.get("kcap", 50000)), t,
                            l, st["kl_ref"], st["gain"], st["tmax"], st["tmin"])
        out.append(dict(kn=kn, t=t, l=l, kl=m.keylines(), mask=m.mask(),
                        reest=[np.float32(m.reestimate(k, n)[1]) for k, n in st.get("reest", [])]))
    return out


def ref_child(tmp_dir, R, jobs, timeout=900):
    """run_ref_job on every job (all of window size R) in a new process: `python tests/plane_fit.py in.pkl out.pkl`."""
    tag = "r%d_%d" % (R, os.getpid())
    k = 0
    while os.path.exists(os.path.join(str(tmp_dir), "%s_%d_in.pkl" % (tag, k))):
        k += 1
    src = os.path.join(str(tmp_dir), "%s_%d_in.pkl" % (tag, k))
    dst = os.path.join(str(tmp_dir), "%s_%d_out.pkl" % (tag, k))
    assert all(j["R"] == R for j in jobs)
    with open(src, "wb") as f:
        pickle.dump(jobs, f)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), src, dst], capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError("reference child (R=%d) failed: %d\n%s" % (R, r.returncode, r.stderr[-3000:]))
    with open(dst, "rb") as f:
        return pickle.load(f)


def ref_detect_child(tmp_dir, frames, R, cam, sigma0, ksigma, thresh, kl_max, kl_ref, gain, tmax, tmin, pos_neg,
                     dog_thresh, track_points=12000, cut=None, timeout=600):
    """The reference's detect + reEstimateThresh with win_s = R on each RGB frame (one edge map per frame, the threshold
    chained through UpdateThresh), then optionally a detect cut at `cut` keylines on the last frame (gain 0) -- in a new
    process.  Returns {name: array}; keylines are KEYLINE arrays."""
    base = dict(per_hist=float(pos_neg), dog_thresh=float(dog_thresh), kl_ref=int(kl_ref), prior=None)
    steps = [dict(base, f=i, kl_max=int(kl_max), gain=float(gain), tmax=float(tmax), tmin=float(tmin),
                  reest=[(int(track_points), 100)]) for i in range(len(frames))]
    if cut:
        steps.append(dict(base, f=len(frames) - 1, kl_max=int(cut), gain=0.0, tmax=1.0, tmin=0.0, reest=[]))
    job = dict(R=int(R), cam=dict(cam), sigma0=float(sigma0), ksigma=float(ksigma), t0=float(thresh),
               rgbs=np.ascontiguousarray(frames, np.uint8), steps=steps)
    res = ref_child(tmp_dir, R, [job], timeout)[0]
    out = {}
    for i in range(len(frames)):
        r = res[i]
        out["f%d_kn_tresh" % i] = np.array([r["kn"], r["t"], r["l"]], np.float64)
        out["f%d_kl" % i] = r["kl"]
        out["f%d_mask" % i] = r["mask"]
        out["f%d_retuned" % i] = np.array(r["reest"], np.float32)
    if cut:
        out["cut_kn"] = np.array([res[-1]["kn"]])
        out["cut_kl"] = res[-1]["kl"]
        out["cut_mask"] = res[-1]["mask"]
    return out


if __name__ == "__main__":
    with open(sys.argv[1], "rb") as fi:
        jobs_in = pickle.load(fi)
    results = [run_ref_job(j) for j in jobs_in]
    with open(sys.argv[2], "wb") as fo:
        pickle.dump(results, fo)

"""DetectorPlaneFitSize R = 1..4: a NumPy restatement of the reference's detector for any window size, and the reference
itself run in a child process.

edge_finder::build_mask caches its pseudo inverse in a function-static sized by the first call of the process
(edge_finder.cpp:83-84); a later call with another win_s aborts in TooN's size check.  The in-process reference
(oracle/refapi.py) is used with R = 2 elsewhere, so every reference result for another R comes from a fresh process:
`python tests/plane_fit.py in.npz out.npz` (ref_detect_child below).

The restatement follows build_mask + join_edges (edge_finder.cpp:67-214, 304-320) with UpdateThresh (:330-335): float32
where the reference computes in float, float64 sums in its k order with no contraction, pixels vectorised, the kl_max
cut in raster order."""
import json
import os
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


def port_detect(img0, dog, R, pos_neg, dog_thresh, kl_max, tresh, l_kl_num, kl_ref, gain, tmax, tmin, ppx, ppy,
                mask=None):
    """edge_finder::detect with win_s = R on the planes Img(0) and DoG (float32 [h, w]).  mask: the map's id mask before
    the call (default all -1), updated like the reference's img_mask_kl.  Returns (kn, tresh, l_kl_num, keylines, mask)."""
    h, w = dog.shape
    tresh = update_thresh(tresh, l_kl_num, kl_ref, gain, tmax, tmin)
    grad_thesh, per_hist, dog_thesh = np.float32(tresh), np.float32(pos_neg), np.float32(dog_thresh)
    mask = np.full((h, w), -1, np.int32) if mask is None else np.array(mask, np.int32)
    ys, xs = np.mgrid[R:h - R, R:w - R]
    ys, xs = ys.ravel(), xs.ravel()
    gx = img0[ys, xs + 1] - img0[ys, xs - 1]                     # sspace::calc_gradient (float32)
    gy = img0[ys + 1, xs] - img0[ys - 1, xs]
    t1 = grad_thesh * MAX_IMG_VALUE
    ok = ~(gx * gx + gy * gy < t1 * t1)
    pn = np.zeros(len(xs), np.int64)
    for i in range(-R, R + 1):
        for j in range(-R, R + 1):
            pn += np.where(dog[ys + i, xs + j] > 0, 1, -1)
    lim = np.float32((2.0 * R + 1.0) * (2.0 * R + 1.0)) * per_hist
    ok &= ~(np.abs(pn).astype(np.float64) > np.float64(lim))
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
    ok &= ~((np.abs(xsub) > 0.5) | (np.abs(ysub) > 0.5))
    mx, my = th[0].astype(np.float32), th[1].astype(np.float32)
    n2_m = mx * mx + my * my
    t5 = grad_thesh * MAX_IMG_VALUE * dog_thesh
    ok &= ~(n2_m < t5 * t5)
    mask[R:h - R, R:w - R] = -1
    cand = np.nonzero(ok)[0]
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
        p_id = np.full(kn, -1, np.int64)
        np.maximum.at(p_id, nxt[has], np.nonzero(has)[0])
        kl["p_id"] = p_id
    return kn, tresh, kn, kl, mask


# ---- the reference in a child process ------------------------------------------------------------------------------
def _child(in_path, out_path):
    sys.path.insert(0, ROOT)
    from oracle import refapi
    z = np.load(in_path)
    spec = json.loads(str(z["spec"]))
    frames = z["frames"]
    cam, R = spec["cam"], spec["R"]
    out = {}
    t, l = spec["thresh"], 0
    maps = []
    for i, fr in enumerate(frames):
        m = refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], spec["sigma0"],
                          spec["ksigma"])
        maps.append(m)
        m.rgb2bw(fr)
        m.build()
        kn, t, l = m.detect(R, spec["pos_neg"], spec["dog_thresh"], spec["kl_max"], t, l, spec["kl_ref"], spec["gain"],
                            spec["tmax"], spec["tmin"])
        out["f%d_kn_tresh" % i] = np.array([kn, t, l], np.float64)
        out["f%d_kl" % i] = m.keylines().view(np.uint8)
        out["f%d_mask" % i] = m.mask()
        out["f%d_retuned" % i] = np.array([m.reestimate(spec["track_points"], 100)[1]], np.float32)
    if spec.get("cut"):
        m = maps[-1]
        kn, _, _ = m.detect(R, spec["pos_neg"], spec["dog_thresh"], spec["cut"], t, l, spec["kl_ref"], 0.0, 1.0, 0.0)
        out["cut_kn"] = np.array([kn])
        out["cut_kl"] = m.keylines().view(np.uint8)
        out["cut_mask"] = m.mask()
    np.savez(out_path, **out)


def ref_detect_child(tmp_dir, frames, R, cam, sigma0, ksigma, thresh, kl_max, kl_ref, gain, tmax, tmin, pos_neg,
                     dog_thresh, track_points=12000, cut=None, timeout=600):
    """The reference's detect + reEstimateThresh with win_s = R on each frame (one edge map per frame, the threshold chained
    through UpdateThresh), then optionally a detect cut at `cut` keylines on the last frame (gain 0) -- in a new process.
    Returns {name: array}; keylines are KEYLINE arrays."""
    tag = "r%d_%d" % (R, os.getpid())
    k = 0
    while os.path.exists(os.path.join(str(tmp_dir), "%s_%d_in.npz" % (tag, k))):
        k += 1
    src = os.path.join(str(tmp_dir), "%s_%d_in.npz" % (tag, k))
    dst = os.path.join(str(tmp_dir), "%s_%d_out.npz" % (tag, k))
    spec = dict(R=int(R), cam={a: (int(v) if a in ("w", "h") else float(v)) for a, v in cam.items()},
                sigma0=float(sigma0), ksigma=float(ksigma), thresh=float(thresh), kl_max=int(kl_max), kl_ref=int(kl_ref),
                gain=float(gain), tmax=float(tmax), tmin=float(tmin), pos_neg=float(pos_neg),
                dog_thresh=float(dog_thresh), track_points=int(track_points), cut=int(cut) if cut else 0)
    np.savez(src, frames=np.ascontiguousarray(frames, np.uint8), spec=np.array(json.dumps(spec)))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), src, dst], capture_output=True, text=True,
                       timeout=timeout, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError("reference child (R=%d) failed: %d\n%s" % (R, r.returncode, r.stderr[-3000:]))
    KL = keyline_dtype()
    z = np.load(dst)
    return {k: (z[k].view(KL) if k.endswith("_kl") else z[k]) for k in z.files}


if __name__ == "__main__":
    _child(sys.argv[1], sys.argv[2])

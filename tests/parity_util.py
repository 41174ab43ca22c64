"""Helpers shared by the parity tests: drive the reference oracle (oracle/refapi.py, TEST ONLY) and the CUDA
library through the same calls and compare."""
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EUROC_CFG = dict(name="euroc", cam=dict(w=752, h=480, zfx=458.654, zfy=457.296, ppx=367.215, ppy=248.375),
                 sigma0=3.56359, ksigma=1.2599, thresh=0.01, gain=5e-7, tmax=0.5, tmin=0.005, kl_max=40000,
                 kl_ref=15000, track_points=12000, radius=40, match_thresh=0.5, iter_max=5, init_type=2,
                 init_iter=2, reweight=2.0, match_num_thresh=0, thr_mod=1.0, thr_ang=45.0, loc_unc_match=2.0,
                 reg_thresh=0.5, q_abs=1e-4, loc_unc=1.0)
TUM_CFG = dict(name="tum", cam=dict(w=640, h=480, zfx=525.0, zfy=525.0, ppx=320.0, ppy=240.0),
               sigma0=1.7818, ksigma=1.2599, thresh=0.01, gain=0.0, tmax=0.05, tmin=0.03, kl_max=25000,
               kl_ref=15000, track_points=12000, radius=20, match_thresh=1.0, iter_max=10, init_type=2,
               init_iter=2, reweight=2.0, match_num_thresh=4, thr_mod=1.0, thr_ang=45.0, loc_unc_match=2.0,
               reg_thresh=0.5, q_abs=1e-4, loc_unc=1.0)
# BASELINE.json configs[3]: synthetic 1280x960, ~30 k keylines
BIG_CFG = dict(name="big", cam=dict(w=1280, h=960, zfx=780.0, zfy=778.0, ppx=640.5, ppy=479.25),
               sigma0=3.56359, ksigma=1.2599, thresh=0.01, gain=5e-7, tmax=0.5, tmin=0.005, kl_max=40000,
               kl_ref=30000, track_points=24000, radius=40, match_thresh=0.5, iter_max=5, init_type=2,
               init_iter=2, reweight=2.0, match_num_thresh=0, thr_mod=1.0, thr_ang=45.0, loc_unc_match=2.0,
               reg_thresh=0.5, q_abs=1e-4, loc_unc=1.0)
POS_NEG, DOG_THRESH, PLANE_FIT = 0.4, 0.095259868922420, 2

# KeyLine fields the reference defines at every stage (m_m0 / n_m0 / score are uninitialised until a match)
KL_EXACT_DETECT = ["p_inx", "m_m", "u_m", "n_m", "c_p", "rho", "s_rho", "rho0", "s_rho0", "p_m", "p_m_0",
                   "m_id", "m_id_f", "m_num", "p_id", "n_id"]


class Report:
    def __init__(self, name):
        self.name = name
        self.items = []

    def add(self, what, ok, info=""):
        self.items.append(dict(what=what, ok=bool(ok), info=str(info)))
        print("[%s] %-46s %s %s" % (self.name, what, "PASS" if ok else "FAIL", info))

    def exact(self, what, a, b):
        a, b = np.asarray(a), np.asarray(b)
        if a.shape != b.shape:
            self.add(what, False, "shape %s vs %s" % (a.shape, b.shape))
            return False
        if a.dtype.kind == "f":
            same = (a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64)
                    == b.view(np.uint32 if b.dtype.itemsize == 4 else np.uint64)) | (np.isnan(a) & np.isnan(b))
        else:
            same = a == b
        nbad = int(same.size - same.sum())
        info = "bitwise n=%d" % same.size
        if nbad:
            idx = np.argwhere(~same)[:3]
            info = "mismatch %d/%d first=%s ref=%s got=%s" % (nbad, same.size, idx.tolist(),
                                                               [a[tuple(i)] for i in idx], [b[tuple(i)] for i in idx])
        self.add(what, nbad == 0, info)
        return nbad == 0

    def close(self, what, ref, got, rtol, atol=0.0):
        ref, got = np.asarray(ref, np.float64), np.asarray(got, np.float64)
        if ref.shape != got.shape:
            self.add(what, False, "shape %s vs %s" % (ref.shape, got.shape))
            return False
        both_nan = np.isnan(ref) & np.isnan(got)
        err = np.abs(ref - got)
        tol = atol + rtol * np.abs(ref)
        bad = ~((err <= tol) | both_nan)
        nbad = int(bad.sum())
        mx = float(np.nanmax(err / (np.abs(ref) + atol + 1e-300))) if err.size else 0.0
        self.add(what, nbad == 0, "max rel err %.3e (rtol %.1e atol %.1e) bad=%d/%d" % (mx, rtol, atol, nbad, err.size))
        return nbad == 0

    def ok(self):
        return all(i["ok"] for i in self.items)

    def dump(self):
        d = os.path.join(ROOT, "gpurun_out")
        try:
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, "parity_%s.json" % self.name), "w") as f:
                json.dump(self.items, f, indent=1)
        except OSError:
            pass

    def failures(self):
        return [i for i in self.items if not i["ok"]]


def compare_keylines(rep, tag, ref, got, exact_fields, close_fields=(), rtol=1e-12):
    if len(ref) != len(got):
        rep.add(tag + " kn", False, "%d vs %d" % (len(ref), len(got)))
        return
    rep.add(tag + " kn", True, "kn=%d" % len(ref))
    for f in exact_fields:
        rep.exact("%s %s" % (tag, f), ref[f], got[f])
    for f in close_fields:
        rep.close("%s %s" % (tag, f), ref[f], got[f], rtol)


def parity_frames(cfg):
    """The frame pair of the stage-level parity tests for one of the configurations above."""
    from rebvo_b200 import synth
    cam = cfg["cam"]
    if cfg["name"] == "tum":
        return synth.frame_pair(seed=42, w=cam["w"], h=cam["h"], nrect=220, shift=(1.5, 0.7))
    if cfg["name"] == "big":
        seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=100, zf=cam["zfx"], nrect_bg=1500, nrect_fg=200)
        return seq.frame(10)[1], seq.frame(11)[1]
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=7, zf=cam["zfx"])
    return seq.frame(10)[1], seq.frame(11)[1]


# ---- seeded edge-map states (tests/test_gpu_mapper_states.py, tests/test_gpu_minimiser_forms.py) --------------------
RHO_MIN, RHO_MAX = 1e-3, 20.0


def _bits(a):
    a = np.ascontiguousarray(a)
    if a.dtype.kind == "f":
        return a.view(np.uint32 if a.dtype.itemsize == 4 else np.uint64)
    return a


def _diff(tag, ref, got):
    """'' if ref and got are equal bit for bit (NaN == NaN), else a short description of the first mismatches."""
    ref, got = np.atleast_1d(ref), np.atleast_1d(got)
    if ref.shape != got.shape:
        return "%s: shape %s vs %s" % (tag, ref.shape, got.shape)
    same = _bits(ref) == _bits(got)
    if ref.dtype.kind == "f":
        same |= np.isnan(ref) & np.isnan(got)
    if same.ndim > 1:
        same = same.reshape(len(same), -1).all(1) if len(same) else np.ones(0, bool)
    bad = np.nonzero(~same)[0]
    if not len(bad):
        return ""
    i = bad[:3]
    return "%s: %d/%d differ, first %s ref %s gpu %s" % (tag, len(bad), len(same), i.tolist(), ref[i].tolist(),
                                                           got[i].tolist())


class Bench:
    """Two detected frames on the reference (two RefMap ring slots) and two GPU maps of one context.  The detector is the
    reference's (its parity with the GPU detector is test_gpu_parity's business); every mapper stage starts from a
    state loaded identically on both sides."""

    def __init__(self, cam, frames, kl_capacity=50000, cfg=EUROC_CFG):
        from oracle import refapi
        from rebvo_b200 import capi
        self.cam = cam
        self.zfm = float(np.float32((np.float32(cam["zfx"]) + np.float32(cam["zfy"])) / np.float32(2)))
        self.ref = [refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], cfg["sigma0"],
                                  cfg["ksigma"]) for _ in range(2)]
        t, l = cfg["thresh"], 0
        self.kl, self.mask = [], []
        for r, fr in zip(self.ref, frames):
            r.rgb2bw(fr)
            r.build()
            _, t, l = r.detect(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], t, l, cfg["kl_ref"], cfg["gain"],
                               cfg["tmax"], cfg["tmin"])
            self.kl.append(r.keylines())
            self.mask.append(r.mask())
        self.ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=kl_capacity)
        self.gpu = [self.ctx.new_map(), self.ctx.new_map()]

    def load(self, i, kl, mask=None):
        mask = self.mask[i] if mask is None else mask
        kl = np.ascontiguousarray(kl)
        self.ref[i].set_keylines(kl)
        self.ref[i].set_mask(mask, len(kl))
        self.gpu[i].load_keylines(kl, mask)

    def close(self):
        for g in self.gpu:
            g.close()
        self.ctx.close()


def _depth_state(kl, rng, new=False):
    """Seeded depth state inside the per-frame flow's domain: rho in [RHO_MIN, RHO_MAX] (log-uniform, plus exact 1e-3,
    1.0 and 20.0, plus runs of equal values), s_rho in [1e-6, 20], m_num in 0..10; new keylines with m_id = -1."""
    kl = kl.copy()
    k = len(kl)
    rho = np.exp(rng.uniform(np.log(RHO_MIN), np.log(RHO_MAX), k))
    u = rng.random(k)
    rho[u < 0.03] = RHO_MIN
    rho[(u >= 0.03) & (u < 0.06)] = 1.0
    rho[(u >= 0.06) & (u < 0.09)] = RHO_MAX
    for s in rng.choice(k, max(1, k // 64), replace=False):   # runs of equal values
        rho[s:s + 8] = rho[s]
    s_rho = np.exp(rng.uniform(np.log(1e-6), np.log(20.0), k))
    kl["rho"] = rho
    kl["s_rho"] = s_rho
    kl["m_num"] = rng.integers(0, 11, k)
    if new:
        kl["m_id"] = -1
    return kl


def _seed_depth(kl):
    kl = kl.copy()
    kl["rho"] = 1.0
    kl["s_rho"] = 0.2
    kl["m_num"] = 5
    return kl


def tracker_parity(rep, cfg, refs, gm, rt):
    """TryVelRot at three poses x three (reweight, procjf) pairs, then Minimizer_RV; returns the reference's result."""
    # old = frame 0 with seeded depth, new = frame 1
    old_r, new_r, old_g, new_g = refs[0], refs[1], gm[0], gm[1]
    old_r.set_keylines(_seed_depth(old_r.keylines()))
    old_g.load_keylines(old_r.keylines(), old_r.mask())
    new_g.load_keylines(new_r.keylines(), new_r.mask())
    q_r = old_r.quantile(1e-3, 20.0, 0.9, 100)
    q_g = old_g.quantile(1e-3, 20.0, 0.9, 100)
    rep.add("EstimateQuantile", q_r == q_g, "ref %.17g gpu %.17g" % (q_r, q_g))
    new_r.build_field(cfg["radius"], rt)
    new_g.build_field(cfg["radius"], rt)
    fr_, fg_ = new_r.field(), new_g.field()
    rep.exact("field ikl", fr_[:, :, 1], fg_[:, :, 1])
    has = fr_[:, :, 1] >= 0
    rep.exact("field dist (where set)", fr_[:, :, 0][has], fg_[:, :, 0][has])
    # single evaluations of TryVelRot
    k0 = old_r.knum()
    pnum = (k0 + 3) & ~3
    rng = np.random.default_rng(3)
    res_prev = np.zeros(pnum)
    Xs = [np.zeros(6), np.array([0.002, -0.001, 0.0005, 0.001, -0.002, 0.003]),
          np.array([-0.004, 0.003, -0.001, -0.003, 0.001, -0.004])]
    for xi, X in enumerate(Xs):
        for (rw, pj) in ((False, True), (True, True), (False, False)):
            s_r, J_r, F_r, res_r = new_r.try_vel_rot(old_r, X, rw, pj, cfg["match_thresh"], q_r,
                                                     cfg["match_num_thresh"], cfg["reweight"], res_prev)
            mf_r = old_r.keylines()["m_id_f"].copy()
            s_g, J_g, F_g, res_g = new_g.try_vel_rot(old_g, X, rw, pj, cfg["match_thresh"], q_r,
                                                     cfg["match_num_thresh"], cfg["reweight"], res_prev)
            mf_g = old_g.keylines()["m_id_f"]
            tag = "TryVelRot X%d rw=%d pj=%d" % (xi, rw, pj)
            rep.close(tag + " score", s_r, s_g, 1e-10)
            if pj:
                rep.close(tag + " JtJ", J_r, J_g, 1e-9, atol=1e-9 * np.abs(J_r).max())
                rep.close(tag + " JtF", F_r, F_g, 1e-9, atol=1e-9 * np.abs(F_r).max())
            rep.exact(tag + " m_id_f", mf_r, mf_g)
            kl0 = old_r.keylines()
            used = (kl0["s_rho"] <= q_r)
            rep.close(tag + " DResidualNew", res_r[:k0][used], res_g[used], 1e-12, atol=1e-12)
            if pj and not rw:
                res_prev = res_r.copy()
                res_prev[~np.isfinite(res_prev)] = 0
    # full minimisation
    V0, W0 = np.zeros(3), np.zeros(3)
    old_r.set_keylines(_seed_depth(old_r.keylines()))
    m_r = new_r.minimizer_rv(old_r, V0, W0, cfg["match_thresh"], cfg["iter_max"], cfg["init_type"], cfg["reweight"],
                             q_r, cfg["match_num_thresh"], cfg["init_iter"])
    new_g.set_frame_count(0)
    m_g = new_g.minimizer_rv(old_g, V0, W0, cfg["match_thresh"], cfg["iter_max"], cfg["init_type"], cfg["reweight"],
                             q_r, cfg["match_num_thresh"], cfg["init_iter"])
    rep.add("Minimizer_RV values", True, "ref V=%s W=%s F=%.6g" % (m_r["V"], m_r["W"], m_r["F"]))
    rep.close("Minimizer_RV V", m_r["V"], m_g["V"], 0.0, atol=1e-9)     # SURVEY 8(c): abs 1e-9
    rep.close("Minimizer_RV W", m_r["W"], m_g["W"], 0.0, atol=1e-9)
    rep.close("Minimizer_RV F", m_r["F"], m_g["F"], 1e-8)
    rep.close("Minimizer_RV RVel", m_r["RVel"], m_g["RVel"], 1e-8, atol=1e-9 * np.abs(m_r["RVel"]).max())
    rep.close("Minimizer_RV RW0", m_r["RW0"], m_g["RW0"], 1e-8, atol=1e-9 * np.abs(m_r["RW0"]).max())
    rep.close("Minimizer_RV W_X", m_r["W_X"], m_g["W_X"], 1e-8, atol=1e-9 * np.abs(m_r["W_X"]).max())
    rep.close("Minimizer_RV rel_err_score", m_r["rel_err_score"], m_g["rel_err_score"], 1e-8)
    rep.exact("Minimizer_RV m_id_f", old_r.keylines()["m_id_f"], old_g.keylines()["m_id_f"])
    return m_r


# ---- rotations for SO3<>(M).ln(): every branch of so3.h:288-334 -------------------------------------------------------
def rot(axis, deg):
    """the rotation by deg degrees about coordinate axis 0, 1 or 2"""
    a = np.deg2rad(deg)
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    R = np.eye(3)
    R[i, i], R[i, j], R[j, i], R[j, j] = c, -s, s, c
    return R


def rodrigues(w):
    w = np.asarray(w, np.float64)
    t = np.linalg.norm(w)
    if t == 0:
        return np.eye(3)
    k = w / t
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(t) * Kx + (1 - np.cos(t)) * Kx @ Kx


def so3_ln_cases():
    """name -> matrix: cos(angle) above sqrt(1/2), between +-sqrt(1/2), below -sqrt(1/2) with the largest diagonal
    term d0, d1 or d2 (the three sub-branches) and with the axis against r2 (the sign flip), the identity, and matrices
    that are not orthonormal (coerce)."""
    rng = np.random.default_rng(12)
    out = {"identity": np.eye(3), "small": rodrigues([0.02, -0.01, 0.03]), "cos_above": rodrigues([0.3, -0.4, 0.2]),
           "cos_between": rodrigues([0.9, 1.1, -0.6]), "cos_between_90": rot(0, 90.0)}
    for ax in range(3):
        w = np.full(3, 0.15)
        w[ax] = 2.8
        out["cos_below_d%d" % ax] = rodrigues(w)
        out["cos_below_d%d_flip" % ax] = rodrigues(-w)
    out["cos_below_179.9"] = rodrigues(np.deg2rad(179.9) * np.array([0.6, -0.64, 0.48]))
    for k, name in enumerate(("above", "between", "below")):
        w = rng.normal(0, 1, 3)
        w *= [0.4, 1.5, 2.9][k] / np.linalg.norm(w)
        out["coerce_" + name] = rodrigues(w) + rng.normal(0, 2e-3, (3, 3))
    return out



def so3_ln_branch(R):
    """(branch, sub-branch, flip) of SO3<>(M).ln() for M = R, from the lines of so3.h:288-334 on the coerced matrix"""
    m = R.copy()
    for i in range(3):   # Gram-Schmidt on the rows, as coerce
        for j in range(i):
            m[i] -= m[j] * (m[j] @ m[i])
        m[i] /= np.sqrt(m[i] @ m[i])
    c = (np.trace(m) - 1) / 2
    if c > np.sqrt(0.5):
        return "above", None, False
    if c > -np.sqrt(0.5):
        return "between", None, False
    d = (np.diag(m) - c) ** 2
    sub = 0 if d[0] > d[1] and d[0] > d[2] else 1 if d[1] > d[2] else 2
    out = np.array([m[2, 1] - m[1, 2], m[0, 2] - m[2, 0], m[1, 0] - m[0, 1]]) / 2
    r2 = np.array([[np.diag(m)[0] - c, (m[1, 0] + m[0, 1]) / 2, (m[0, 2] + m[2, 0]) / 2],
                   [(m[1, 0] + m[0, 1]) / 2, np.diag(m)[1] - c, (m[2, 1] + m[1, 2]) / 2],
                   [(m[0, 2] + m[2, 0]) / 2, (m[2, 1] + m[1, 2]) / 2, np.diag(m)[2] - c]])[sub]
    return "below", sub, bool(r2 @ out < 0)


# ---- the mapper stages' seeded cases (tests/test_gpu_mapper_states.py, tests/test_gpu_map_chain_states.py) ------------
MIN_HITS = 50          # keylines (or tie groups, bins ...) a case must put on its target branch


def _compare(kl_r, kl_g, fields, matched_fields=()):
    """Bitwise comparison of keyline fields; matched_fields only where the reference has m_id >= 0."""
    out = []
    if len(kl_r) != len(kl_g):
        return ["kn %d vs %d" % (len(kl_r), len(kl_g))]
    for f in fields:
        out.append(_diff(f, kl_r[f], kl_g[f]))
    mk = kl_r["m_id"] >= 0
    for f in matched_fields:
        out.append(_diff(f + " (matched)", kl_r[f][mk], kl_g[f][mk]))
    return [o for o in out if o]


def _cut(kl, mask, k):
    """The first k keylines of a detected map and its mask without the others (a map cut at kl_max = k)."""
    m = mask.copy()
    m[m >= k] = -1
    return kl[:k].copy(), m


def _search_setup(bench, kl_new, V, BackRot, max_radius, loc_unc):
    """NumPy restatement of search_match's set-up lines (edge_tracker.cpp:179-229): branch, search window and t_steps of
    every new keyline.  float64 like the reference, the projected point rounded to float as Point2DF does."""
    zf = bench.zfm
    Vb = BackRot @ np.asarray(V, np.float64)
    pm = kl_new["p_m"].astype(np.float64)
    p3 = np.stack([pm[:, 0], pm[:, 1], np.full(len(pm), zf)], 1) @ BackRot.T
    pmx = (p3[:, 0] * zf / p3[:, 2]).astype(np.float32).astype(np.float64)
    pmy = (p3[:, 1] * zf / p3[:, 2]).astype(np.float32).astype(np.float64)
    k_rho = kl_new["rho"] * zf / p3[:, 2]
    ks = kl_new["s_rho"]
    t_x = -(Vb[0] * zf - Vb[2] * pmx)
    t_y = -(Vb[1] * zf - Vb[2] * pmy)
    norm_t = np.sqrt(t_x * t_x + t_y * t_y)
    perp = ~(norm_t > 1e-6)
    with np.errstate(all="ignore"):
        dq_rho = norm_t * k_rho
        dq_min = np.maximum(0.0, norm_t * (k_rho - ks)) - loc_unc
        dq_max_raw = norm_t * (k_rho + ks)
        dq_max = np.minimum(max_radius, dq_max_raw) + loc_unc
        mid = ~perp & (dq_rho > dq_max)
        dq_c = np.where(mid, (dq_max + dq_min) / 2, dq_rho)
        span = np.where(mid, dq_c, np.maximum(dq_max - dq_rho, dq_rho - dq_min))
        t_steps = np.floor(span + 0.5).astype(np.int64)
        t_steps[perp] = int(max_radius + loc_unc)
        # direction of the probes (perpendicular search: the gradient)
        ux = np.where(perp, kl_new["m_m"][:, 0] / kl_new["n_m"], t_x / np.where(perp, 1.0, norm_t))
        uy = np.where(perp, kl_new["m_m"][:, 1] / kl_new["n_m"], t_y / np.where(perp, 1.0, norm_t))
        lo = np.where(perp, -(max_radius + loc_unc), dq_min)
        hi = np.where(perp, max_radius + loc_unc, dq_max)
    x0, y0 = pmx + bench.cam["ppx"], pmy + bench.cam["ppy"]
    ends = [(x0 + ux * lo, y0 + uy * lo), (x0 + ux * hi, y0 + uy * hi)]
    w, h = bench.cam["w"], bench.cam["h"]
    edges = np.zeros((len(pm), 4), bool)   # a probe of the window lies left / right / above / below the image
    for ex, ey in ends:
        edges |= np.stack([ex < -0.5, ex >= w - 0.5, ey < -0.5, ey >= h - 0.5], 1)
    edges &= (t_steps > 0)[:, None]
    return dict(perp=perp, mid=mid, normal=~perp & ~mid, t_steps=t_steps,
                cut=~perp & (dq_max_raw > max_radius), edges=edges)


V_TYP = np.array([0.004, -0.003, 0.0005])
RV_SPD = np.array([[2e-4, 5e-5, -3e-5], [5e-5, 1e-4, 2e-5], [-3e-5, 2e-5, 4e-4]])
DM_BASE = dict(V=V_TYP, RVel=np.eye(3) * 1e-4, BackRot=np.eye(3), thr_mod=1.0, thr_ang=45.0, radius=40.0, loc_unc=2.0)
# name -> (overrides of DM_BASE, {branch: least keyline count})
DM_CASES = {
    "V0": (dict(V=np.zeros(3), RVel=np.zeros((3, 3))), {"perp": -1}),
    "V1e-9": (dict(V=np.array([1e-9, 0, 0])), {"perp": -1}),
    "V0_loc0.5": (dict(V=np.zeros(3), loc_unc=0.5), {"perp": -1}),
    "V0_radius12.5_loc0": (dict(V=np.zeros(3), radius=12.5, loc_unc=0.0), {"perp": -1}),
    "Vz": (dict(V=np.array([0, 0, 0.02])), {"mid": MIN_HITS, "normal": MIN_HITS}),
    "fast": (dict(V=np.array([0.06, -0.05, 0.03]), RVel=RV_SPD), {"mid": MIN_HITS, "cut": MIN_HITS}),
    "fast_radius12.5": (dict(V=np.array([-0.04, 0.07, -0.02]), radius=12.5, loc_unc=0.5), {"mid": MIN_HITS, "cut": MIN_HITS}),
    "typ_radius12.5_loc0": (dict(radius=12.5, loc_unc=0.0), {"normal": MIN_HITS, "cut": MIN_HITS}),
    "loc0": (dict(loc_unc=0.0), {"normal": MIN_HITS}),
    "loc0.5": (dict(loc_unc=0.5), {"normal": MIN_HITS}),
    "loc5": (dict(loc_unc=5.0), {"normal": MIN_HITS}),
    "RVel0": (dict(RVel=np.zeros((3, 3))), {"normal": MIN_HITS}),
    "RVel_spd": (dict(RVel=RV_SPD), {"normal": MIN_HITS}),
    "rot_x3": (dict(BackRot=rot(0, 3.0)), {"normal": MIN_HITS}),
    "rot_y3": (dict(BackRot=rot(1, -3.0)), {"normal": MIN_HITS}),
    "rot_z3": (dict(BackRot=rot(2, 3.0)), {"normal": MIN_HITS}),
    "rot_y25": (dict(BackRot=rot(1, 25.0)), {"normal": MIN_HITS}),
    "rot_y-25": (dict(BackRot=rot(1, -25.0), V=V_TYP[[1, 0, 2]]), {"normal": MIN_HITS}),
    "ang10_mod0.1": (dict(thr_ang=10.0, thr_mod=0.1), {"normal": MIN_HITS}),
    "ang90_mod10": (dict(thr_ang=90.0, thr_mod=10.0), {"normal": MIN_HITS}),
    "ang45_mod10": (dict(thr_mod=10.0, V=np.zeros(3)), {"perp": -1}),
    "tsteps0to8": (dict(V=np.array([0.0015, 0.001, 0.0]), loc_unc=0.0), {"tsteps": MIN_HITS}),
}


def _reg_gates(kl, thresh):
    """NumPy restatement of Regularize_1_iter's two gates (edge_tracker.cpp:98-118) for keylines with both neighbours."""
    ni, pi = kl["n_id"], kl["p_id"]
    nb = (ni >= 0) & (pi >= 0)
    n, p = ni[nb], pi[nb]
    d = kl["rho"][n] - kl["rho"][p]
    g1 = ~(d * d > kl["s_rho"][n] ** 2 + kl["s_rho"][p] ** 2)
    mm = kl["m_m"]
    alpha = ((mm[n, 0] * mm[p, 0] + mm[n, 1] * mm[p, 1]) / (kl["n_m"][n] * kl["n_m"][p])).astype(np.float64)
    g2 = ~(alpha - thresh < 0)
    return nb.sum(), g1, g2



EKF_CASES = {   # name -> (vel, q_abs, loc_unc, fraction of matched keylines set to rho = 1)
    "vel0": (np.zeros(3), 1e-4, 1.0, 0.0),                       # H = 0
    "vel0_loc0": (np.zeros(3), 1e-4, 0.0, 0.0),                  # H = 0 and S = 0: K = NaN
    "typical": (np.array([0.004, -0.003, 0.0005]), 1e-4, 1.0, 0.0),
    "typical_q0_loc0": (np.array([0.004, -0.003, 0.0005]), 0.0, 0.0, 0.0),
    "vz-1": (np.array([0.003, 0.002, -1.0]), 1e-4, 1.0, 0.3),     # rho = 1: rho_p = inf
    "vz+0.5": (np.array([0.01, -0.004, 0.5]), 1e-4, 1.0, 0.0),
    "vz+0.5_q0": (np.array([0.01, -0.004, 0.5]), 0.0, 1.0, 0.0),
    "vz-0.06": (np.array([0.002, 0.001, -0.06]), 1e-4, 1.0, 0.0),   # rho > ~9: rho_p beyond RHO_MAX or negative
}

"""Seeded edge-map states for the IMU-mode stages (TryVel, Minimizer_V<double>, ExtRotVel) and what the reference does on
them, shared by tests/test_cpu_imu_states.py (the states are valid) and tests/test_gpu_imu_states.py (the device agrees).

The maps are test_gpu_minimiser_forms.py's: frame 11 of the EuRoC-like sequence as the reference detects it is the new
map with its field; the old map is frame 10's keylines tiled with sub-pixel jitter up to K0, with the depth, gate and
gradient state each case needs.  FrameCount (global_tracker.cpp:854's min(MatchNumThresh, FrameCount)) is raised on
the reference by cheap minimisations on a one-keyline map, on the device by Map.set_frame_count.

Two NumPy restatements prove that a case reaches what it is for:
- tv_setup: TryVel's per-keyline set-up (global_tracker.cpp:843-896): the min_mod, s_rho and m_num gates, z_p <= 0,
  the projection, its rounding and the image border, and, for each miss inside the image, the last match before it whose
  fi it inherits (Residuals[ikl] = fabs(fi), :917 with the function-level fi of :839).  It never restates the sums.
- minimizer_v: Minimizer_V<double> (global_tracker.cpp:1036-1093) on the reference's own TryVel, recording every
  evaluation and every LM decision with its relative margin."""
import numpy as np

from parity_util import DOG_THRESH, EUROC_CFG, PLANE_FIT, POS_NEG, parity_frames
from test_gpu_minimiser_forms import _runs, _tile, _turn

CFG = EUROC_CFG
KEYLINE_MAX = 50000
MIN_HITS = 50            # keylines, runs or decisions a case must put on its target
MIN_RUNS = 10            # runs of carried misses per boundary class
MARGIN = 1e-9            # least relative margin of an LM decision (F against Fnew)
H_TINY = 1e-11           # steps at most this long decide nothing that moves V
CUT = 1e9                # TooN SVD<>: singular values s with s * 1e9 <= smax are dropped
RW = CFG["reweight"]     # ReweigthDistance (also ExtRotVel's Huber threshold in the IMU flow)
Q = 0.3                  # s_rho_min
LOC_UNC = 1.0            # LocationUncertainty
V_FAR = np.array([0.02, -0.015, 0.01])
BLOCK, WARP = 256, 32    # STAGE_T (csrc/stage_reduce.cuh): k_tv_eval / k_extrotvel run 256-keyline blocks of eight warps

# path codes of tv_setup
P_MOD, P_SRHO, P_MNUM, P_ZP, P_BORDER, P_IN = range(6)


# ---- the states --------------------------------------------------------------------------------------------------------
TV = {}
for _k in (0, 1, 31, 32, 33, 255, 256, 257, 15000, 50000):
    TV["K%d" % _k] = dict(K0=_k, want=["evals"])
TV["K15000_min_mod_off"] = dict(K0=15000, min_mod=0.0, want=["evals"])
for _mnt in (0, 3):
    for _fc in (0, 2, 1000):
        TV["gates_mnt%d_fc%d" % (_mnt, _fc)] = dict(K0=15000, kind="gates", mnt=_mnt, fc=_fc, want=["gates"])
TV["stale"] = dict(K0=15000, kind="stale", want=["stale", "miss_kinds", "reweight"])
TV["stale_gated"] = dict(K0=20000, kind="stale", gated_runs=True, want=["stale", "gated_between", "reweight"])
TV["stale_50000"] = dict(K0=50000, kind="stale", want=["stale", "reweight"])
TV["z_p"] = dict(K0=8000, kind="z_p", poses=["z0", "zero", "near"], want=["z_p"])
TV["border"] = dict(K0=15000, kind="border", poses=["zero", "near", "near2"], want=["border"])
TV["min_mod"] = dict(K0=15000, kind="min_mod", want=["min_mod"])

MV = {}
for _m in (0, 1, 5, 10):
    for _p in ("near", "far"):
        MV["iter%d_%s" % (_m, _p)] = dict(tv="K15000", iter_max=_m, prior=_p, want=["rejected"] if _m == 10 else [])
# once converged every step is rejected: u *= v overflows to inf (at the 46th step) and the steps after it are NaN poses
MV["u_overflow"] = dict(tv="stale", iter_max=60, prior="near", want=["u_inf"])
MV["all_gated"] = dict(tv="all_gated", iter_max=5, prior="near", want=["jtj_zero"])
MV["two_usable"] = dict(tv="two_usable", iter_max=5, prior="near", want=["degenerate"])
MV["empty"] = dict(tv="K0", iter_max=5, prior="near", want=["empty"])
MV["stale"] = dict(tv="stale_gated", iter_max=5, prior="zero", want=["stale"])
MV["gates_mnt3_fc2"] = dict(tv="gates_mnt3_fc2", iter_max=5, prior="zero", want=["gates"])
MV["gates_mnt3_fc1000"] = dict(tv="gates_mnt3_fc1000", iter_max=5, prior="far", want=["gates"])
TV["all_gated"] = dict(K0=3000, kind="all_gated", want=[])
TV["two_usable"] = dict(K0=3000, kind="two_usable", want=[])

ERV = {}
for _n in (0, 1, 5, 6, 7, 255, 256, 257, 15000, 50000):
    ERV["n%d" % _n] = dict(kind="count", n=_n, want=["count"])
ERV["huber"] = dict(kind="count", n=4000, shift=4.0, want=["huber"])
for _r in range(1, 6):
    ERV["rank%d" % _r] = dict(kind="rank", rank=_r, want=["rank"])
for _c in (1e6, 1e7, 5e7):
    ERV["cond%.0e" % _c] = dict(kind="cond", cond=_c, want=["cond"])
ERV["z_inf"] = dict(kind="z_inf", want=["nan"])


# ---- the reference side -------------------------------------------------------------------------------------------------
def mat3_inv(A):
    """util::Matrix3x3Inv (include/UtilLib/toon_util.h:32-41): cofactors over TooN::determinant (Gaussian elimination with
    partial pivoting, TooN/determinant.h)"""
    A = np.asarray(A, np.float64)
    a = A.ravel()
    t = np.array([a[8] * a[4] - a[7] * a[5], -(a[8] * a[1] - a[7] * a[2]), a[5] * a[1] - a[4] * a[2],
                  -(a[8] * a[3] - a[6] * a[5]), a[8] * a[0] - a[6] * a[2], -(a[5] * a[0] - a[3] * a[2]),
                  a[7] * a[3] - a[6] * a[4], -(a[7] * a[0] - a[6] * a[1]), a[4] * a[0] - a[3] * a[1]])
    M = [[np.float64(A[r, c]) for c in range(3)] for r in range(3)]   # (IEEE division: x / 0 is inf or NaN)
    det = np.float64(1.0)
    with np.errstate(all="ignore"):
        for i in range(3):
            am, mx = i, abs(M[i][i])
            for k in range(i + 1, 3):
                if abs(M[k][i]) > mx:
                    am, mx = k, abs(M[k][i])
            piv = M[am][i]
            if am != i:
                det *= -1
                M[i], M[am] = M[am], M[i]
            det *= M[i][i]
            if det == 0:
                det = 0.0
                break
            for u in range(i + 1, 3):
                f = M[u][i] / piv
                for c in range(i + 1, 3):
                    M[u][c] = M[u][c] - f * M[i][c]
        return (t / np.float64(det)).reshape(3, 3)


def _dot(a, b):
    s = 0.0
    for x, y in zip(a, b):
        s += x * y
    return s


class RefBase:
    """Frames 10 and 11 detected on the reference, and the states built from them (cached)."""

    def __init__(self):
        from oracle import refapi
        self.refapi = refapi
        self.cam = c = CFG["cam"]
        refs = [self.refmap() for _ in range(2)]
        t, l = CFG["thresh"], 0
        kl, mask = [], []
        for r, fr in zip(refs, parity_frames(CFG)):
            r.rgb2bw(fr)
            r.build()
            _, t, l = r.detect(PLANE_FIT, POS_NEG, DOG_THRESH, CFG["kl_max"], t, l, CFG["kl_ref"], CFG["gain"],
                               CFG["tmax"], CFG["tmin"])
            kl.append(r.keylines())
            mask.append(r.mask())
        _, self.rt = refs[1].reestimate(CFG["track_points"], 100)
        self.kl10, self.kl11, self.mask11 = kl[0], kl[1], mask[1]
        self.empty = np.full((c["h"], c["w"]), -1, np.int32)
        self.zfm = float(np.float32((np.float32(c["zfx"]) + np.float32(c["zfy"])) / np.float32(2)))
        self.pp = (float(np.float32(c["ppx"])), float(np.float32(c["ppy"])))
        self.min_mod = float(np.float32(self.rt))
        new, old = self.ref_maps(_tile(self.kl10, 8000, np.random.default_rng(1)), 0)
        self.field = new.field()[:, :, 1].copy()
        m = new.minimizer_v(old, np.zeros(3), CFG["match_thresh"], 10, Q, 0, RW, self.min_mod)
        self.near = m["V"].copy()
        self.cache = {}

    def refmap(self):
        c = self.cam
        return self.refapi.RefMap(c["w"], c["h"], c["ppx"], c["ppy"], c["zfx"], c["zfy"], CFG["sigma0"], CFG["ksigma"])

    def ref_maps(self, old_kl, fc):
        """fresh reference maps: new = frame 11 with its field, FrameCount = fc; old = old_kl"""
        new = self.refmap()
        new.set_keylines(self.kl11)
        new.set_mask(self.mask11, len(self.kl11))
        new.build_field(CFG["radius"], self.rt)
        if fc:   # FrameCount is private: fc cheap minimisations on a one-keyline map raise it
            one = self.refmap()
            one.set_keylines(self.kl10[:1])
            one.set_mask(self.empty, 1)
            for _ in range(fc):
                new.minimizer_rv(one, np.zeros(3), np.zeros(3), 0.5, 0, 0, 2.0, 1e3, 0, 0)
        old = self.refmap()
        old.set_keylines(old_kl)
        old.set_mask(self.empty, len(old_kl))
        return new, old

    def pose(self, name):
        return {"zero": np.zeros(3), "near": self.near, "near2": 1.5 * self.near + np.array([2e-3, -1e-3, 5e-3]),
                "far": V_FAR, "z0": np.array([0.0, 0.0, -2.0])}[name]

    # ---- TryVel -------------------------------------------------------------------------------------------------------
    def tv_spec(self, name):
        sp = dict(K0=0, kind=None, mnt=0, fc=0, min_mod=self.min_mod, mt=CFG["match_thresh"], q=Q, rw=RW,
                  poses=["zero", "near", "near2", "near"])
        sp.update(TV[name])
        return sp

    def tv_old(self, name, sp):
        rng = np.random.default_rng(sum(map(ord, "tv_" + name)))
        K0 = sp["K0"]
        kl = _tile(self.kl10, K0, rng)
        ev = {}
        kind = sp["kind"]
        if kind == "gates":   # s_rho log-spread with exactly q and one ulp above; m_num 0..10, a third of them 0..2
            kl["s_rho"] = np.exp(rng.uniform(np.log(0.05), np.log(3.0 * Q), K0))
            eq = rng.random(K0) < 0.05
            up = ~eq & (rng.random(K0) < 0.05)
            kl["s_rho"][eq] = Q
            kl["s_rho"][up] = np.nextafter(Q, np.inf)
            m = rng.integers(0, 11, K0)
            low = rng.random(K0) < 0.3
            m[low] = rng.integers(0, 3, int(low.sum()))
            kl["m_num"] = m
            ev.update(s_rho_eq=int(eq.sum()), s_rho_ulp=int(up.sum()))
        elif kind == "stale":   # runs of misses from the first keyline and across warp and block boundaries
            st = {0}
            for s in rng.choice(np.arange(BLOCK, K0, BLOCK), min(24, K0 // BLOCK), replace=False):
                st.add(int(s) - int(rng.integers(1, 20)))
            for s in rng.choice(np.arange(WARP, K0, WARP), min(60, K0 // WARP), replace=False):
                st.add(int(s) - int(rng.integers(1, 12)))
            st = sorted(st)
            _runs(kl, rng, st, [int(rng.integers(40, 120)) for _ in st])
            if sp.get("gated_runs"):   # gated keylines between a match and the misses that inherit its fi
                sk = [s + 3 for s in st[1::2]]
                _runs(kl, rng, sk, [int(rng.integers(5, 30)) for _ in sk], skipped=True)
        elif kind == "z_p":   # 1/rho + V_z at V_z = -2: exactly 0 (rho = 0.5), negative, positive
            u = rng.random(K0)
            kl["rho"] = np.where(u < 0.4, 0.5, np.where(u < 0.7, rng.uniform(0.55, 2.0, K0), rng.uniform(0.1, 0.45, K0)))
        elif kind == "border":   # at V = 0 on x in {0, 1, w-2, w-1} (and the same for y); 0.2 px off the integer
            w, h = self.cam["w"], self.cam["h"]
            n = K0 // 8
            sel = rng.permutation(K0)[:8 * n].reshape(8, n)
            for a, tx in enumerate((0, 1, w - 2, w - 1)):
                kl["p_m"][sel[a], 0] = np.float32(tx + 0.2 * rng.choice([-1, 1], n) - self.pp[0])
            for a, ty in enumerate((0, 1, h - 2, h - 1)):
                kl["p_m"][sel[4 + a], 1] = np.float32(ty + 0.2 * rng.choice([-1, 1], n) - self.pp[1])
            kl["rho"][sel.ravel()] = 1.0
        elif kind == "min_mod":   # n_m exactly min_mod (kept) and one float ulp below (gated)
            mm = np.float32(sp["min_mod"])
            u = rng.random(K0)
            kl["n_m"][u < 0.05] = mm
            kl["n_m"][(u >= 0.05) & (u < 0.1)] = np.nextafter(mm, np.float32(-np.inf))
        elif kind == "all_gated":
            kl["s_rho"] = 10.0 * Q
        elif kind == "two_usable":
            kl["s_rho"][2:] = 10.0 * Q
        return kl, ev

    def tv_state(self, name):
        key = ("tv", name)
        if key in self.cache:
            return self.cache[key]
        sp = self.tv_spec(name)
        kl, ev = self.tv_old(name, sp)
        new, old = self.ref_maps(kl, sp["fc"])
        res = np.zeros(sp["K0"])
        evals = []
        for p in sp["poses"]:
            V = self.pose(p)
            s, J, F, out = new.try_vel(old, V, sp["mt"], sp["q"], sp["mnt"], res, sp["rw"], sp["min_mod"])
            evals.append(dict(V=V, res_in=res, res=out, s=s, JtJ=J, JtF=F, m_id_f=old.keylines()["m_id_f"].copy()))
            res = out
        st = dict(sp=sp, kl=kl, ev=ev, evals=evals)
        self.cache[key] = st
        return st

    def tv_setup(self, kl, V, sp):
        """TryVel's set-up per keyline: path code, rounded pixel (x, y), in-image field keyline (or -1)"""
        K0 = len(kl)
        gate = min(sp["mnt"], sp["fc"])
        path = np.full(K0, P_IN)
        with np.errstate(all="ignore"):
            zp = 1.0 / kl["rho"] + V[2]
            rho_p = 1.0 / zp
            pm = kl["p_m"].astype(np.float64)
            pjx = rho_p * (V[0] * self.zfm - V[2] * pm[:, 0]) + pm[:, 0]
            pjy = rho_p * (V[1] * self.zfm - V[2] * pm[:, 1]) + pm[:, 1]
            fx, fy = np.trunc(pjx + self.pp[0] + 0.5), np.trunc(pjy + self.pp[1] + 0.5)
        w, h = self.cam["w"], self.cam["h"]
        out = ~((fx >= 1) & (fy >= 1) & (fx < w - 1) & (fy < h - 1))
        x = np.where(out, 0, fx).astype(np.int64)
        y = np.where(out, 0, fy).astype(np.int64)
        path[out] = P_BORDER
        path[~(zp > 0)] = P_ZP
        path[kl["m_num"].astype(np.int64) < gate] = P_MNUM
        path[kl["s_rho"] > sp["q"]] = P_SRHO
        if sp["min_mod"] > 0:
            path[kl["n_m"] < np.float32(sp["min_mod"])] = P_MOD
        fk = np.where(path == P_IN, self.field[y, x], -1)
        return path, x, y, fk, zp

    def tv_check(self, st):
        """Restate each evaluation's set-up and the stale carry against the reference's outputs; returns (errors, hits)"""
        sp, kl = st["sp"], st["kl"]
        K0 = sp["K0"]
        idx = np.arange(K0)
        errs = []
        hits = dict(st["ev"])
        runs = {}
        add = lambda k, n: hits.__setitem__(k, hits.get(k, 0) + int(n))   # noqa: E731
        for k, e in enumerate(st["evals"]):
            path, x, y, fk, zp = self.tv_setup(kl, e["V"], sp)
            mt = e["m_id_f"] >= 0
            if (mt & (path != P_IN)).any():
                errs.append("eval %d: %d matches outside the restated in-image set" % (k, int((mt & (path != P_IN)).sum())))
            if not np.array_equal(e["res"][path != P_IN], e["res_in"][path != P_IN]):
                errs.append("eval %d: the reference wrote residuals the restatement does not reach" % k)
            miss = (path == P_IN) & ~mt
            lastm = np.maximum.accumulate(np.where(mt, idx, -1))
            prev = np.concatenate([[-1], lastm])[:K0].astype(np.int64)
            want = np.where(prev >= 0, e["res"][np.maximum(prev, 0)], 0.0)
            if not np.array_equal(e["res"][miss], want[miss]):
                errs.append("eval %d: %d misses do not carry the last match's fi" % (k, int((e["res"][miss] != want[miss]).sum())))
            j, i = prev[miss], idx[miss]
            cls = np.where(j < 0, "start", np.where(j // BLOCK != i // BLOCK, "block",
                                                    np.where(j // WARP != i // WARP, "warp", "none")))
            for c in ("start", "warp", "block"):
                add("carried_" + c, (cls == c).sum())
                runs[c] = runs.get(c, 0) + len(set(j[cls == c].tolist()))
            if K0:
                gated = np.cumsum(np.isin(path, (P_MOD, P_SRHO, P_MNUM)))
                between = gated[np.maximum(i - 1, 0)] - gated[np.maximum(j, 0)]
                add("carried_over_gated", ((cls != "none") & (j >= 0) & (between > 0)).sum())
            add("empty_field_miss", (miss & (fk < 0)).sum())
            add("test_f_k_miss", (miss & (fk >= 0)).sum())
            add("matched", mt.sum())
            add("reweighted", ((path != P_MOD) & (path != P_SRHO) & (path != P_MNUM) & (e["res_in"] > sp["rw"])).sum())
            add("z_p_zero", ((path == P_ZP) & (zp == 0)).sum())
            add("z_p_neg", ((path == P_ZP) & (zp < 0)).sum())
            add("border", (path == P_BORDER).sum())
            add("gate_m_num", (path == P_MNUM).sum())
            add("gate_s_rho", (path == P_SRHO).sum())
            add("gate_min_mod", (path == P_MOD).sum())
            if k == 0 and sp["kind"] == "border":
                px = np.trunc(kl["p_m"][:, 0].astype(np.float64) + self.pp[0] + 0.5)
                py = np.trunc(kl["p_m"][:, 1].astype(np.float64) + self.pp[1] + 0.5)
                w, h = self.cam["w"], self.cam["h"]
                for t in (0, 1, w - 2, w - 1):
                    add("x=%d" % t, (px == t).sum())
                for t in (0, 1, h - 2, h - 1):
                    add("y=%d" % t, (py == t).sum())
            if sp["kind"] == "min_mod":
                mm = np.float32(sp["min_mod"])
                ok = (kl["s_rho"] <= sp["q"])
                add("n_m_eq_used", (ok & (kl["n_m"] == mm)).sum())
                add("n_m_ulp_gated", (ok & (kl["n_m"] == np.nextafter(mm, np.float32(-np.inf)))).sum())
        hits.update({"runs_" + c: n for c, n in runs.items()})
        return errs, hits

    def tv_vacuous(self, st, hits):
        sp = st["sp"]
        msgs = []
        for w in sp["want"]:
            if w == "gates":
                if min(hits["s_rho_eq"], hits["s_rho_ulp"]) < MIN_HITS:
                    msgs.append("s_rho at and one ulp above q: %d, %d" % (hits["s_rho_eq"], hits["s_rho_ulp"]))
                if min(sp["mnt"], sp["fc"]) > 0 and hits["gate_m_num"] < MIN_HITS:
                    msgs.append("the m_num gate closes for %d keylines" % hits["gate_m_num"])
            elif w == "stale":
                for c in ("start", "warp", "block"):
                    if hits.get("runs_" + c, 0) < (len(sp["poses"]) if c == "start" else MIN_RUNS):
                        msgs.append("%d runs carried across %s" % (hits.get("runs_" + c, 0), c))
                if sum(hits.get("carried_" + c, 0) for c in ("start", "warp", "block")) < MIN_HITS:
                    msgs.append("too few carried misses")
            elif w == "gated_between" and hits.get("carried_over_gated", 0) < MIN_HITS:
                msgs.append("%d carried misses over gated keylines" % hits.get("carried_over_gated", 0))
            elif w == "miss_kinds" and min(hits["empty_field_miss"], hits["test_f_k_miss"]) < MIN_HITS:
                msgs.append("misses: empty field %d, Test_f_k %d" % (hits["empty_field_miss"], hits["test_f_k_miss"]))
            elif w == "reweight" and hits["reweighted"] < MIN_HITS:
                msgs.append("%d reweighted keylines" % hits["reweighted"])
            elif w == "z_p" and min(hits["z_p_zero"], hits["z_p_neg"]) < MIN_HITS:
                msgs.append("z_p == 0: %d, z_p < 0: %d" % (hits["z_p_zero"], hits["z_p_neg"]))
            elif w == "border":
                c, h = self.cam, hits
                low = [k for k in h if (k.startswith("x=") or k.startswith("y=")) and h[k] < MIN_HITS]
                if low or len([k for k in h if k[:2] in ("x=", "y=")]) != 8:
                    msgs.append("border targets %s" % {k: h[k] for k in h if k[:2] in ("x=", "y=")})
            elif w == "min_mod" and min(hits["n_m_eq_used"], hits["n_m_ulp_gated"]) < MIN_HITS:
                msgs.append("n_m at min_mod %d, one ulp below %d" % (hits["n_m_eq_used"], hits["n_m_ulp_gated"]))
        return msgs

    # ---- Minimizer_V ----------------------------------------------------------------------------------------------------
    def mv_state(self, name):
        key = ("mv", name)
        if key in self.cache:
            return self.cache[key]
        sp = dict(MV[name])
        tv = self.tv_state(sp["tv"])
        a = tv["sp"]
        kl = tv["kl"]
        V0 = {"zero": np.zeros(3), "near": self.near, "far": V_FAR}[sp["prior"]]
        new, old = self.ref_maps(kl, a["fc"])
        drv, tr = minimizer_v(new, old, V0, sp["iter_max"], a)
        mf_drv = old.keylines()["m_id_f"].copy()
        new, old = self.ref_maps(kl, a["fc"])
        ref = new.minimizer_v(old, V0, a["mt"], sp["iter_max"], a["q"], a["mnt"], a["rw"], a["min_mod"])
        st = dict(sp=sp, a=a, kl=kl, V0=V0, drv=drv, tr=tr, ref=ref, m_id_f=old.keylines()["m_id_f"].copy(),
                  m_id_f_drv=mf_drv)
        self.cache[key] = st
        return st

    # ---- ExtRotVel ------------------------------------------------------------------------------------------------------
    def erv_keylines(self, sp, rng, s_rho_last=None):
        """the new map: frame 11's keylines tiled to K keylines, p_m_0 a few pixels from p_m, m_id >= 0 on the matched set"""
        kind = sp["kind"]
        K = 50000 if kind == "count" else 600
        kl = _tile(self.kl11, K, rng)
        kl["rho"] = np.exp(rng.uniform(np.log(0.3), np.log(2.0), K))
        sh = sp.get("shift", 1.0)
        kl["p_m_0"] = (kl["p_m"].astype(np.float64) + rng.uniform(-sh, sh, (K, 2))).astype(np.float32)
        kl["m_id"] = -1
        if kind == "count":
            n = sp["n"]
            if n in (5, 6, 7):      # around the first block boundary
                sel = np.arange(BLOCK - 3, BLOCK - 3 + n)
            elif n <= 257:          # a contiguous set across two blocks
                sel = np.arange(100, 100 + n)
            elif n < K:
                sel = np.sort(rng.choice(K, n, replace=False))
            else:
                sel = np.arange(K)
            kl["m_id"][sel] = rng.integers(0, len(self.kl10), len(sel))
        elif kind in ("rank", "cond"):
            r = sp.get("rank", 5)
            rows = kl[rng.choice(K, r + 1, replace=False)].copy()
            sel = np.arange(40, 340)
            kl[sel] = rows[np.arange(len(sel)) % r]             # r distinct rows, each repeated
            zero = np.arange(400, 450)                           # matched keylines without a gradient: zero rows
            kl[zero] = rows[0]
            kl["u_m"][zero] = 0
            kl["m_id"][sel] = 1
            kl["m_id"][zero] = 1
            if kind == "cond":                                   # one more row, scaled down by its s_y
                kl[500] = rows[r]
                kl["s_rho"][500] = s_rho_last
                kl["m_id"][500] = 1
        elif kind == "z_inf":   # 1/rho + vel_z == 0 on one matched keyline
            kl["rho"] = 0.25
            kl["m_id"][:300] = 1
            kl["rho"][150] = 0.5
        return kl

    def erv_vel(self, sp):
        return np.array([0.0, 0.0, -2.0]) if sp["kind"] == "z_inf" else self.near

    def erv_run(self, kl, V):
        m = self.refmap()
        m.set_keylines(kl)
        m.set_mask(self.empty, len(kl))
        return m.ext_rot_vel(V, LOC_UNC, RW)

    def erv_state(self, name):
        key = ("erv", name)
        if key in self.cache:
            return self.cache[key]
        sp = dict(ERV[name])
        seed = sum(map(ord, "erv_" + name))
        V = self.erv_vel(sp)
        s_last = None
        if sp["kind"] == "cond":   # the s_rho of the last row that puts cond(Wx) at the target: bisection in log s_rho
            lo, hi = np.log(1e-3), np.log(1e6)
            for _ in range(60):
                mid = 0.5 * (lo + hi)
                kl = self.erv_keylines(sp, np.random.default_rng(seed), np.exp(mid))
                s = np.linalg.svd(self.erv_run(kl, V)[1], compute_uv=False)
                if s[0] / s[-1] < sp["cond"]:
                    lo = mid
                else:
                    hi = mid
            s_last = np.exp(0.5 * (lo + hi))
        kl = self.erv_keylines(sp, np.random.default_rng(seed), s_last)
        ok, Wx, Rx, X = self.erv_run(kl, V)
        st = dict(sp=sp, kl=kl, V=V, ok=ok, Wx=Wx, Rx=Rx, X=X)
        self.cache[key] = st
        return st

    def erv_hits(self, st):
        """matched count and blocks, Huber-reweighted matches (|Y| > hub, restated in double), the spectrum of Wx"""
        kl, V = st["kl"], st["V"]
        m = kl["m_id"] >= 0
        info = dict(matched=int(m.sum()), blocks=len(set((np.nonzero(m)[0] // BLOCK).tolist())))
        with np.errstate(all="ignore"):
            rho_t = 1.0 / (1.0 / kl["rho"][m] + V[2])
            p0 = kl["p_m_0"][m].astype(np.float64)
            qt = p0 + rho_t[:, None] * (np.array([V[0], V[1]]) * self.zfm - V[2] * p0)
            Y = (kl["u_m"][m].astype(np.float64) * (kl["p_m"][m].astype(np.float64) - qt)).sum(1)
        info["huber"] = int((np.abs(Y) > RW).sum())
        if st["ok"] and np.isfinite(st["Wx"]).all() and np.abs(st["Wx"]).max() > 0:
            s = np.linalg.svd(st["Wx"], compute_uv=False)
            kept = s * CUT > s[0]
            info.update(kept=int(kept.sum()), cond=float(s[0] / s[kept][-1]),
                        cut_margin=float(min(np.min(s[kept] * CUT / s[0]), np.min(s[0] / (s[~kept] * CUT + 1e-300)))
                                         if (~kept).any() else np.min(s[kept] * CUT / s[0])))
        return info


def minimizer_v(new, old, V0, iter_max, a):
    """Minimizer_V<double> (global_tracker.cpp:1036-1093) with every evaluation done by the reference's TryVel.  Returns
    the outputs and a trace: evaluations (pose, residuals) and LM decisions (relative margin of F against Fnew, |h|, u)."""
    K0 = old.knum()
    tr = dict(evals=[], dec=[], rejected=0, u=[])
    res = np.zeros(K0)

    def tv(V):
        nonlocal res
        s, J, F, out = new.try_vel(old, V, a["mt"], a["q"], a["mnt"], res, a["rw"], a["min_mod"])
        tr["evals"].append(dict(V=np.array(V), res_in=res, res=out, s=s, JtJ=J))
        res = out
        return s, J, F

    V = np.array(V0, np.float64)
    F, JtJ, JtF = tv(V)
    v, u = 2.0, 1e-3 * JtJ.max()
    with np.errstate(all="ignore"):
        for _ in range(iter_max):
            ApI = JtJ + np.eye(3) * u
            inv = mat3_inv(ApI)
            h = np.array([_dot(inv[r], -JtF) for r in range(3)])
            Vn = V + h
            Fn, Jn, Fvn = tv(Vn)
            gain = (F - Fn) / _dot(0.5 * h, u * h - JtF)
            m = abs(F - Fn) / max(abs(F), abs(Fn), 1e-300) if np.isfinite(gain) else np.inf
            tr["dec"].append((float(m), float(np.linalg.norm(h)) if np.isfinite(h).all() else np.inf, u))
            if gain > 0:
                F, V, JtJ, JtF = Fn, Vn, Jn, Fvn
                u *= max(0.33, 1 - (2 * gain - 1) ** 3)
                v = 2.0
            else:
                tr["rejected"] += 1
                u *= v
                v *= 2
            tr["u"].append(u)
        RV = mat3_inv(JtJ)
    return dict(F=F, V=V, RVel=RV, JtJ=JtJ), tr


def knife(tr):
    """(ill-posed decisions: within the margin on a step that moves V, whether every decision clears the margin)"""
    ill = [d for d in tr["dec"] if d[0] < MARGIN and d[1] > H_TINY]
    return ill, all(d[0] >= MARGIN for d in tr["dec"])


def mv_vacuous(st):
    sp, tr, drv = st["sp"], st["tr"], st["drv"]
    msgs, info = [], dict(evals=len(tr["evals"]), rejected=tr["rejected"],
                          margin=min([d[0] for d in tr["dec"]], default=np.inf))
    for w in sp["want"]:
        if w == "rejected" and not tr["rejected"]:
            msgs.append("no rejected step")
        elif w == "u_inf":
            n_inf = sum(1 for u in tr["u"] if np.isinf(u))
            n_nan = sum(1 for e in tr["evals"] if not np.isfinite(e["V"]).all())
            info.update(u_inf_steps=n_inf, nan_poses=n_nan)
            if not (n_inf and n_nan):
                msgs.append("u stays finite (%d) or no NaN pose (%d)" % (n_inf, n_nan))
        elif w == "jtj_zero":
            info["K0"] = len(st["kl"])
            if np.abs(tr["evals"][0]["JtJ"]).max() != 0 or not len(st["kl"]):
                msgs.append("JtJ != 0")
        elif w == "degenerate":
            usable = int((st["kl"]["s_rho"] <= st["a"]["q"]).sum())
            info["usable"] = usable
            if usable >= 3:
                msgs.append("%d usable keylines" % usable)
        elif w == "empty" and len(st["kl"]):
            msgs.append("the old map is not empty")
    return msgs, info

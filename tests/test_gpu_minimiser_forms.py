"""Every form of Minimizer_RV against the reference: the four-cluster kernel (the default), the one-cluster kernel
(REBVO_B200_MIN_G=1), two and three clusters, the cluster kernels with a 32-keyline shared-memory slice (every other
keyline spills to global memory, REBVO_B200_MIN_KPC=32), and operands staged after the launch dependency
(REBVO_B200_MIN_EARLY=0).  Every form runs a minimisation in one launch, and shares the per-keyline body with the
stage-level TryVelRot (rb_try_vel_rot, one launch of 256-keyline blocks).

test_minimiser_form runs test_gpu_parity.py's tracker block on the EuRoC frame pair, with its bars: the stage-level
TryVelRot at three poses x three (reweight, procjf) pairs, then Minimizer_RV, m_id_f exact.

test_minimiser_state runs Minimizer_RV on seeded old maps against the reference, one case per state and form.  The new map
is frame 11 of the EuRoC-like sequence as the reference detects it; the old map is frame 10's keylines, tiled with
sub-pixel jitter up to any K0 <= KEYLINE_MAX, with the depth, gate and gradient state each case needs: CTA slices that
are empty, partial, full and one past full, the s_rho and m_num gates (m_num beyond the kernel's 8-bit flag), runs of
misses whose stale residual (DResidualNew[ikl] = fi of the last match, global_tracker.cpp:341,406) crosses every
virtual-warp, slice, cluster, column and block boundary, projections on the image border, every LM schedule, degenerate
maps, two minimisations on one new map, and schedules of more than 32 rounds.  Its last call also runs as the per-frame
pipeline runs it (rb_minimizer_rv_forward: FordwardMatch's arg-max folded into the last round, then the apply), and the new
map must be the reference's Minimizer_RV + FordwardMatch and rb_minimizer_rv + rb_forward_match bit for bit; fold_ties
puts tie groups across slices, clusters and the spilled range, and slice ends on every step shape of the fold's loop.  Every case also runs a NumPy restatement of the LM driver
(global_tracker.cpp:598-817) on the reference's own TryVelRot: it must agree with the reference, and its trace proves that
the case reached its target (a vacuous case fails) and that no LM decision sits on a knife edge.

test_try_vel_rot_stale runs the stage-level TryVelRot on the stale-residual states against the reference: its misses
inherit the fi of the last match across warp and block boundaries, and each evaluation reads the residuals of the one
before it."""
import numpy as np
import pytest

from parity_util import (DOG_THRESH, EUROC_CFG, PLANE_FIT, POS_NEG, Bench, Report, _diff, parity_frames,
                         tracker_parity)
from parity_util import _compare as _compare_kl

pytestmark = pytest.mark.gpu

FORMS = {"four_clusters": {}, "one_cluster": {"REBVO_B200_MIN_G": "1"}, "two_clusters": {"REBVO_B200_MIN_G": "2"}, "three_clusters": {"REBVO_B200_MIN_G": "3"},
         "spill_g4": {"REBVO_B200_MIN_KPC": "32"}, "spill_g1": {"REBVO_B200_MIN_G": "1", "REBVO_B200_MIN_KPC": "32"},
         "late_operands": {"REBVO_B200_MIN_EARLY": "0"}}
CLUSTERS = {"four_clusters": 4, "one_cluster": 1, "two_clusters": 2, "three_clusters": 3,
            "spill_g4": 4, "spill_g1": 1, "late_operands": 4}
ENV_KEYS = ("REBVO_B200_MIN_G", "REBVO_B200_MIN_KPC", "REBVO_B200_MIN_EARLY")


def _set_form_env(monkeypatch, form):
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in FORMS[form].items():   # read by rb_ctx_create (MIN_EARLY: by each Minimizer_RV call)
        monkeypatch.setenv(k, v)


@pytest.mark.parametrize("form", sorted(FORMS))
def test_minimiser_form(built, monkeypatch, form):
    from oracle import refapi
    from rebvo_b200 import capi
    _set_form_env(monkeypatch, form)
    cfg = EUROC_CFG
    cam = cfg["cam"]
    rep = Report("minimiser " + form)
    refs = [refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], cfg["sigma0"],
                          cfg["ksigma"]) for _ in range(2)]
    ctx = capi.Ctx(cam, cfg["sigma0"], cfg["ksigma"], kl_capacity=50000)
    assert ctx.minimizer_clusters() == CLUSTERS[form]
    gm = [ctx.new_map(), ctx.new_map()]
    # the detector state test_gpu_parity.py's tracker block starts from (its detector stages are checked there)
    det = capi.DetectParams(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["kl_ref"], cfg["gain"], cfg["tmax"],
                            cfg["tmin"])
    t_ref, l_ref = cfg["thresh"], 0
    t_gpu, l_gpu = cfg["thresh"], 0
    for r, g, fr in zip(refs, gm, parity_frames(cfg)):
        r.rgb2bw(fr)
        r.build()
        g.upload_rgb(fr)
        g.dog_build()
        _, t_ref, l_ref = r.detect(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], t_ref, l_ref, cfg["kl_ref"],
                                   cfg["gain"], cfg["tmax"], cfg["tmin"])
        _, t_gpu, l_gpu = g.detect(det, t_gpu, l_gpu)
    refs[1].detect(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], t_ref, l_ref, cfg["kl_ref"], 0.0, 1, 0)
    gm[1].detect(capi.DetectParams(PLANE_FIT, POS_NEG, DOG_THRESH, cfg["kl_max"], cfg["kl_ref"], 0.0, 1.0, 0.0),
                 t_ref, l_ref)
    _, rt = refs[1].reestimate(cfg["track_points"], 100)
    gm[1].reestimate(cfg["track_points"], 100)

    m_r = tracker_parity(rep, cfg, refs, gm, rt)
    # a minimisation is one launch in every form
    n0 = ctx.launches()
    gm[1].minimizer_rv(gm[0], m_r["V"], m_r["W"], cfg["match_thresh"], cfg["iter_max"], cfg["init_type"],
                       cfg["reweight"], 1e3, cfg["match_num_thresh"], cfg["init_iter"])
    launches = ctx.launches() - n0
    assert launches <= 2, launches
    for g in gm:
        g.close()
    ctx.close()
    fails = rep.failures()
    assert not fails, "\n".join("%s: %s" % (f["what"], f["info"]) for f in fails)


# =====================================================================================================================
# Seeded states
# =====================================================================================================================
CFG = EUROC_CFG
KEYLINE_MAX = 50000
MIN_HITS = 50            # keylines (misses, decisions ...) a case must put on its target
MARGIN = 1e-9            # least relative margin of an LM decision (gain > 0, F > Ft)
H_TINY = 1e-11           # steps at most this long decide nothing that moves the pose
MAX_R = 40.0             # build_field radius = TryVelRot's max_r
V_FAR = np.array([0.02, -0.015, 0.01])       # a prior far from the frame pair's motion
W_FAR = np.array([0.01, 0.012, -0.008])
BASE = dict(mt=CFG["match_thresh"], iter_max=5, init_type=2, init_iter=2, k_huber=2.0, mnt=0, q=1e3, prior="zero")


def _kpc(K0, G):
    k = -(-K0 // (16 * G))
    return min((k + 31) & ~31, 3584)


BLOCKS = dict(G=0)       # the geometry of rb_try_vel_rot: 256-keyline blocks


def _geometry(form, K0):
    """How the form splits K0 keylines: slice size kpc, shared-memory keylines S, clusters G, CTA threads T"""
    G = CLUSTERS[form]
    spill = "REBVO_B200_MIN_KPC" in FORMS[form]
    S = 32 if spill else {1: 1280, 2: 640, 3: 448, 4: 320}[G]
    kpc = _kpc(K0, G)
    return dict(G=G, kpc=kpc, S=S, T=512 if G == 1 else 256, J=-(-kpc // (512 if G == 1 else 256)))


def _crossing(geo, j, i):
    """Boundary class between the last match j and the miss i that inherits its fi."""
    out = np.full(len(i), "none", object)
    out[j < 0] = "start"
    ok = j >= 0
    jj, ii = j[ok], i[ok]
    if geo["G"] == 0:
        c = np.where(jj // 256 != ii // 256, "block", np.where(jj // 32 != ii // 32, "warp", "none"))
    else:
        kpc, G = geo["kpc"], geo["G"]
        sj, si = jj // kpc, ii // kpc
        lj, li = jj - sj * kpc, ii - si * kpc
        c = np.where(sj // G != si // G, "column", np.where(sj != si, "cluster",
                     np.where((lj < geo["S"]) != (li < geo["S"]), "spill",
                              np.where(lj // 32 != li // 32, "vwarp", "none"))))
    out[ok] = c
    return out


def _classes(geo, K0):
    """The boundary classes the geometry has at K0 keylines."""
    if geo["G"] == 0:
        return ["warp"] + (["block"] if K0 > 256 else [])
    c = ["vwarp", "column"]
    if geo["G"] > 1 and K0 > geo["kpc"]:
        c.append("cluster")
    if geo["kpc"] > geo["S"]:
        c.append("spill")
    return c


# ---- the old map ------------------------------------------------------------------------------------------------------
def _tile(kl10, K0, rng):
    """frame 10's keylines tiled up to K0, every copy after the first moved by a sub-pixel offset (never to x.5)"""
    n = len(kl10)
    idx = np.arange(K0) % n
    kl = kl10[idx].copy()
    cp = np.arange(K0) // n
    jit = rng.uniform(0.1, 0.4, (K0, 2)) * rng.choice([-1, 1], (K0, 2))
    kl["p_m"] = (kl["p_m"].astype(np.float64) + jit * (cp > 0)[:, None]).astype(np.float32)
    kl["rho"] = np.exp(rng.uniform(np.log(0.5), np.log(2.0), K0))
    kl["s_rho"] = np.exp(rng.uniform(np.log(0.05), np.log(0.5), K0))
    kl["m_num"] = rng.integers(3, 11, K0)
    kl["m_id_f"] = -1
    return kl


def _turn(kl, sel):
    """gradients turned by 90 degrees: Test_f_k fails against any field keyline of the same edge (a miss)"""
    mx, my = kl["m_m"][sel, 0].copy(), kl["m_m"][sel, 1].copy()
    kl["m_m"][sel, 0] = -my
    kl["m_m"][sel, 1] = mx


def _runs(kl, rng, starts, lengths, skipped=False):
    """runs of misses (or skipped keylines) [s, s + L); the keyline before each run is moved 3 px along its gradient, so
    that the fi it leaves behind is larger than k_huber"""
    K0 = len(kl)
    sel = np.zeros(K0, bool)
    for s, L in zip(starts, lengths):
        sel[max(s, 0):min(s + L, K0)] = True
    # the keyline before a run keeps its gradient and is moved
    lead = np.array([s - 1 for s in starts if 0 < s <= K0 and not sel[s - 1]], np.int64)
    if len(lead):
        u = kl["m_m"][lead].astype(np.float64) / np.maximum(kl["n_m"][lead].astype(np.float64), 1e-6)[:, None]
        sgn = rng.choice([-1.0, 1.0], len(lead))[:, None]
        kl["p_m"][lead] = (kl["p_m"][lead].astype(np.float64) + 3.2 * sgn * u).astype(np.float32)
    if skipped:
        kl["s_rho"][sel] = 1e6
    else:
        _turn(kl, sel)
    return sel


def _boundary_runs(K0, rng):
    """run starts on the boundaries of every form at K0: virtual warps, every form's slices (kpc at G = 1..4), spill
    edges (32 and S into a slice), 256-keyline blocks, the first and the last keylines"""
    st = {0, max(K0 - 300, 0)}
    for G in (1, 2, 3, 4):
        kpc = _kpc(K0, G)
        for s in range(kpc, K0, kpc):
            st.add(s - int(rng.integers(1, 40)))
        for s in range(0, K0, kpc):
            for S in (32, {1: 1280, 2: 640, 3: 448, 4: 320}[G]):
                if S < kpc:
                    st.add(s + S - int(rng.integers(1, 8)))
    for s in rng.choice(np.arange(256, K0, 256), min(12, K0 // 256), replace=False):
        st.add(int(s) - int(rng.integers(1, 20)))
    for s in rng.choice(np.arange(32, K0, 32), min(40, K0 // 32), replace=False):
        st.add(int(s) - int(rng.integers(1, 12)))
    st = sorted(s for s in st if 0 <= s < K0)
    # runs long enough to reach past the boundary, not so long that they cover most of the map
    return st, [int(rng.integers(60, 140)) for _ in st]


def _state_old(name, sp, kl10, ppxy, wh):
    rng = np.random.default_rng(sum(map(ord, name)))
    K0 = sp["K0"]
    kl = _tile(kl10, K0, rng)
    ev = {}
    kind = sp.get("kind")
    if kind == "gates":   # s_rho log-spread, exactly max_s_rho and one ulp above; m_num 0..300
        q = sp["q"]
        kl["s_rho"] = np.exp(rng.uniform(np.log(1e-3), np.log(3.0 * q), K0))
        eq = rng.random(K0) < 0.05
        up = ~eq & (rng.random(K0) < 0.05)
        kl["s_rho"][eq] = q
        kl["s_rho"][up] = np.nextafter(q, np.inf)
        kl["m_num"] = rng.integers(0, 301, K0)
        ev.update(s_rho_eq=int(eq.sum()), s_rho_ulp=int(up.sum()))
    elif kind == "stale":
        st, ln = _boundary_runs(K0, rng)
        ev["runs"] = len(st)
        _runs(kl, rng, st, ln)
        if sp.get("skipped_runs"):   # skipped keylines between a match and later misses: the carry passes over them
            sk, skl = _boundary_runs(K0, np.random.default_rng(rng.integers(1 << 30)))
            sk = [s + 2 for s in sk[1::3]]
            _runs(kl, rng, sk, [min(l, 40) for l in skl[1::3]], skipped=True)
    elif kind == "outside":   # at X = 0 on x in {0, 1, w-2, w-1} (and the same for y); 0.2 px off the integer
        w, h = wh
        n = K0 // 8
        tgt = np.array([0, 1, w - 2, w - 1])
        sel = rng.permutation(K0)[:8 * n].reshape(8, n)
        for a in range(4):
            kl["p_m"][sel[a], 0] = np.float32(tgt[a] + 0.2 * rng.choice([-1, 1], n) - ppxy[0])
            kl["rho"][sel[a]] = 1.0
        tgt = np.array([0, 1, h - 2, h - 1])
        for a in range(4):
            kl["p_m"][sel[4 + a], 1] = np.float32(tgt[a] + 0.2 * rng.choice([-1, 1], n) - ppxy[1])
            kl["rho"][sel[4 + a]] = 1.0
        ev["border"] = n
    elif kind == "ties":
        kl["rho"] = kl["rho"][np.arange(K0) % len(kl10)]
    elif kind == "all_skipped":
        kl["s_rho"] = 10.0 * sp["q"]
    elif kind == "five":
        kl["s_rho"][5:] = 10.0 * sp["q"]
    if "m_num" in sp:
        kl["m_num"] = sp["m_num"](rng, K0)
    return kl, ev


# ---- the states: name -> spec ---------------------------------------------------------------------------------------
def _mn2(rng, K0):
    m = rng.integers(0, 11, K0)
    m[rng.random(K0) < 0.2] = 2
    return m


STATES = {}
for _k in (1, 31, 33, 500, 2048, 2049, 15000, 20480, 20481, 50000):
    STATES["K%d" % _k] = dict(K0=_k, fc=0, want=["evals"])
STATES["K1"].update(init_iter=0, iter_max=1)   # (further steps fit the one keyline exactly: F would be rounding noise)
for _mnt in (0, 3, 255, 256):
    for _fc in (0, 2, 1000):
        STATES["gates_mnt%d_fc%d" % (_mnt, _fc)] = dict(K0=15000, kind="gates", q=0.3, mnt=_mnt, fc=_fc,
                                                       want=["gates"])
STATES["stale_k2"] = dict(K0=15000, kind="stale", k_huber=2.0, fc=0, want=["stale"])
STATES["stale_k0.5_skipped"] = dict(K0=20481, kind="stale", skipped_runs=True, k_huber=0.5, fc=0, want=["stale"])
STATES["stale_k2_50000"] = dict(K0=50000, kind="stale", k_huber=2.0, fc=0, init_iter=1, iter_max=3, want=["stale"])
STATES["outside"] = dict(K0=15000, kind="outside", fc=0, want=["outside"])
for _t in (0, 1):
    for _m in (0, 1, 5, 10):
        STATES["init%d_iter%d" % (_t, _m)] = dict(K0=8000, init_type=_t, iter_max=_m, prior="near", fc=0,
                                                   want=["evals"] + (["rejected"] if _m == 10 else []))
for _n in (0, 1, 3):
    for _m in (0, 5):
        STATES["init2_n%d_iter%d_far" % (_n, _m)] = dict(K0=8000, init_iter=_n, iter_max=_m, prior="far", fc=0,
                                                          want=["zero_wins"])
    STATES["init2_n%d_near" % _n] = dict(K0=8000, init_iter=_n, iter_max=1, prior="near", fc=0, want=["prior_wins"])
STATES["init2_n0_iter0_zero"] = dict(K0=8000, init_iter=0, iter_max=0, prior="far", fc=0, want=["eff0"])
STATES["ns32"] = dict(K0=8000, init_iter=2, iter_max=25, prior="near", fc=0, want=["ns32"])
STATES["ns33"] = dict(K0=8000, init_iter=2, iter_max=26, prior="near", fc=0, want=["ns33"])
# the longest well-posed schedule near the API's limit (64 evaluations, 63 rounds at init_iter 0, iter_max 61), twice on
# one map, so that the second minimisation's sequence numbers of the multi-cluster exchange follow those of a 48-round
# one.  This map converges after one step and every later step is rejected: the 45th rejection in a row overflows u *= v
# to inf, and every evaluation after it runs at a NaN pose.  So 46 iterations, the last of them that rejection: 49
# evaluations in 48 rounds.
STATES["ns49"] = dict(K0=8000, init_iter=0, iter_max=46, prior="near", fc=0, calls=["main", "main"], want=["ns49"])
STATES["K0_then_gate"] = dict(K0=8000, fc=2, mnt=3, m_num=_mn2, calls=["empty", "main"], want=["empty"])
STATES["back_to_back"] = dict(K0=8000, fc=2, mnt=3, m_num=_mn2, calls=["main", "main"], want=["gate_change"])
# FordwardMatch's arg-max folded into the last round: every tile copy of a keyline has its rho, so that copies that land on
# one new keyline tie, with their offers in different slices, clusters and spilled ranges
STATES["fold_ties"] = dict(K0=50000, kind="ties", fc=0, init_iter=1, iter_max=3, want=["ties"])
STATES["all_skipped"] = dict(K0=3000, kind="all_skipped", fc=0, want=["degenerate"])
STATES["five_usable"] = dict(K0=3000, kind="five", fc=0, want=["degenerate"])


# ---- NumPy restatement of the LM driver -------------------------------------------------------------------------------
def _svd_backsub(A, b):
    """TooN SVD<>::backsub: singular values below max / 1e9 are dropped"""
    U, s, Vt = np.linalg.svd(A)
    inv = np.where(s * 1e9 > s[0], 1.0 / np.where(s > 0, s, 1.0), 0.0) if s[0] > 0 else np.zeros_like(s)
    return Vt.T @ (inv * (U.T @ b))


def _gain(num, den):
    with np.errstate(divide="ignore", invalid="ignore"):   # (0 / 0 = NaN on an all-skipped map: the step is rejected)
        return num / den


def _chol_solve(A, b):
    try:
        np.linalg.cholesky(A)
        return np.linalg.solve(A, b)
    except np.linalg.LinAlgError:
        return np.full(len(b), np.nan)


def _lm_driver(new_r, old_r, a, V, W):
    """Minimizer_RV (global_tracker.cpp:598-817) with every evaluation done by the reference's TryVelRot; returns the
    outputs and a trace: evaluations (pose, residual buffers, matches) and LM decisions (kind, relative margin, |h|)."""
    K0 = old_r.knum()
    tr = dict(evals=[], dec=[], merge=None)
    if K0 <= 0:
        return None, tr
    pnum = (K0 + 3) & ~3
    buf = {"Res0": np.zeros(pnum), "Res1": np.zeros(pnum), "Rest": np.zeros(pnum)}

    def tvr(X, rw, pj, rin, rout):
        s, J, Fv, out = new_r.try_vel_rot(old_r, X, rw, pj, a["mt"], a["q"], a["mnt"], a["k_huber"], buf[rin])
        wrote = ~np.isnan(out)
        buf[rout] = np.where(wrote, out, buf[rout])
        tr["evals"].append(dict(X=np.array(X, np.float64), rw=rw, res=out[:K0].copy(), matched=old_r.keylines()["m_id_f"] >= 0,
                                wrote=wrote[:K0]))
        return s, J, Fv

    def decide(kind, f, fn, h):
        m = abs(f - fn) / max(abs(f), abs(fn), 1e-300)
        tr["dec"].append((kind, m, float(np.linalg.norm(h)) if h is not None else np.inf))

    VW = np.concatenate([V, W])
    tau, v, eff = 1e-3, 2.0, 0
    h = np.zeros(6)
    Residual, ResidualNew = "Res0", "Res1"
    if a["init_type"] in (0, 1):
        X = np.zeros(6) if a["init_type"] == 0 else VW.copy()
    else:
        tries = []
        for t, (X0, rout) in enumerate(((np.zeros(6), "Rest"), (VW.copy(), None))):
            rout = rout or ResidualNew
            X = X0
            F, JtJ, JtF = tvr(X, False, True, Residual, rout)
            F0 = F
            u = tau * JtJ.max()
            v, eff = 2.0, 0
            for i in range(a["init_iter"]):
                h = _svd_backsub(JtJ + np.eye(6) * u, -JtF)
                Xn = X + h
                if i == a["init_iter"] - 1:
                    Fn, _, _ = tvr(Xn, False, False, Residual, rout)
                    gain = F - Fn
                    Jn = Fnv = None
                else:
                    Fn, Jn, Fnv = tvr(Xn, False, True, Residual, rout)
                    gain = _gain(F - Fn, 0.5 * h @ (u * h - JtF))
                decide("init%d" % t, F, Fn, h)
                if gain > 0:
                    F, X = Fn, Xn
                    if Jn is not None:
                        JtJ, JtF = Jn, Fnv
                    u *= max(0.33, 1 - (2 * gain - 1) ** 3)
                    v = 2.0
                    eff += 1
                else:
                    tr["rejected"] = tr.get("rejected", 0) + 1
                    u *= v
                    v *= 2
            tries.append(dict(X=X, F=F, F0=F0, eff=eff))
        z, p = tries
        tr["merge"] = "zero" if p["F"] > z["F"] else "prior"
        if not np.array_equal(z["X"], p["X"]):
            decide("merge", p["F"], z["F"], None)
        X, eff = (z["X"], z["eff"]) if p["F"] > z["F"] else (p["X"], p["eff"])
        if p["F"] > z["F"]:
            ResidualNew = "Rest"
        Residual, ResidualNew = ResidualNew, Residual
    F, JtJ, JtF = tvr(X, True, True, Residual, ResidualNew)
    F0 = F
    u = tau * JtJ.max()
    v = 2.0
    for _ in range(a["iter_max"]):
        h = _chol_solve(JtJ + np.eye(6) * u, -JtF)
        Xn = X + h
        Fn, Jn, Fnv = tvr(Xn, True, True, Residual, ResidualNew)
        gain = _gain(F - Fn, 0.5 * h @ (u * h - JtF))
        decide("main", F, Fn, h)
        if gain > 0:
            F, X, JtJ, JtF = Fn, Xn, Jn, Fnv
            u *= max(0.33, 1 - (2 * gain - 1) ** 3)
            v = 2.0
            eff += 1
            Residual, ResidualNew = ResidualNew, Residual
        else:
            tr["rejected"] = tr.get("rejected", 0) + 1
            u *= v
            v *= 2
    tr["eff"] = eff
    rel_err = np.linalg.norm(h) / (np.linalg.norm(X) + 1e-30) if eff > 0 else 1e20
    return dict(V=X[:3], W=X[3:], F=F, rel_err=rel_err, rel_err_score=F / F0 if eff > 0 else 1e20), tr


# ---- the reference side, once per state ---------------------------------------------------------------------------------
class Base:
    def __init__(self):
        from oracle import refapi
        self.refapi = refapi
        self.b = Bench(CFG["cam"], parity_frames(CFG))
        self.cam = CFG["cam"]
        _, self.rt = self.b.ref[1].reestimate(CFG["track_points"], 100)
        self.kl10, self.kl11, self.mask11 = self.b.kl[0], self.b.kl[1], self.b.mask[1]
        self.empty = np.full((self.cam["h"], self.cam["w"]), -1, np.int32)
        self.cache = {}
        self.ctx = {}
        # the frame pair's motion (prior "near"): the reference's minimisation on the plain tiled map
        r_new, r_old = self.ref_maps(_tile(self.kl10, 8000, np.random.default_rng(1)), 0)
        m = r_new.minimizer_rv(r_old, np.zeros(3), np.zeros(3), CFG["match_thresh"], 5, 2, 2.0, 1e3, 0, 2)
        self.near = (m["V"].copy(), m["W"].copy())

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

    def state(self, name):
        if name in self.cache:
            return self.cache[name]
        sp = dict(BASE)
        sp.update(STATES[name])
        kl, ev = _state_old(name, sp, self.kl10, (np.float32(self.cam["ppx"]), np.float32(self.cam["ppy"])),
                            (self.cam["w"], self.cam["h"]))
        V, W = {"zero": (np.zeros(3), np.zeros(3)), "near": self.near, "far": (V_FAR, W_FAR)}[sp["prior"]]
        new, old = self.ref_maps(kl, sp["fc"])
        empty_old = self.refmap()
        empty_old.set_mask(self.empty, 0)
        runs = []
        for c in sp.get("calls", ["main"]):
            o = empty_old if c == "empty" else old
            drv, tr = _lm_driver(new, o, sp, V, W)
            m = new.minimizer_rv(o, V, W, sp["mt"], sp["iter_max"], sp["init_type"], sp["k_huber"], sp["q"], sp["mnt"],
                                 sp["init_iter"])
            runs.append(dict(old=c, ref=m, drv=drv, tr=tr, m_id_f=o.keylines()["m_id_f"].copy() if c != "empty" else None))
        # the last call followed by FordwardMatch, into a map of frame 11's keylines as detected
        fwd = self.refmap()
        fwd.set_keylines(self.kl11)
        fwd.set_mask(self.mask11, len(self.kl11))
        (empty_old if runs[-1]["old"] == "empty" else old).forward_match(fwd)
        runs[-1]["fwd"] = fwd.keylines()
        st = dict(sp=sp, kl=kl, ev=ev, V=V, W=W, runs=runs)
        self.cache[name] = st
        return st


@pytest.fixture(scope="module")
def base(built):
    b = Base()
    yield b
    for c in b.ctx.values():
        c.close()
    b.b.close()


BARS = (("V", 0.0, 1e-9, False), ("W", 0.0, 1e-9, False), ("F", 1e-8, 0.0, False), ("rel_err_score", 1e-8, 0.0, False),
        ("RVel", 1e-8, 1e-9, True), ("RW0", 1e-8, 1e-9, True), ("W_X", 1e-8, 1e-9, True))


def _close(tag, ref, got, rtol, atol):
    ref, got = np.asarray(ref, np.float64), np.asarray(got, np.float64)
    fin = np.isfinite(ref)
    errs = []
    if not np.array_equal(np.isnan(ref), np.isnan(got)) or not np.array_equal(np.isposinf(ref), np.isposinf(got)) \
            or not np.array_equal(np.isneginf(ref), np.isneginf(got)):
        errs.append("%s: NaN/inf positions differ: ref %s gpu %s" % (tag, ref.ravel()[:6], got.ravel()[:6]))
    bad = fin & ~(np.abs(ref - got) <= atol + rtol * np.abs(ref))
    if bad.any():
        errs.append("%s: ref %s gpu %s" % (tag, ref[bad][:3], got[bad][:3]))
    return errs


def _singular(JtJ):
    """JtJ numerically singular (fewer than six usable keylines): the covariance, Cholesky<6>(JtJ).get_inverse(), is then
    rounding noise amplified by 1 / eps, or NaN from 0 / 0, and depends on the order of the sums"""
    J = np.asarray(JtJ, np.float64)
    if not np.isfinite(J).all() or not np.abs(J).max() > 0:
        return True
    ev = np.linalg.eigvalsh((J + J.T) / 2)
    return ev[0] <= 1e-12 * ev[-1]


def _compare(m_r, m_g, with_rel_err):
    errs = []
    cov = not _singular(m_r["W_X"])
    for k, rtol, atol, scaled in BARS:
        if k in ("RVel", "RW0") and not cov:
            continue
        fin = np.asarray(m_r[k], np.float64)
        amax = np.abs(fin[np.isfinite(fin)]).max() if np.isfinite(fin).any() else 0.0
        errs += _close(k, m_r[k], m_g[k], rtol, atol * amax if scaled else atol)
    if with_rel_err:
        errs += _close("rel_err", m_r["rel_err"], m_g["rel_err"], 1e-8, 0.0)
    return errs


def _evidence(st, form):
    """what the case must show it reached; returns (failures, summary)"""
    sp, runs = st["sp"], st["runs"]
    K0 = sp["K0"]
    geo = _geometry(form, K0)
    msgs, info = [], {}
    tr = runs[-1]["tr"]
    for w in sp["want"]:
        if w == "evals":
            info["evals"] = len(tr["evals"])
        elif w == "gates":
            kl = st["kl"]
            fc = sp["fc"]
            gate = min(sp["mnt"], fc)
            n_s = int((kl["s_rho"] > sp["q"]).sum())
            n_m = int(((kl["m_num"] < gate) & (kl["s_rho"] <= sp["q"])).sum())
            info.update(st["ev"], s_rho_gate=n_s, m_num_gate=n_m, big_m_num_used=int((kl["m_num"] >= 255).sum()))
            if min(st["ev"]["s_rho_eq"], st["ev"]["s_rho_ulp"], n_s) < MIN_HITS:
                msgs.append("s_rho gate %s" % info)
            if gate > 0 and n_m < MIN_HITS:
                msgs.append("m_num gate closes for %d keylines" % n_m)
        elif w == "stale":
            cnt = _carried(geo, tr["evals"], K0, sp["k_huber"])
            info["carried misses"] = cnt
            msgs += _too_few_carried(geo, K0, cnt)
        elif w == "outside":
            e0 = tr["evals"][0]   # the zero-initialised try's first pose: X = 0
            n_out = int((e0["wrote"] & (e0["res"] == MAX_R) & ~e0["matched"]).sum())
            info["outside at X=0"] = n_out
            if n_out < 2 * MIN_HITS:
                msgs.append("only %d projections outside" % n_out)
        elif w == "rejected":
            info["rejected"] = tr.get("rejected", 0)
            if not tr.get("rejected"):
                msgs.append("no rejected step")
        elif w in ("zero_wins", "prior_wins"):
            info["merge"] = tr["merge"]
            if tr["merge"] != w.split("_")[0]:
                msgs.append("the %s try won" % tr["merge"])
        elif w == "eff0":
            info["eff_steps"] = tr.get("eff")
            if tr.get("eff") != 0:
                msgs.append("eff_steps %s" % tr.get("eff"))
        elif w in ("ns32", "ns33", "ns49"):
            info["evals"] = len(tr["evals"])
            if len(tr["evals"]) != int(w[2:]):
                msgs.append("%d evaluations" % len(tr["evals"]))
        elif w in ("empty", "gate_change"):
            kl = st["kl"]
            n2 = int((kl["m_num"] == 2).sum())
            info["m_num==2"] = n2
            if n2 < MIN_HITS:
                msgs.append("gate change touches %d keylines" % n2)
            if w == "empty" and runs[0]["tr"]["evals"]:
                msgs.append("the empty map was evaluated")
        elif w == "ties":
            msgs += _fold_reach(st, form, info)
        elif w == "degenerate":
            usable = int((st["kl"]["s_rho"] <= sp["q"]).sum())
            info["usable"] = usable
            if usable >= 6:
                msgs.append("%d usable keylines" % usable)
    return msgs, info


def _fold_reach(st, form, info):
    """FordwardMatch's arg-max in the last round: each thread offers the keylines li and li + T - 96 of its slice per step
    (li = tid - 96, tid - 96 + 2 (T - 96), ...).  The slices of the forms together must be empty, end in a step without a
    second keyline and in one with it, and hold a full step; every form must have MIN_HITS tie groups (equal largest rho
    on one new keyline) with offers in different slices, and in different clusters and in the spilled range where it has
    them."""
    K0 = st["sp"]["K0"]
    ends = set()
    for f in FORMS:
        g = _geometry(f, K0)
        stp = g["T"] - 96
        for s in range(16 * g["G"]):
            cnt = min(max(K0 - s * g["kpc"], 0), g["kpc"])
            r = cnt % (2 * stp)
            ends |= {"empty"} if cnt == 0 else set()
            ends |= {"second -1" if 0 < r <= stp else "second" if r else "whole"}
            ends |= {"full step"} if cnt >= 2 * stp else set()
    msgs = [] if {"empty", "second -1", "second", "full step"} <= ends else ["slice ends %s" % sorted(ends)]
    geo = _geometry(form, K0)
    kl, f = st["kl"], st["runs"][-1]["m_id_f"]
    idx = np.nonzero(f >= 0)[0]
    key = np.lexsort((-kl["rho"][idx], f[idx]))   # by target, the largest rho first
    idx = idx[key]
    tgt, rho = f[idx], kl["rho"][idx]
    first = np.r_[True, tgt[1:] != tgt[:-1]]
    top = rho == np.maximum.reduceat(rho, np.nonzero(first)[0])[np.cumsum(first) - 1]
    cnt = dict(slices=0, clusters=0, spill=0)
    for t in np.unique(tgt[top]):
        o = idx[top & (tgt == t)]
        if len(o) < 2:
            continue
        sl = o // geo["kpc"]
        cnt["slices"] += len(set(sl)) > 1
        cnt["clusters"] += len(set(sl % geo["G"])) > 1
        cnt["spill"] += bool(((o - sl * geo["kpc"]) >= geo["S"]).any())
    need = ["slices"] + (["clusters"] if geo["G"] > 1 else []) + (["spill"] if geo["kpc"] > geo["S"] else [])
    info.update(tie_groups=cnt, slice_ends=sorted(ends))
    return msgs + ["%d tie groups across %s" % (cnt[k], k) for k in need if cnt[k] < MIN_HITS]


def _carried(geo, evals, K0, k_huber):
    """misses per boundary class between the miss and the last match before it whose inherited fi the evaluations wrote
    (a miss at the start inherits 0; elsewhere only an fi beyond k_huber counts, one that changes a re-weighting)"""
    cnt = {}
    idx = np.arange(K0)
    for e in evals:
        res, mt, wr = e["res"], e["matched"], e["wrote"]
        lastm = np.maximum.accumulate(np.where(mt, idx, -1))
        prev = np.concatenate([[-1], lastm[:-1]])
        miss = wr & ~mt & (res != MAX_R)
        cls = _crossing(geo, prev[miss], idx[miss])
        big = np.abs(res[miss]) > k_huber
        for c in set(cls):
            sel = cls == c
            cnt[c] = cnt.get(c, 0) + int((sel & (big | (c == "start"))).sum())
    return cnt


def _too_few_carried(geo, K0, cnt):
    return ["only %d carried misses across %s" % (cnt.get(c, 0), c) for c in _classes(geo, K0) + ["start"]
            if cnt.get(c, 0) < MIN_HITS]


def _knife(tr):
    """(ill-posed decisions, whether every decision clears the margin)"""
    ill = [d for d in tr["dec"] if d[1] < MARGIN and d[2] > H_TINY]
    clear = all(d[1] >= MARGIN for d in tr["dec"])
    return ill, clear


def _ctx(base, form):
    from rebvo_b200 import capi
    if form not in base.ctx:
        base.ctx[form] = capi.Ctx(CFG["cam"], CFG["sigma0"], CFG["ksigma"], kl_capacity=KEYLINE_MAX)
    return base.ctx[form]


@pytest.mark.parametrize("form", sorted(FORMS))
@pytest.mark.parametrize("state", list(STATES))
def test_minimiser_state(base, monkeypatch, state, form):
    _set_form_env(monkeypatch, form)
    st = base.state(state)
    sp = st["sp"]
    msgs = []
    # the restatement agrees with the reference, and the case is well posed and reaches its target
    rel_ok = True
    for k, run in enumerate(st["runs"]):
        if run["drv"] is None:
            continue
        ill, clear = _knife(run["tr"])
        assert not ill, "ill-posed case: LM decisions on a knife edge %s" % ill
        rel_ok &= clear
        m_r, d = run["ref"], run["drv"]
        if np.isfinite(m_r["F"]) and np.isfinite(m_r["V"]).all():
            de = _close("driver V", m_r["V"], d["V"], 0, 1e-9) + _close("driver W", m_r["W"], d["W"], 0, 1e-9) + \
                _close("driver F", m_r["F"], d["F"], 1e-8, 0)
            if clear:
                de += _close("driver rel_err", m_r["rel_err"], d["rel_err"], 1e-8, 0)
            assert not de, "the LM restatement disagrees with the reference (call %d): %s" % (k, de)
    vac, info = _evidence(st, form)
    print("%s / %s: %s%s" % (state, form, info, "" if rel_ok else "  [rel_err exempt: a decision within the margin]"))
    assert not vac, "vacuous case: %s" % vac

    ctx = _ctx(base, form)
    assert ctx.minimizer_clusters() == CLUSTERS[form]
    # newf repeats the calls on new, the last one as the per-frame pipeline runs it: FordwardMatch's arg-max folded into
    # its last round, then the apply (rb_minimizer_rv_forward); fwd gets rb_forward_match after the last call on new
    new, old, empty, newf, fwd = [ctx.new_map() for _ in range(5)]
    try:
        for m in (new, newf, fwd):
            m.load_keylines(base.kl11, base.mask11)
        for m in (new, newf):
            m.build_field(CFG["radius"], base.rt)
            m.set_frame_count(sp["fc"])
        old.load_keylines(st["kl"], base.empty)
        empty.load_keylines(st["kl"][:0], base.empty)
        for k, run in enumerate(st["runs"]):
            o = empty if run["old"] == "empty" else old
            n0 = ctx.launches()
            m_g = new.minimizer_rv(o, st["V"], st["W"], sp["mt"], sp["iter_max"], sp["init_type"], sp["k_huber"], sp["q"],
                                   sp["mnt"], sp["init_iter"])
            launches = ctx.launches() - n0
            m_r = run["ref"]
            if run["old"] == "empty":   # "if(klist.KNum()<=0) return 0;": the caller's values stay, no FrameCount++
                if not (m_g["F"] == m_r["F"] == 0 and np.array_equal(m_g["V"], st["V"])
                        and np.array_equal(m_g["W"], st["W"]) and np.array_equal(m_r["V"], st["V"])):
                    msgs.append("call %d (K0 = 0): ref %s gpu %s" % (k, m_r, m_g))
                continue
            msgs += ["call %d: %s" % (k, e) for e in _compare(m_r, m_g, rel_ok)]
            if _singular(m_r["W_X"]):
                print("%s / %s call %d: JtJ singular, RVel / RW0 not compared" % (state, form, k))
            mf = o.keylines()["m_id_f"]
            if not np.array_equal(run["m_id_f"], mf):
                msgs.append("call %d: m_id_f differs at %d keylines" % (k, int((run["m_id_f"] != mf).sum())))
            if launches > 2:
                msgs.append("%d launches for %d evaluations" % (launches, len(run["tr"]["evals"])))
        o = empty if st["runs"][-1]["old"] == "empty" else old
        args = (st["V"], st["W"], sp["mt"], sp["iter_max"], sp["init_type"], sp["k_huber"], sp["q"], sp["mnt"], sp["init_iter"])
        for run in st["runs"][:-1]:
            newf.minimizer_rv(empty if run["old"] == "empty" else old, *args)
        m_f = newf.minimizer_rv_forward(o, *args)
        n_s = o.forward_match(fwd)
        for f in ("V", "W", "F", "RVel", "RW0", "W_X"):
            if _diff(f, m_g[f], m_f[f]):
                msgs.append("with the fold: " + _diff(f, m_g[f], m_f[f]))
        r, g, s_ = st["runs"][-1]["fwd"], newf.keylines(), fwd.keylines()
        fields, matched = ["rho", "s_rho", "m_id", "m_num", "p_m_0"], ["m_m0", "n_m0"]
        msgs += ["FordwardMatch vs the reference: " + e for e in _compare_kl(r, g, fields, matched)]
        msgs += ["fold vs rb_forward_match: " + e for e in _compare_kl(s_, g, fields, matched)]
        n_r = int((r["m_id"] >= 0).sum())
        if not m_f["fwd_match"] == n_s == n_r:
            msgs.append("FordwardMatch count: fold %d, stage %d, reference keylines %d" % (m_f["fwd_match"], n_s, n_r))
        print("%s / %s: FordwardMatch matched %d new keylines" % (state, form, n_r))
    finally:
        for m in (new, old, empty, newf, fwd):
            m.close()
    assert not msgs, "\n".join(msgs)


# =====================================================================================================================
# The stage-level TryVelRot on the stale-residual states
# =====================================================================================================================
@pytest.mark.parametrize("state", [k for k in STATES if STATES[k].get("kind") == "stale"])
def test_try_vel_rot_stale(base, state):
    """rb_try_vel_rot against the reference's TryVelRot at every pose of the state's minimisation, with (reweight,
    procjf) in (0, 1), (1, 1), (0, 0), each evaluation reading the residuals of the one before it; tracker_parity's bars.
    Its 256-keyline blocks hand the stale fi of a miss's last match across warps and blocks: MIN_HITS carried misses per
    crossing class."""
    st = base.state(state)
    sp, kl = st["sp"], st["kl"]
    K0 = sp["K0"]
    r_new, r_old = base.ref_maps(kl, sp["fc"])
    ctx = _ctx(base, "try_vel_rot")
    new, old = ctx.new_map(), ctx.new_map()
    msgs, evals = [], []
    try:
        new.load_keylines(base.kl11, base.mask11)
        new.build_field(CFG["radius"], base.rt)
        old.load_keylines(kl, base.empty)
        new.set_frame_count(sp["fc"])
        used = kl["s_rho"] <= sp["q"]
        res_in = np.zeros((K0 + 3) & ~3)
        for xi, e in enumerate(st["runs"][-1]["tr"]["evals"]):
            for rw, pj in ((False, True), (True, True), (False, False)):
                args = (e["X"], rw, pj, sp["mt"], sp["q"], sp["mnt"], sp["k_huber"], res_in)
                s_r, J_r, F_r, res_r = r_new.try_vel_rot(r_old, *args)
                mf_r = r_old.keylines()["m_id_f"].copy()
                s_g, J_g, F_g, res_g = new.try_vel_rot(old, *args)
                tag = "X%d rw=%d pj=%d " % (xi, rw, pj)
                errs = _close("score", s_r, s_g, 1e-10, 0.0)
                if pj:
                    errs += _close("JtJ", J_r, J_g, 1e-9, 1e-9 * np.abs(J_r).max())
                    errs += _close("JtF", F_r, F_g, 1e-9, 1e-9 * np.abs(F_r).max())
                if not np.array_equal(mf_r, old.keylines()["m_id_f"]):
                    errs.append("m_id_f differs")
                errs += _close("DResidualNew", res_r[:K0][used], res_g[used], 1e-12, 1e-12)
                msgs += [tag + m for m in errs]
                wrote = ~np.isnan(res_r)
                evals.append(dict(res=res_r[:K0], matched=mf_r >= 0, wrote=wrote[:K0]))
                res_in = np.where(wrote, res_r, res_in)
    finally:
        new.close()
        old.close()
    cnt = _carried(BLOCKS, evals, K0, sp["k_huber"])
    print("%s: %d evaluations, carried misses %s" % (state, len(evals), cnt))
    assert not _too_few_carried(BLOCKS, K0, cnt), "vacuous case: %s" % _too_few_carried(BLOCKS, K0, cnt)
    assert not msgs, "\n".join(msgs[:20])


def test_kl_capacity_bound(built):
    """a context holds up to the reference's KEYLINE_MAX keylines; rb_ctx_create refuses more with RB_ERR_ARG (-2)"""
    from rebvo_b200 import capi
    ctx = capi.Ctx(CFG["cam"], CFG["sigma0"], CFG["ksigma"], kl_capacity=KEYLINE_MAX)
    assert ctx.minimizer_clusters() >= 1
    ctx.close()
    with pytest.raises(capi.RbError, match=r"rb_ctx_create failed \(-2\)"):
        capi.Ctx(CFG["cam"], CFG["sigma0"], CFG["ksigma"], kl_capacity=KEYLINE_MAX + 1)

"""The pipeline's per-frame map chain on seeded edge-map states, against the reference compiled into oracle/_ref.

A normal frame runs none of the stage kernels that test_gpu_mapper_states.py pins: after the minimiser, k_match applies
the FordwardMatch winner and runs directed_matching against the UNROTATED old map, rotating each probed keyline by R0 on
the fly, and k_reg_ekf evaluates the match-count gate in every thread, regularises from k_match's scratch pair, runs the
EKF, rotates the old map in place and integrates the frame's pose in a spare thread.  rb_map_match_update runs those two
kernels on loaded maps (FordwardMatch's arg-max from the old map's m_id_f), and each case compares the result bit for bit
with the reference's sequence, RefMap.forward_match -> rotate(R0) -> directed_matching(V, P_V, BackRot) -> the gate
(do_match && nmatch >= MatchThreshold, rebvo_second_t.cpp:410-423) -> regularize -> ekf, and with the stage kernels in
that order: the new map, the rotated old map, the counts and the gate's outputs.

Every case proves its reach (a vacuous case fails) from the reference's own outputs, with at least MIN_HITS keylines:
new keylines with a forward winner and a directed hit, a winner and no hit, a hit and no winner, neither; no-hit keylines
with a winner whose search range (t_steps, from _search_setup) differs between the winner's (rho, s_rho) and the
detector's; keylines whose match changes when the reference searches the unrotated old map; old keylines probed and hit
with q2 == 0 (no finite rotated depth); regularised keylines whose neighbours took different paths across 256-keyline
block edges; and each EKF clamp branch.  The pose tail is held to a NumPy restatement (Pose, Pos) and to TooN's
SO3::ln (RotLie, PoseLie, within 4e-15: CUDA's asin / acos are not glibc's) in every branch of the logarithm."""
import numpy as np
import pytest

from parity_util import (DM_CASES, EKF_CASES, EUROC_CFG, MIN_HITS, RHO_MAX, RHO_MIN, V_TYP, Bench, _compare,
                         _cut, _depth_state, _diff, _reg_gates, _search_setup, rot, so3_ln_branch, so3_ln_cases)

pytestmark = pytest.mark.gpu

CFG = EUROC_CFG
KITTI_CAM = dict(w=1241, h=376, zfx=718.856, zfy=718.856, ppx=1241 / 2.0 - 13.3, ppy=376 / 2.0 - 2.8)
CAP = 50000            # the benches' kl_capacity
NEW_FIELDS, NEW_MATCHED = ["rho", "s_rho", "rho0", "s_rho0", "m_id", "m_num", "p_m_0"], ["m_m0", "n_m0"]
OLD_FIELDS = ["p_m", "rho", "s_rho", "m_m"]
BASE = dict(V=V_TYP, P_V=np.eye(3) * 1e-4, BackRot=np.eye(3), R0=np.eye(3), do_match=1, thr_mod=1.0, thr_ang=45.0,
            radius=40.0, loc_unc_m=2.0, match_threshold=500, reg_thresh=0.5, q_abs=1e-4, loc_unc=1.0)
PATHS = ("fw_hit", "fw_only", "hit_only", "neither")


def _frames(cam, seed):
    from rebvo_b200 import synth
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=seed, zf=cam["zfx"])
    return seq.frame(10)[1], seq.frame(11)[1]


class ChainBench(Bench):
    """Bench with two more GPU maps for the stage kernels and two more reference maps for the reach probes"""

    def __init__(self, cam, frames):
        from oracle import refapi
        super().__init__(cam, frames, kl_capacity=CAP)
        self.stage = [self.ctx.new_map(), self.ctx.new_map()]
        self.probe = [refapi.RefMap(cam["w"], cam["h"], cam["ppx"], cam["ppy"], cam["zfx"], cam["zfy"], CFG["sigma0"],
                                    CFG["ksigma"]) for _ in range(2)]

    def load_all(self, i, kl, mask):
        self.load(i, kl, mask)
        self.stage[i].load_keylines(np.ascontiguousarray(kl), mask)

    def close(self):
        for g in self.stage:
            g.close()
        super().close()


@pytest.fixture(scope="module")
def bench(built):
    b = ChainBench(CFG["cam"], _frames(CFG["cam"], 7))
    assert min(len(k) for k in b.kl) > 5000
    yield b
    b.close()


@pytest.fixture(scope="module")
def bench_kitti(built):
    b = ChainBench(KITTI_CAM, _frames(KITTI_CAM, 11))
    assert min(len(k) for k in b.kl) > 2000
    yield b
    b.close()


def _offers(kl_old, kn_new, rng, share=2 / 3):
    """m_id_f of the old map: ~70 % of the old keylines offer themselves to a new keyline among the first `share` of the
    new map (so the rest has no winner), a few point at kn_new and beyond (skipped), runs of equal rho make ties"""
    ko = len(kl_old)
    f = np.full(ko, -1, np.int32)
    if kn_new and ko:
        f = rng.integers(0, max(1, int(kn_new * share)), ko).astype(np.int32)
        f[rng.random(ko) < 0.3] = -1
    if ko:
        beyond = rng.choice(ko, min(ko, 6), replace=False)
        f[beyond] = kn_new + np.arange(len(beyond)) * 5
    kl_old["m_id_f"] = f
    return kl_old


def _tiled(kl, mask, k, rng):
    """k keylines: kl tiled (copies after the first moved by a sub-pixel offset); the mask keeps the first copy"""
    if k <= len(kl):
        return _cut(kl, mask, k)
    idx = np.arange(k) % len(kl)
    t = kl[idx].copy()
    cp = (np.arange(k) // len(kl) > 0)[:, None]
    t["p_m"] = (t["p_m"].astype(np.float64) + rng.uniform(-0.3, 0.3, (k, 2)) * cp).astype(np.float32)
    return t, mask


def _ref_chain(ref, probe, kl_old, kl_new, mo, mn, a):
    """the reference's sequence on loaded maps, plus the reach probes; returns what the comparisons and the evidence use"""
    old, new = ref
    dm = (a["V"], a["P_V"], a["BackRot"], a["thr_mod"], a["thr_ang"], a["radius"], a["loc_unc_m"])
    old.forward_match(new)
    fw = new.keylines()
    old.rotate(a["R0"])
    nm = new.directed_matching(old, *dm) if a["do_match"] else 0
    matched = new.keylines()
    r = dict(fw=fw, matched=matched, nmatch=nm, fwd_match=int((fw["m_id"] >= 0).sum()))
    # gate (rebvo_second_t.cpp:410-423); Kp, P_Kp enter as 0, est_ok as 1, klm_num as 0
    g = dict(do_map=0, est_ok=1, klm_num=0, V=np.array(a["V"], np.float64), Kp=0.0, P_Kp=0.0,
             P_V=np.array(a["P_V"], np.float64))
    if a["do_match"]:
        g["klm_num"] = nm
        if nm < a["match_threshold"]:
            g.update(P_V=np.eye(3) * 1e50, V=np.zeros(3), Kp=1.0, P_Kp=10.0, est_ok=0)
        else:
            g["do_map"] = 1
    r["gate"] = g
    r["reg_num"] = 0
    if g["do_map"]:
        r["reg_num"] = new.regularize(a["reg_thresh"])
        new.ekf(g["V"], g["P_V"], np.eye(3) * 1e-4, a["q_abs"], 1.6968e-4, a["loc_unc"])
    r["new"], r["old"] = new.keylines(), old.keylines()
    if not a["do_match"]:
        return r
    # directed hits alone: the searched state after FordwardMatch without its m_id, against the rotated old map
    p_new, p_old = probe
    s = fw.copy()
    s["m_id"] = -1
    p_new.set_keylines(s)
    p_new.set_mask(mn, len(s))
    p_new.directed_matching(old, *dm)
    r["hit"] = p_new.keylines()["m_id"] >= 0
    # the same search against the old map unrotated
    p_old.set_keylines(kl_old)
    p_old.set_mask(mo, len(kl_old))
    p_new.set_keylines(fw)
    p_new.set_mask(mn, len(fw))
    p_new.directed_matching(p_old, *dm)
    r["m_id_unrot"] = p_new.keylines()["m_id"]
    return r


def _gpu_stage(stage, a):
    old, new = stage
    fwd = old.forward_match(new)
    old.rotate(a["R0"])
    nm = new.directed_matching(old, a["V"], a["P_V"], a["BackRot"], a["thr_mod"], a["thr_ang"], a["radius"],
                               a["loc_unc_m"]) if a["do_match"] else 0
    reg = 0
    if a["do_match"] and nm >= a["match_threshold"]:
        reg = new.regularize(a["reg_thresh"])
        new.ekf(a["V"], a["q_abs"], a["loc_unc"])
    return dict(nmatch=nm, fwd_match=fwd, reg_num=reg, new=new.keylines(), old=old.keylines())


def _run(bench, kl_old, kl_new, mo, mn, case, pose=None):
    """the chain on the reference, on the pipeline's kernels and on the stage kernels; (failures, reference result,
    rb_map_match_update's record, arguments)"""
    a = dict(BASE)
    a.update(case)
    mo = bench.mask[0] if mo is None else mo
    mn = bench.mask[1] if mn is None else mn
    bench.load_all(0, kl_old, mo)
    bench.load_all(1, kl_new, mn)
    Pose, Pos, K = pose if pose is not None else (np.eye(3), np.zeros(3), 1.0)
    out = bench.gpu[1].match_update(bench.gpu[0], a["V"], a["P_V"], a["BackRot"], a["R0"], a["do_match"], a["thr_mod"],
                                    a["thr_ang"], a["radius"], a["loc_unc_m"], a["match_threshold"], a["reg_thresh"],
                                    a["q_abs"], a["loc_unc"], Pose, Pos, K)
    chain = dict(new=bench.gpu[1].keylines(), old=bench.gpu[0].keylines())
    r = _ref_chain(bench.ref, bench.probe, kl_old, kl_new, mo, mn, a)
    st = _gpu_stage(bench.stage, a)
    errs = []
    for tag, ref_side, got in (("chain", r, chain), ("stage kernels", st, chain), ("stage kernels vs reference", r, st)):
        errs += ["%s, new map: %s" % (tag, e) for e in _compare(ref_side["new"], got["new"], NEW_FIELDS, NEW_MATCHED)]
        errs += ["%s, old map: %s" % (tag, e) for e in _compare(ref_side["old"], got["old"], OLD_FIELDS)]
    for k in ("nmatch", "fwd_match", "reg_num"):
        if not r[k] == st[k] == out[k]:
            errs.append("%s: reference %d, stage kernels %d, chain %d" % (k, r[k], st[k], out[k]))
    for k, v in r["gate"].items():
        e = _diff("gate " + k, np.asarray(v), np.asarray(out[k]))
        if e:
            errs.append(e)
    return errs, r, out, a


def _paths(r):
    fw = r["fw"]["m_id"] >= 0
    hit = r["hit"]
    return dict(fw_hit=fw & hit, fw_only=fw & ~hit, hit_only=~fw & hit, neither=~fw & ~hit)


def _evidence(bench, r, a, kl_new, want):
    msgs, info = [], {}
    if "paths" in want:
        p = _paths(r)
        info.update({k: int(v.sum()) for k, v in p.items()})
        msgs += ["%s on %d keylines" % (k, v.sum()) for k, v in p.items() if v.sum() < MIN_HITS]
    if "tsteps" in want:   # no hit, a winner, and a search range that depends on which (rho, s_rho) it starts from
        p = _paths(r)["fw_only"]
        t_w = _search_setup(bench, r["fw"], a["V"], a["BackRot"], a["radius"], a["loc_unc_m"])["t_steps"]
        t_d = _search_setup(bench, kl_new, a["V"], a["BackRot"], a["radius"], a["loc_unc_m"])["t_steps"]
        n = int((p & (t_w != t_d)).sum())
        info["t_steps from the winner"] = n
        if n < MIN_HITS:
            msgs.append("t_steps of the winner differ on %d no-hit keylines" % n)
    if "rotation" in want:
        n = int((r["matched"]["m_id"] != r["m_id_unrot"]).sum())
        info["decided by the rotation"] = n
        if n < MIN_HITS:
            msgs.append("the rotation decides %d matches" % n)
    if "reg_edges" in want:   # regularised keylines whose neighbours took different paths, across 256-keyline blocks
        kl = r["matched"]
        nb = (kl["n_id"] >= 0) & (kl["p_id"] >= 0)
        _, g1, g2 = _reg_gates(kl, a["reg_thresh"])
        i = np.nonzero(nb)[0][g1 & g2]
        path = np.select(list(_paths(r).values()), np.arange(4))
        n, pp = kl["n_id"][i], kl["p_id"][i]
        cross = (n // 256 != i // 256) | (pp // 256 != i // 256)
        n_e = int((cross & (path[n] != path[pp])).sum())
        info["regularised across block edges, mixed paths"] = n_e
        if n_e < MIN_HITS or not r["gate"]["do_map"]:
            msgs.append("%d regularised keylines across block edges with mixed paths (gate %d)"
                        % (n_e, r["gate"]["do_map"]))
    return msgs, info


def _state(bench, name, kl_old=None, kl_new=None):
    rng = np.random.default_rng(sum(map(ord, name)))
    kl_new = bench.kl[1] if kl_new is None else kl_new
    kl_old = bench.kl[0] if kl_old is None else kl_old
    kl_new = _depth_state(kl_new, rng, new=True) if len(kl_new) else kl_new.copy()
    kl_old = _depth_state(kl_old, rng) if len(kl_old) else kl_old.copy()
    return _offers(kl_old, len(kl_new), rng), kl_new


# name -> (overrides of BASE, reach to prove)
CASES = {
    "typ": (dict(), ("paths", "tsteps", "reg_edges")),
    "fast": (dict(V=DM_CASES["fast"][0]["V"], P_V=DM_CASES["fast"][0]["RVel"]), ("paths", "tsteps")),
    "V0": (dict(V=np.zeros(3), P_V=np.zeros((3, 3))), ("paths",)),
    "tsteps0to8": (dict(V=DM_CASES["tsteps0to8"][0]["V"], loc_unc_m=0.0), ("paths", "tsteps")),
    "ang10_mod0.1": (dict(thr_ang=10.0, thr_mod=0.1), ("tsteps",)),
}
# rotation cases (_rot_state): V = 0, so each new keyline's search starts at its own pixel of the old frame; every old
# rho sits within 5 % of LocationUncertaintyMatch with a tiny s_rho, so that the depth test turns on q2 (x and y turns),
# and for turns about z (q2 = 1) the angle window is 2 degrees, so that a 3 degree turn of the gradient closes it
ROT = dict(V=np.zeros(3), P_V=np.zeros((3, 3)), loc_unc_m=1.0, match_threshold=0)
for _ax, _n in enumerate("xyz"):
    _a = dict(ROT, thr_ang=2.0 if _n == "z" else 45.0)
    CASES["R0_%s3" % _n] = (dict(_a, R0=rot(_ax, 3.0), BackRot=rot(_ax, 3.0).T), ("rotation",))
    CASES["R0_%s3_indep" % _n] = (dict(_a, R0=rot(_ax, 3.0), BackRot=rot((_ax + 1) % 3, -2.0)), ("rotation",))
CASES["R0_y25"] = (dict(ROT, thr_ang=45.0, R0=rot(1, 25.0), BackRot=rot(1, 25.0).T), ("rotation",))
CASES["R0_x-25_indep"] = (dict(ROT, thr_ang=45.0, R0=rot(0, -25.0), BackRot=rot(2, 4.0)), ("rotation",))


def _rot_state(bench, name):
    kl_old, kl_new = _state(bench, name, bench.kl[0], bench.kl[0])
    rng = np.random.default_rng(sum(map(ord, name)) + 1)
    kl_old["rho"] = ROT["loc_unc_m"] * rng.uniform(0.95, 1.05, len(kl_old))
    kl_old["s_rho"] = rng.uniform(1e-4, 1e-3, len(kl_old))
    return kl_old, kl_new


@pytest.mark.parametrize("name", list(CASES))
def test_chain(bench, name):
    case, want = CASES[name]
    if "rotation" in want:
        (kl_old, kl_new), masks = _rot_state(bench, name), (bench.mask[0], bench.mask[0])
    else:
        (kl_old, kl_new), masks = _state(bench, name), (None, None)
    errs, r, out, a = _run(bench, kl_old, kl_new, *masks, case)
    vac, info = _evidence(bench, r, a, kl_new, want)
    print("%s: nmatch %d fwd %d reg %d gate %d; %s" % (name, r["nmatch"], r["fwd_match"], r["reg_num"],
                                                        r["gate"]["do_map"], info))
    assert not vac, "vacuous case: %s" % vac
    assert not errs, "\n".join(errs)


def test_chain_q2_zero(bench):
    """R0 = 90 degrees about x exactly: q2 = p_m.y / zf, so an old keyline with p_m.y = 0 has no finite rotated depth
    (fabs(q2) > 0 fails) and keeps p_m, rho, s_rho.  The new map is the old frame's keylines, V = 0 (the search starts at
    the keyline's own pixel), and the gradients of the seeded keylines horizontal, so that their rotated gradient passes
    the angle test: they are probed and hit."""
    R0 = np.array([[1.0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]])
    rng = np.random.default_rng(90)
    kl = bench.kl[0]
    kl_old = _depth_state(kl, rng)
    kl_new = _depth_state(kl, rng, new=True)
    sel = np.sort(rng.choice(len(kl), 400, replace=False))
    kl_old["p_m"][sel, 1] = 0.0
    for k in (kl_old, kl_new):
        k["m_m"][sel, 1] = 0.0
        k["m_m"][sel, 0] = np.where(kl["m_m"][sel, 0] < 0, -1, 1) * kl["n_m"][sel]
    kl_old = _offers(kl_old, len(kl_new), rng)
    case = dict(V=np.zeros(3), P_V=np.zeros((3, 3)), R0=R0, BackRot=np.eye(3), match_threshold=0)
    errs, r, out, a = _run(bench, kl_old, kl_new, bench.mask[0], bench.mask[0], case)
    q2_zero = np.zeros(len(kl_old), bool)
    q2_zero[sel] = True
    m = r["matched"]["m_id"]
    hit = r["hit"] & (m >= 0)
    n = int(q2_zero[m[hit]].sum())
    print("old keylines with q2 == 0: %d, hit %d times; nmatch %d" % (len(sel), n, r["nmatch"]))
    assert n >= 8, "only %d hits on keylines with q2 == 0" % n
    assert not errs, "\n".join(errs)


def test_chain_no_match(bench):
    """do_match = 0 (the minimiser's NaN guard): no search, the winners kept, the gate closed, the old map still rotated"""
    kl_old, kl_new = _state(bench, "do_match0")
    case = dict(do_match=0, R0=rot(1, 3.0), BackRot=rot(1, 3.0).T, match_threshold=0)
    errs, r, out, a = _run(bench, kl_old, kl_new, None, None, case)
    fw = int((r["fw"]["m_id"] >= 0).sum())
    print("do_match 0: %d winners, nmatch %d, do_map %d" % (fw, out["nmatch"], out["do_map"]))
    assert fw >= MIN_HITS and out["nmatch"] == 0 and out["do_map"] == 0 and out["reg_num"] == 0
    assert _diff("old p_m", kl_old["p_m"], r["old"]["p_m"]), "the old map was not rotated"
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("offset", [0, 1])
def test_chain_match_threshold(bench, offset):
    """MatchThreshold at the reference's own count (the gate opens: nmatch >= MatchThreshold) and one above it"""
    kl_old, kl_new = _state(bench, "typ")
    _, r, _, _ = _run(bench, kl_old, kl_new, None, None, {})
    assert r["nmatch"] >= MIN_HITS
    errs, r2, out, _ = _run(bench, kl_old, kl_new, None, None, dict(match_threshold=r["nmatch"] + offset))
    print("MatchThreshold %d: nmatch %d, do_map %d" % (r["nmatch"] + offset, out["nmatch"], out["do_map"]))
    assert out["do_map"] == (offset == 0) and r2["nmatch"] == r["nmatch"]
    assert not errs, "\n".join(errs)


SIZES = [(nk, ok) for nk in (0, 1, 31, 32, 33, 4001, CAP) for ok in ("zero", "more", "cap") if not (nk == CAP and ok == "more")]


@pytest.mark.parametrize("nk,ok", SIZES)
def test_chain_sizes(bench, nk, ok):
    """new kn at the kernels' block edges (32 keylines per k_match block, 256 per k_reg_ekf block) and at the capacity;
    old kn 0, above the new map's, and the capacity (tiled)"""
    rng = np.random.default_rng(nk * 3 + len(ok))
    ko = dict(zero=0, more=nk + 37, cap=CAP)[ok]
    kl_new, mn = _tiled(bench.kl[1], bench.mask[1], nk, rng)
    kl_old, mo = _tiled(bench.kl[0], bench.mask[0], ko, rng)
    if ko == 0:
        mo = np.full_like(bench.mask[0], -1)
    kl_old, kl_new = _state(bench, "sizes%d%s" % (nk, ok), kl_old, kl_new)
    errs, r, out, _ = _run(bench, kl_old, kl_new, mo, mn, dict(match_threshold=min(500, nk // 4)))
    print("new %d old %d: nmatch %d fwd %d reg %d gate %d" % (nk, ko, r["nmatch"], r["fwd_match"], r["reg_num"],
                                                               r["gate"]["do_map"]))
    assert not errs, "\n".join(errs)


def test_chain_ekf_clamps(bench):
    """the EKF after the regularisation, in every clamp branch of UpdateInverseDepthKalmanARLU (EKF_CASES' velocities,
    Q and localisation uncertainties; the gate open)"""
    seen = dict(min=0, max=0, nan=0, normal=0)
    fails = []
    for name, (vel, q_abs, loc_unc, ones) in EKF_CASES.items():
        kl_old, kl_new = _state(bench, "ekf" + name)
        kl_old["rho"][np.random.default_rng(len(name)).random(len(kl_old)) < ones] = 1.0
        case = dict(V=vel, q_abs=q_abs, loc_unc=loc_unc, match_threshold=0)
        errs, r, _, _ = _run(bench, kl_old, kl_new, None, None, case)
        fails += ["%s: %s" % (name, e) for e in errs]
        kl = r["new"]
        mk = kl["m_id"] >= 0
        rho, s = kl["rho"][mk], kl["s_rho"][mk]
        nan_br = (rho == 1.0) & (s == RHO_MAX)
        br = dict(min=rho == RHO_MIN, max=rho == RHO_MAX, nan=nan_br, normal=(rho > RHO_MIN) & (rho < RHO_MAX) & ~nan_br)
        print("%s: %s" % (name, {b: int(m.sum()) for b, m in br.items()}))
        for b, m in br.items():
            seen[b] += int(m.sum())
    print("clamp branches over all cases:", seen)
    assert not fails, "\n".join(fails[:20])
    assert min(seen.values()) >= MIN_HITS, seen


@pytest.mark.parametrize("name", ["typ", "fast"])
def test_chain_1241x376(bench_kitti, name):
    kl_old, kl_new = _state(bench_kitti, name)
    errs, r, _, a = _run(bench_kitti, kl_old, kl_new, None, None, CASES[name][0])
    vac, info = _evidence(bench_kitti, r, a, kl_new, ("paths",))
    print("1241x376 %s: %s" % (name, info))
    assert not vac, "vacuous case: %s" % vac
    assert not errs, "\n".join(errs)


# ---- the pose tail ------------------------------------------------------------------------------------------------------
def _mat3_mul(A, B):
    """TooN's Matrix * Matrix: each dot product accumulates from 0 in index order"""
    C = np.zeros((3, 3))
    for i in range(3):
        for j in range(3):
            s = 0.0
            for k in range(3):
                s = s + float(A[i, k]) * float(B[k, j])
            C[i, j] = s
    return C


def _pose_step(Pose, R, V, Pos, K):
    """rebvo_second_t.cpp:545-551: Pose = Pose * R; Pos += -Pose * V * K"""
    P = _mat3_mul(Pose, R)
    out = np.zeros(3)
    for i in range(3):
        s = 0.0
        for k in range(3):
            s = s + (-P[i, k]) * float(V[k])
        out[i] = float(Pos[i]) + s * K
    return P, out


def test_chain_pose_tail(bench):
    """Pose * R in every branch of SO3::ln (and matrices coerce must re-orthonormalise), R itself in every branch"""
    from oracle import refapi
    rng = np.random.default_rng(4)
    kl_old, kl_new = _state(bench, "pose", _cut(bench.kl[0], bench.mask[0], 64)[0], _cut(bench.kl[1], bench.mask[1], 64)[0])
    mo, mn = _cut(bench.kl[0], bench.mask[0], 64)[1], _cut(bench.kl[1], bench.mask[1], 64)[1]
    B = rot(1, 3.0).T
    runs = []
    for name, M in so3_ln_cases().items():
        runs.append(("Pose*R " + name, M @ B.T, B))
        if np.allclose(M @ M.T, np.eye(3), atol=1e-12):
            runs.append(("R " + name, np.eye(3), M))
    seen_pose, seen_rot, fails = set(), set(), []
    for name, Pose, R in runs:
        Pos, K = rng.normal(0, 1, 3), 1.3
        # (do_match = 0: a back-rotation by up to 180 degrees leaves nothing to search for; the gate keeps V)
        errs, r, out, a = _run(bench, kl_old, kl_new, mo, mn, dict(BackRot=R, R0=R.T, do_match=0), pose=(Pose, Pos, K))
        fails += ["%s: %s" % (name, e) for e in errs]
        P, p = _pose_step(Pose, R, r["gate"]["V"], Pos, K)
        for tag, want, got in (("Pose", P, out["Pose"]), ("Pos", p, out["Pos"])):
            if _diff(tag, want, got):
                fails.append("%s: %s" % (name, _diff(tag, want, got)))
        for tag, M, got in (("RotLie", R, out["RotLie"]), ("PoseLie", P, out["PoseLie"])):
            err = np.abs(refapi.so3_ln(M) - got).max()
            if not err <= 4e-15:
                fails.append("%s: %s off TooN's SO3::ln by %.3g" % (name, tag, err))
        seen_pose.add(so3_ln_branch(P))
        seen_rot.add(so3_ln_branch(R))
    want = {("above", None, False), ("between", None, False)} | {("below", s, f) for s in range(3) for f in (False, True)}
    print("branches of Pose: %s; of R: %s" % (sorted(map(str, seen_pose)), sorted(map(str, seen_rot))))
    assert want <= seen_pose and want <= seen_rot, (want - seen_pose, want - seen_rot)
    assert not fails, "\n".join(fails[:20])

"""The mapper stages on edge-map states that reach every branch, against the reference compiled into oracle/_ref.

DESIGN.md section 3 says directed matching, FordwardMatch, Regularize_1_iter, the EKF, EstimateQuantile and the
rescaling are bit-identical to the reference (per-keyline float64, contraction off).  The stage test of
test_gpu_parity.py runs them once, on an old map whose keylines all hold rho = 1, s_rho = 0.2: most branches never run
there.  Here the depth state of two detected 752x480 EuRoC-like frames is overwritten with seeded values chosen per
branch, loaded on both sides (RefMap.set_keylines + set_mask, Map.load_keylines), and each stage is compared bit for bit.
Every case proves that it reached its target branch, either through a NumPy restatement of the set-up lines (never the
search or the update itself) or through the outputs, for at least MIN_HITS keylines; a case that does not is vacuous and
fails.

Domain.  The states stay inside what the per-frame flow produces: rho in [RHO_MIN, RHO_MAX] (log-uniform, plus exact
1e-3, 1.0 and 20.0, plus runs of equal values), s_rho in [1e-6, 20] (s_rho > rho included), m_num in 0..10, and new
keylines with m_id = -1 before FordwardMatch, as after detection.  Signed-zero or NaN rho and a pre-set m_id on the new
map are outside it: there FordwardMatch's arg-max over a monotonic integer key of rho and the reference's sequential
"replace unless strictly larger" rule part ways (-0.0 < +0.0 for the key, equal for `>`; NaN compares false).

The second half runs the whole per-frame pipeline against the reference's own three-thread REBVO on streams that take
the rescaling, the serial quantile, a static stretch and a fast camera, with the bars of test_long_run_752x480."""
import numpy as np
import pytest

from parity_util import (DM_BASE, DM_CASES, EKF_CASES, EUROC_CFG, MIN_HITS, RHO_MAX, RHO_MIN, V_TYP, Bench, _bits, _compare,
                         _cut, _depth_state, _diff, _reg_gates, _search_setup)
from pipeline_util import assert_tight, euroc_stream, run_both, run_pipeline

pytestmark = pytest.mark.gpu

CFG = EUROC_CFG
KITTI_CAM = dict(w=1241, h=376, zfx=718.856, zfy=718.856, ppx=1241 / 2.0 - 13.3, ppy=376 / 2.0 - 2.8)


def _frames(cam, seed):
    from rebvo_b200 import synth
    seq = synth.Sequence(w=cam["w"], h=cam["h"], seed=seed, zf=cam["zfx"])
    return seq.frame(10)[1], seq.frame(11)[1]


@pytest.fixture(scope="module")
def bench(built):
    b = Bench(CFG["cam"], _frames(CFG["cam"], 7))
    assert min(len(k) for k in b.kl) > 5000
    yield b
    b.close()


@pytest.fixture(scope="module")
def bench_kitti(built):
    b = Bench(KITTI_CAM, _frames(KITTI_CAM, 11))
    assert min(len(k) for k in b.kl) > 2000
    yield b
    b.close()


# ---- 1. directed_matching ---------------------------------------------------------------------------------------------
def _run_dm(bench, kl_old, kl_new, mo, mn, case):
    a = dict(DM_BASE)
    a.update(case)
    bench.load(0, kl_old, mo)
    bench.load(1, kl_new, mn)
    args = (a["V"], a["RVel"], a["BackRot"], a["thr_mod"], a["thr_ang"], a["radius"], a["loc_unc"])
    n_r = bench.ref[1].directed_matching(bench.ref[0], *args)
    n_g = bench.gpu[1].directed_matching(bench.gpu[0], *args)
    r, g = bench.ref[1].keylines(), bench.gpu[1].keylines()
    errs = [] if n_r == n_g else ["count ref %d gpu %d" % (n_r, n_g)]
    errs += _compare(r, g, ["rho", "s_rho", "m_id", "m_num", "p_m_0"], ["m_m0", "n_m0"])
    return errs, n_r, a


def _check_branches(st, want, kn):
    msgs = []
    for br, least in want.items():
        if br == "tsteps":
            got = [int((st["t_steps"][st["normal"]] == v).sum()) for v in range(9)]
            if min(got) < least:
                msgs.append("t_steps 0..8 counts %s" % got)
            continue
        got = int(st[br].sum())
        if (least < 0 and got != kn) or (least >= 0 and got < least):
            msgs.append("branch %s on %d of %d keylines" % (br, got, kn))
    return msgs


@pytest.mark.parametrize("name", list(DM_CASES))
def test_directed_matching(bench, name):
    case, want = DM_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    kl_old = _depth_state(bench.kl[0], rng)
    kl_new = _depth_state(bench.kl[1], rng, new=True)
    errs, n, a = _run_dm(bench, kl_old, kl_new, None, None, case)
    st = _search_setup(bench, kl_new, a["V"], a["BackRot"], a["radius"], a["loc_unc"])
    vac = _check_branches(st, want, len(kl_new))
    print("%s: %d matches of %d; perp %d mid %d normal %d cut %d" % (name, n, len(kl_new), st["perp"].sum(),
                                                                      st["mid"].sum(), st["normal"].sum(),
                                                                      st["cut"].sum()))
    assert not vac, "vacuous case: %s" % vac
    assert n >= MIN_HITS, "only %d matches" % n
    assert not errs, "\n".join(errs)


def test_directed_matching_probes_leave_every_edge(bench):
    """The back-rotations together put search windows across all four image edges (GetIndexRC's -1)."""
    edges = np.zeros(4, np.int64)
    for name in ("rot_x3", "rot_y3", "rot_z3", "rot_y25", "rot_y-25", "V0"):
        case, _ = DM_CASES[name]
        a = dict(DM_BASE)
        a.update(case)
        kl_new = _depth_state(bench.kl[1], np.random.default_rng(sum(map(ord, name))), new=True)
        st = _search_setup(bench, kl_new, a["V"], a["BackRot"], a["radius"], a["loc_unc"])
        edges += st["edges"].sum(0)
    print("windows across the left / right / top / bottom edge:", edges.tolist())
    assert (edges >= MIN_HITS).all(), edges


def test_directed_matching_kn_not_multiple_of_32(bench):
    rng = np.random.default_rng(5)
    ko, mo = _cut(bench.kl[0], bench.mask[0], 4001)
    kn, mn = _cut(bench.kl[1], bench.mask[1], 3001)
    assert len(ko) % 32 and len(kn) % 32
    errs, n, _ = _run_dm(bench, _depth_state(ko, rng), _depth_state(kn, rng, new=True), mo, mn, {})
    assert n >= MIN_HITS and not errs, errs


@pytest.mark.parametrize("name", ["typ", "rot_y25", "V0"])
def test_directed_matching_1241x376(bench_kitti, name):
    case = {"typ": {}, "rot_y25": DM_CASES["rot_y25"][0], "V0": DM_CASES["V0"][0]}[name]
    rng = np.random.default_rng(17)
    errs, n, _ = _run_dm(bench_kitti, _depth_state(bench_kitti.kl[0], rng),
                         _depth_state(bench_kitti.kl[1], rng, new=True), None, None, case)
    assert n >= MIN_HITS and not errs, errs


# ---- 2. FordwardMatch -------------------------------------------------------------------------------------------------
def test_forward_match_injected(bench):
    """m_id_f of the old map injected: -1, in range with many offers per new keyline (exact rho ties among them), and
    >= the new map's kn (the reference skips those, edge_tracker.cpp:402).  Winner of a target = the offer with the
    largest rho, ties to the largest old index.  The count returned is the number of new keylines that got a match; the
    reference's counts every accepted offer, overwritten ones included, so only the keylines are compared with it."""
    rng = np.random.default_rng(23)
    old = _depth_state(bench.kl[0], rng)
    new = _depth_state(bench.kl[1], rng, new=True)
    ko, kn = len(old), len(new)
    f = rng.integers(0, kn // 3, ko)                       # ~3 offers per target on average
    u = rng.random(ko)
    f[u < 0.3] = -1
    beyond = rng.choice(ko, 12, replace=False)
    f[beyond] = kn + np.arange(12) * 7                    # kn itself included
    old["m_id_f"] = f
    disc = rng.random(ko) < 0.5                           # exact ties: half of the offers from three values
    old["rho"][disc] = rng.choice([0.25, 1.0, 4.0], disc.sum())
    offers = (f >= 0) & (f < kn)
    tgt, rho = f[offers], old["rho"][offers]
    mx = np.full(kn, -np.inf)
    np.maximum.at(mx, tgt, rho)
    ties = np.bincount(tgt[rho == mx[tgt]], minlength=kn)
    print("targets %d, tie groups %d" % ((mx > -np.inf).sum(), (ties >= 2).sum()))
    assert (ties >= 2).sum() >= MIN_HITS, "no tie groups"
    bench.load(0, old)
    bench.load(1, new)
    bench.ref[0].forward_match(bench.ref[1])
    n_g = bench.gpu[0].forward_match(bench.gpu[1])
    r, g = bench.ref[1].keylines(), bench.gpu[1].keylines()
    errs = _compare(r, g, ["rho", "s_rho", "m_num", "m_id", "p_m_0"], ["m_m0", "n_m0"])
    assert not errs, "\n".join(errs)
    assert (r["m_id"] >= 0).sum() == (mx > -np.inf).sum()
    assert n_g == int((r["m_id"] >= 0).sum()), n_g


# ---- 3. Regularize_1_iter ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("thresh", [0.0, 0.5, 0.95])
def test_regularize(bench, thresh):
    rng = np.random.default_rng(int(thresh * 100) + 3)
    kl = _depth_state(bench.kl[1], rng)
    # spread: neighbours of a third of the keylines get a nearby depth, so that the uncertainty gate opens often too
    ni = kl["n_id"]
    near = (ni >= 0) & (rng.random(len(kl)) < 0.35)
    kl["rho"][ni[near]] = np.clip(kl["rho"][near] * np.exp(rng.normal(0, 0.05, near.sum())), RHO_MIN, RHO_MAX)
    # ... and a sixth of the gradients turn by a random angle (edges along a chain are nearly parallel: the angle gate
    # would hardly ever close)
    turn = rng.random(len(kl)) < 0.17
    a = rng.uniform(-np.pi, np.pi, turn.sum())
    mx, my = kl["m_m"][turn, 0].astype(np.float64), kl["m_m"][turn, 1].astype(np.float64)
    kl["m_m"][turn, 0] = mx * np.cos(a) - my * np.sin(a)
    kl["m_m"][turn, 1] = mx * np.sin(a) + my * np.cos(a)
    nnb, g1, g2 = _reg_gates(kl, thresh)
    frac = lambda m: m.sum() / float(nnb)   # noqa: E731
    print("thresh %.2f: %d keylines with neighbours; uncertainty gate open %.3f, angle gate open %.3f (of those open: "
          "%.3f), both %.3f" % (thresh, nnb, frac(g1), frac(g2), (g2 & g1).sum() / max(g1.sum(), 1), frac(g1 & g2)))
    assert 0.05 <= frac(g1) <= 0.95, "uncertainty gate does not both open and close"
    assert frac(g1 & g2) >= 0.05 and frac(g1 & ~g2) >= 0.05, "angle gate does not both open and close"
    bench.load(1, kl)
    n_r = bench.ref[1].regularize(thresh)
    n_g = bench.gpu[1].regularize(thresh)
    assert n_r == n_g == int((g1 & g2).sum()), (n_r, n_g, int((g1 & g2).sum()))
    errs = _compare(bench.ref[1].keylines(), bench.gpu[1].keylines(), ["rho", "s_rho"])
    assert not errs, "\n".join(errs)


# ---- 4. EKF -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def matched_state(bench):
    """A new map after directed matching on the reference (m_id, p_m_0, m_m0, n_m0 of real matches)."""
    rng = np.random.default_rng(31)
    bench.load(0, _depth_state(bench.kl[0], rng))
    bench.load(1, _depth_state(bench.kl[1], rng, new=True))
    n = bench.ref[1].directed_matching(bench.ref[0], V_TYP, np.eye(3) * 1e-4, np.eye(3), 1.0, 45.0, 40.0, 2.0)
    assert n > 1000
    return bench.ref[1].keylines()


def test_ekf_every_clamp_branch(bench, matched_state):
    """UpdateInverseDepthKalmanARLU's clamps (edge_tracker.cpp:1035-1050) from the outputs: rho = RHO_MIN (the s_rho
    correction), rho = RHO_MAX, the NaN/inf reset to (RhoInit, RHO_MAX), and the normal path.  The fourth clamp,
    s_rho < 0, cannot be reached: s_rho = sqrt(v) is NaN (caught before it) or >= +0."""
    seen = dict(min=0, max=0, nan=0, normal=0)
    fails = []
    for name, (vel, q_abs, loc_unc, ones) in EKF_CASES.items():
        rng = np.random.default_rng(sum(map(ord, name)))
        kl = matched_state.copy()
        k = len(kl)
        kl["rho"] = np.exp(rng.uniform(np.log(RHO_MIN), np.log(RHO_MAX), k))
        kl["s_rho"] = np.exp(rng.uniform(np.log(1e-6), np.log(20.0), k))
        kl["rho"][rng.random(k) < ones] = 1.0
        bench.load(1, kl)
        bench.ref[1].ekf(vel, np.eye(3) * 1e-4, np.eye(3) * 1e-4, q_abs, 1.6968e-4, loc_unc)
        bench.gpu[1].ekf(vel, q_abs, loc_unc)
        r, g = bench.ref[1].keylines(), bench.gpu[1].keylines()
        errs = _compare(r, g, ["rho", "s_rho", "rho0", "s_rho0", "m_id"])
        fails += ["%s: %s" % (name, e) for e in errs]
        mk = r["m_id"] >= 0
        rho, s = r["rho"][mk], r["s_rho"][mk]
        nan_br = (rho == 1.0) & (s == RHO_MAX)
        br = dict(min=rho == RHO_MIN, max=rho == RHO_MAX, nan=nan_br,
                  normal=(rho > RHO_MIN) & (rho < RHO_MAX) & ~nan_br)
        print("%s: %s" % (name, {b: int(m.sum()) for b, m in br.items()}))
        for b, m in br.items():
            seen[b] += int(m.sum())
        assert len(errs) or mk.sum() > 1000
    print("clamp branches over all cases:", seen)
    assert not fails, "\n".join(fails)
    assert min(seen.values()) >= MIN_HITS, seen


# ---- 5. EstimateQuantile --------------------------------------------------------------------------------------------
def _specials(n, smin=RHO_MIN, smax=RHO_MAX):
    rng_ = smax - smin
    big = 2.0 ** 31 * rng_ / n + smin   # n * (s - smin) / range = 2^31: the first value out of int range
    return np.array([smin + 3 * rng_ / n, smin + (n - 1) * rng_ / n, smin, 0.0, 5e-4, smax, 25.0, 1e4,
                     np.nextafter(big, 0), big, np.nextafter(big, np.inf), 1e12, 1e300, np.inf])


def _quantile_both(bench, s_rho, smin, smax, perc, n):
    kl = np.zeros(len(s_rho), bench.kl[0].dtype)
    kl["s_rho"] = s_rho
    empty = np.full((bench.cam["h"], bench.cam["w"]), -1, np.int32)
    bench.load(0, kl, empty)
    return bench.ref[0].quantile(smin, smax, perc, n), bench.gpu[0].quantile(smin, smax, perc, n)


def test_quantile(bench):
    """Both bin-scan paths (n <= 128: warp scan; n > 128: serial loop), every threshold position, and s_rho on bin edges,
    outside [smin, smax], at n (s - smin) / range = 2^31 and beyond, and +inf.  Out of int range the reference's
    conversion (x86-64 cvttsd2si) gives INT_MIN, clamped to bin 0; a saturating conversion would put it in bin n-1."""
    rng = np.random.default_rng(41)
    fails, hits = [], 0
    for n in (1, 7, 100, 128, 129, 1000, 4096):
        sp = _specials(n)
        for perc in (0.0, 0.9, 1.0):
            for kn in (0, 33, 20000):
                s = np.exp(rng.uniform(np.log(1e-6), np.log(20.0), kn))
                if kn:
                    s[rng.choice(kn, min(kn, len(sp)), replace=False)] = sp[:kn]
                q_r, q_g = _quantile_both(bench, s, RHO_MIN, RHO_MAX, perc, n)
                if _bits(np.float64(q_r)) != _bits(np.float64(q_g)):
                    fails.append("n=%d perc=%g kn=%d: ref %.17g gpu %.17g" % (n, perc, kn, q_r, q_g))
            for v in sp:   # kn = 1: perc = 0 returns the edge after the value's bin
                q_r, q_g = _quantile_both(bench, np.array([v]), RHO_MIN, RHO_MAX, perc, n)
                if _bits(np.float64(q_r)) != _bits(np.float64(q_g)):
                    fails.append("n=%d perc=%g s_rho=%r: ref %.17g gpu %.17g" % (n, perc, v, q_r, q_g))
                hits += perc == 0.0 and v >= sp[9] and q_r == RHO_MIN + (RHO_MAX - RHO_MIN) / n
    assert not fails, "\n".join(fails[:20])
    assert hits >= 7 * 4, "out-of-range values not in bin 0 on the reference: %d" % hits


def test_reestimate_one_keyline(bench):
    """reEstimateThresh on a one-keyline map: range 0, bin n (max - n_m) / range = 0/0 = NaN -> bin 0 on both sides."""
    kl, m = _cut(bench.kl[1], bench.mask[1], 1)
    bench.load(1, kl, m)
    _, t_r = bench.ref[1].reestimate(CFG["track_points"], 100)
    t_g = bench.gpu[1].reestimate(CFG["track_points"], 100)
    assert _bits(np.float32(t_r)) == _bits(np.float32(t_g)), (t_r, t_g)
    assert np.float32(t_r) == kl["n_m"][0]


# ---- 6. EstimateReScalingOpt ----------------------------------------------------------------------------------------
def _rescale_state(k, rng, valid_tail=0):
    from oracle import refapi
    kl = np.zeros(k, refapi.KEYLINE)
    kl["rho"] = np.exp(rng.uniform(np.log(RHO_MIN), np.log(RHO_MAX), k))
    kl["rho0"] = kl["rho"] * np.exp(rng.normal(0, 0.1, k))
    kl["s_rho"] = np.exp(rng.uniform(np.log(1e-6), np.log(20.0), k))
    kl["s_rho0"] = np.exp(rng.uniform(np.log(1e-6), np.log(20.0), k))
    kl["s_rho0"][rng.random(k) < 0.05] = 0.0
    kl["m_num"] = rng.integers(0, 11, k)
    kl["m_id"] = -1
    if valid_tail:   # keylines past the kernel's register window (16384 per cluster) weigh as much as the heaviest others
        t = slice(k - valid_tail, k)
        kl["m_num"][t], kl["s_rho"][t], kl["s_rho0"][t] = 10, 1e-6, 1e-6
        kl["rho"][t] = np.exp(rng.uniform(0.0, np.log(RHO_MAX), valid_tail))
        kl["rho0"][t] = kl["rho"][t] * 3.0
    return kl


RS_CASES = [(kn, mnm) for kn in (1, 16384, 16385, 30000) for mnm in (0, 1, 5)]


@pytest.mark.parametrize("re_escale", [0, 1])
@pytest.mark.parametrize("kn,mnm", RS_CASES)
def test_rescale(bench, kn, mnm, re_escale):
    rng = np.random.default_rng(kn + 10 * mnm + 100 * re_escale)
    kl = _rescale_state(kn, rng, valid_tail=min(kn, max(0, kn - 16384) + 1))
    s_rho_min = float(np.median(kl["s_rho"])) if kn > 1 else RHO_MAX
    valid = ~((kl["m_num"] < mnm) | (kl["s_rho0"] <= 0) | (kl["s_rho"] > s_rho_min))
    assert valid.sum() >= min(kn, MIN_HITS) and (~valid).sum() >= (MIN_HITS if kn > 1 else 0)
    empty = np.full((bench.cam["h"], bench.cam["w"]), -1, np.int32)
    bench.load(1, kl, empty)
    kp_r, rkp_r = bench.ref[1].rescale(s_rho_min, mnm, re_escale)
    kp_g, rkp_g = bench.gpu[1].rescale(s_rho_min, mnm, re_escale)
    assert kp_r != 1.0
    assert abs(kp_g - kp_r) <= 1e-12 * abs(kp_r) and abs(rkp_g - rkp_r) <= 1e-12 * abs(rkp_r), (kp_r, kp_g, rkp_r, rkp_g)
    g = bench.gpu[1].keylines()
    want_r = kl["rho"] / kp_g if re_escale else kl["rho"]
    want_s = kl["s_rho"] / kp_g if re_escale else kl["s_rho"]
    errs = [_diff("rho", want_r, g["rho"]), _diff("s_rho", want_s, g["s_rho"])]
    assert not any(errs), errs


def test_rescale_degenerate(bench):
    """kn = 0 (Kp = 1, RKp left to the caller) and a map without one valid keyline (Kp = 1, RKp = 1 / 0 = inf)."""
    empty = np.full((bench.cam["h"], bench.cam["w"]), -1, np.int32)
    for re_escale in (0, 1):
        bench.load(1, _rescale_state(0, np.random.default_rng(1)), empty)
        assert bench.ref[1].rescale(RHO_MAX, 1, re_escale)[0] == bench.gpu[1].rescale(RHO_MAX, 1, re_escale)[0] == 1.0
        kl = _rescale_state(20000, np.random.default_rng(2))
        for mnm, s_rho_min in ((11, RHO_MAX), (0, 1e-9)):
            bench.load(1, kl, empty)
            r = bench.ref[1].rescale(s_rho_min, mnm, re_escale)
            g = bench.gpu[1].rescale(s_rho_min, mnm, re_escale)
            assert r == g == (1.0, np.inf), (r, g)
            assert not _diff("rho", kl["rho"], bench.gpu[1].keylines()["rho"])


# ---- B. the per-frame pipeline against the reference's three-thread REBVO -------------------------------------------
NAV_FIELDS = ("Pos", "Pose", "kn", "matches", "Kp", "RKp", "score", "s_rho_p")


def test_pipeline_rescaling(built, tmp_path, monkeypatch):
    """DoReScaling = 1: the rescaled map goes into the next frame (the inline map update); batch 7 == batch 20 and graph
    replay == eager launches, bit for bit."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(60)
    p = capi.default_params(synth.EUROC, DoReScaling=1.0)
    rec, nav = run_both(tmp_path, ts, fr, p, batch=20)
    assert_tight(rec, nav, 58)
    assert np.abs(nav["Kp"][2:] - 1.0).max() > 1e-6, "no rescaling happened"
    b7 = run_pipeline(p, ts, fr, 7).nav
    monkeypatch.setenv("REBVO_B200_NO_GRAPH", "1")
    eager = run_pipeline(p, ts, fr, 20).nav
    monkeypatch.delenv("REBVO_B200_NO_GRAPH")
    for f in NAV_FIELDS:
        assert not _diff(f, nav[f], b7[f][:len(nav)]), ("batch 7", f)
        assert not _diff(f, nav[f], eager[f][:len(nav)]), ("eager", f)


def test_pipeline_static_stretch(built, tmp_path):
    """12 identical frames inside a walk, as at the start of a EuRoC sequence: V shrinks towards 0 and directed matching
    searches along shorter and shorter epipolar segments."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(40)
    fr = np.concatenate([fr[:20], np.repeat(fr[20:21], 12, axis=0), fr[21:]])
    ts = np.arange(len(fr)) / 20.0
    rec, nav = run_both(tmp_path, ts, fr, capi.default_params(synth.EUROC), batch=10)
    assert_tight(rec, nav, len(fr) - 2)
    vz = np.linalg.norm(nav["V"][21:32], axis=1) * synth.EUROC["zfx"]
    print("smallest |V| * zf in the static stretch: %.3e px" % vz.min())
    assert vz.min() < 0.5


def test_pipeline_serial_quantile(built, tmp_path):
    """QCutOffNumBins = 200: EstimateQuantile's serial bin loop in every frame."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(60)
    rec, nav = run_both(tmp_path, ts, fr, capi.default_params(synth.EUROC, QCutOffNumBins=200), batch=20)
    assert_tight(rec, nav, 58)
    plain = run_pipeline(capi.default_params(synth.EUROC), ts, fr, 20).nav
    assert not np.array_equal(nav["s_rho_p"][2:], plain["s_rho_p"][2:])


def test_pipeline_fast_stream(built, tmp_path):
    """Four times the default camera speed: the directed search window is clamped at SearchRange."""
    from rebvo_b200 import capi, synth
    ts, fr = euroc_stream(40, speed=0.024)
    p = capi.default_params(synth.EUROC)
    rec, nav = run_both(tmp_path, ts, fr, p, batch=20)
    assert_tight(rec, nav, 38)
    px = np.linalg.norm(nav["V"][2:, :2], axis=1) * synth.EUROC["zfx"] * RHO_MAX
    print("largest |V_xy| * zf * RHO_MAX: %.1f px (SearchRange %d)" % (px.max(), p.SearchRange))
    assert px.max() > p.SearchRange

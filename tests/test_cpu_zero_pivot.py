"""TooN's Cholesky<N> past a zero pivot, and the IMU filter on the degenerate inputs that reach one.  Runs on the CPU.

TooN's do_compute stops at the first zero pivot and leaves the rest of the matrix as it stands; get_inverse then
back-substitutes through that partial factor, so an inverse of a singular matrix keeps finite entries in the rows and
columns after the zero pivot.  A factor that goes on past the pivot with 1/0 = inf turns them all into NaN.  lm.cuh's
ldlt_inverse<N, STOP_AT_ZERO> has both; every get_inverse site of the product runs STOP_AT_ZERO = true.

test_inverse_by_class compares both variants with the reference's own TooN::Cholesky<N> (oracle/_ref/libref_mtrack.so)
at N = 3, 6, 7 on structural zero pivots at every position, by class: the same NaN, +inf and -inf positions, and finite
entries bit for bit (not the bytes: x86's default NaN has its sign bit set).  test_est_ka_gmek_bias runs the IMU filter
(imu_filter.h) against the reference's ScaleEstimator::estKaGMEKBias on a frame without forward matches (a zero
velocity block in Wvw), on one whose edges are all vertical (a zero Vy row and column) and on the two forms of Rf the
frame loop can pass (NaN, and 1e50 I as the NaN guard leaves P_V), and on inputs that put a zero pivot in ka_problem's
Pz or prior Pp: there the reference's filter is all NaN too, so ka_problem keeps the factor without the stop.

toon_factor / zero_pivot are a NumPy restatement of do_compute; tests/test_gpu_zero_pivot.py uses them to prove that its
edge-map states reach the zero pivot they target."""
import ctypes as C

import numpy as np
import pytest


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ---- NumPy restatement of TooN's Cholesky<N> (Cholesky.h do_compute / backsub of a matrix) -------------------------------
def toon_factor(M, stop=True):
    """(factor, rank) of do_compute: L below the diagonal, D on it, L*D above it.  stop=False goes on past a zero pivot
    with 1/0 = inf (lm.cuh's STOP_AT_ZERO = false); rank is then the size."""
    a = np.array(M, np.float64)
    n = len(a)
    with np.errstate(all="ignore"):
        for col in range(n):
            inv_diag = np.float64(1)
            for row in range(col, n):
                val = a[row, col]
                for col2 in range(col):
                    val = val - a[col2, col] * a[row, col2]
                if row == col:
                    a[row, col] = val
                    if stop and val == 0:
                        return a, row
                    inv_diag = np.float64(1) / val
                else:
                    a[col, row] = val
                    a[row, col] = val * inv_diag
    return a, n


def zero_pivot(M):
    """Index of the pivot at which TooN's factor of M stops, or None when it factors every column."""
    r = toon_factor(M)[1]
    return None if r == len(M) else r


def toon_inverse(M, stop=True):
    """get_inverse = backsub(Identity) through the factor (the matrix overload: y *= 1/diag)."""
    a, _ = toon_factor(M, stop)
    n = len(a)
    inv = np.zeros((n, n))
    with np.errstate(all="ignore"):
        for c in range(n):
            y = np.zeros(n)
            for i in range(n):
                val = np.float64(i == c)
                for j in range(i):
                    val = val - a[i, j] * y[j]
                y[i] = val
            for i in range(n):
                y[i] = y[i] * (np.float64(1) / a[i, i])
            x = np.zeros(n)
            for i in range(n - 1, -1, -1):
                val = y[i]
                for j in range(i + 1, n):
                    val = val - a[j, i] * x[j]
                x[i] = val
            inv[:, c] = x
    return inv


def class_errors(tag, ref, got, rtol=0.0, atol=0.0):
    """Differences of got from ref by class: NaN, +inf and -inf positions, then finite entries (bit for bit at
    rtol = atol = 0).  Returns a list of messages."""
    ref, got = np.asarray(ref, np.float64), np.asarray(got, np.float64)
    errs = []
    for what, f in (("NaN", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
        if not np.array_equal(f(ref), f(got)):
            errs.append("%s: %s positions differ: ref %s got %s" % (tag, what, np.argwhere(f(ref)).tolist()[:6],
                                                                   np.argwhere(f(got)).tolist()[:6]))
    fin = np.isfinite(ref) & np.isfinite(got)
    bad = fin & ~(np.abs(ref - got) <= atol + rtol * np.abs(ref)) if (rtol or atol) else fin & (ref != got)
    if bad.any():
        errs.append("%s: finite entries differ at %s: ref %s got %s" % (tag, np.argwhere(bad).tolist()[:4], ref[bad][:4],
                                                                       got[bad][:4]))
    return errs


# ---- the product's two variants, and TooN --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def libs(built):
    from oracle import refapi
    from rebvo_b200 import capi
    if not refapi.available():
        pytest.skip("compiled reference not available")
    return C.CDLL(capi.LIB_PATH), refapi


def _inverse(L, A, stop):
    A = np.ascontiguousarray(A, np.float64)
    inv = np.zeros_like(A)
    getattr(L, "rb_hostmath_ldlt%d_inverse%s" % (len(A), "_stop" if stop else ""))(_p(A), _p(inv))
    return inv


def _spd(rng, n):
    A = rng.normal(size=(n + 4, n))
    return A.T @ A + np.eye(n)


def _case(kind, n, pos, seed):
    """(matrix, index of the zero pivot TooN stops at) of one structural zero pivot"""
    rng = np.random.default_rng(seed)
    if kind == "zero_row_col":                  # row and column pos exactly zero
        A = _spd(rng, n)
        A[pos, :] = 0
        A[:, pos] = 0
        return A, pos
    if kind == "zero_block":                     # [[0, 0], [0, B]]: the leading pos + 1 rows and columns zero
        A = np.zeros((n, n))
        A[pos + 1:, pos + 1:] = _spd(rng, n - pos - 1)
        return A, 0
    if kind == "jtj_one_col":                    # J^T J of a Jacobian with column pos exactly zero
        J = rng.normal(size=(40, n)) * rng.uniform(0.1, 100, n)
        J[:, pos] = 0
        return J.T @ J, pos
    if kind == "jtj_two_cols":                   # ... with columns pos and pos + 2 (mod n) exactly zero
        J = rng.normal(size=(40, n)) * rng.uniform(0.1, 100, n)
        J[:, [pos, (pos + 2) % n]] = 0
        return J.T @ J, min(pos, (pos + 2) % n)
    if kind == "ldl_zero_d":                     # L D L^T with D[pos] = 0 and a full row pos: exact in float64
        Lm = np.tril(rng.integers(-2, 3, size=(n, n)), -1) + np.eye(n)
        d = rng.integers(1, 5, size=n).astype(np.float64)
        d[pos] = 0
        return (Lm * d) @ Lm.T, pos
    if kind == "all_zero":
        return np.zeros((n, n)), 0
    raise ValueError(kind)


CASES = [(k, n, p) for n in (3, 6, 7) for k in ("zero_row_col", "jtj_one_col", "jtj_two_cols", "ldl_zero_d")
         for p in range(n)] + [("zero_block", n, p) for n in (3, 6, 7) for p in range(n - 1)] + \
        [("all_zero", n, 0) for n in (3, 6, 7)]


@pytest.mark.parametrize("kind,n,pos", CASES)
def test_inverse_by_class(libs, kind, n, pos):
    """STOP_AT_ZERO = true is TooN's get_inverse by class, finite entries bit for bit, and so is the NumPy restatement;
    the case reaches the zero pivot it targets."""
    L, refapi = libs
    A, want = _case(kind, n, pos, 100 * n + 10 * pos + len(kind))
    A = np.ascontiguousarray(A)
    assert zero_pivot(A) == want, (kind, n, pos, zero_pivot(A))
    with np.errstate(all="ignore"):
        _, toon = refapi.cholesky(A, np.ones(n))
    errs = class_errors("stop", toon, _inverse(L, A, True)) + class_errors("numpy", toon, toon_inverse(A))
    errs += class_errors("numpy no-stop", _inverse(L, A, False), toon_inverse(A, stop=False))
    assert not errs, "\n".join(errs)


def test_no_stop_variant_differs_from_toon(libs):
    """What the factor without the stop gets wrong, recorded: where TooN's inverse keeps finite entries after a zero pivot,
    the no-stop factor's are NaN.  The IMU flow's W_Xgv after BiasCorrect on a frame without forward matches is the
    zero_block case at N = 6 (a zero velocity block and the gyro prior on the rotation block), and a JtJ whose Vy
    column is zero (every keyline edge vertical) the jtj_one_col case at position 1."""
    L, refapi = libs
    table = {}
    for kind, n, pos in CASES:
        A, _ = _case(kind, n, pos, 100 * n + 10 * pos + len(kind))
        A = np.ascontiguousarray(A)
        with np.errstate(all="ignore"):
            _, toon = refapi.cholesky(A, np.ones(n))
        table[kind, n, pos] = (int(np.isfinite(toon).sum()), not class_errors("", toon, _inverse(L, A, False)))
    print("\n".join("%s N=%d pivot %d: TooN finite entries %d, no-stop agrees %s" % (k + v) for k, v in table.items()))
    imu = table["zero_block", 6, 2]
    assert imu[0] == 18 and not imu[1], imu                  # the rotation rows are finite, the no-stop factor's are not
    vy = table["jtj_one_col", 6, 1]
    assert vy[0] == 24 and not vy[1], vy                     # rows 2..5 finite
    assert not table["all_zero", 6, 0][1]                    # even JtJ = 0: TooN's (5, 5) is +inf, not NaN
    # wherever TooN keeps a finite entry after the zero pivot, the no-stop factor disagrees with it
    keeps = [k for k, v in table.items() if v[0] > 0]
    assert all(not table[k][1] for k in keeps), [k for k in keeps if table[k][1]]


# ---- the IMU filter: estKaGMEKBias ------------------------------------------------------------------------------------
G = 9.8


def _ka_inputs(rng, wvw_kind, rf_kind):
    X = np.array([np.pi / 4, 0.1, G, -0.2, 0, 0, 0.0])
    P = np.diag([1.2e-3 ** 2, 100, 100, 100, 1e-13, 1e-13, 1e-13]).astype(np.float64)
    a_v = rng.normal(0, 0.5, 3)
    a_s = 1.3 * a_v - X[1:4] + rng.normal(0, 2e-3, 3)
    from oracle import refapi
    Rot = np.ascontiguousarray(refapi.so3_exp(rng.normal(0, 5e-3, 3)))
    A = rng.normal(0, 1, (6, 6))
    Wvw = (A @ A.T + np.eye(6) * 50) * 1e4
    Rf = np.linalg.inv(Wvw)[:3, :3] / 0.05 ** 4   # a velocity measurement as informative as test_cpu_imu_filter.py's
    if wvw_kind == "vel_block_zero":   # W_Xgv after BiasCorrect on a frame without forward matches
        Wvw[:3, :] = 0
        Wvw[:, :3] = 0
    elif wvw_kind == "vy_zero":        # every edge vertical: the Vy row and column of JtJ exactly zero
        Wvw[1, :] = 0
        Wvw[:, 1] = 0
    with np.errstate(all="ignore"):
        Rx = refapi.cholesky(Wvw, np.ones(6))[1]   # what the frame loop derives from W_Xgv: R_Xgv, its P_W and P_V
    Qrot = np.ascontiguousarray(Rx[3:, 3:]) if np.isfinite(Rx[3:, 3:]).all() else np.eye(3) * 1e-6
    if rf_kind == "nan":
        Rf = Rx[:3, :3] / 0.05 ** 4 if wvw_kind != "full" else np.full((3, 3), np.nan)
        assert np.isnan(Rf).any()
    elif rf_kind == "1e50":
        Rf = np.eye(3) * 1e50
    xvw = rng.normal(0, 1e-3, 6)
    d = dict(X=X, P=P, a_v=a_v, a_s=a_s, Rot=Rot, Wvw=np.ascontiguousarray(Wvw), Qrot=Qrot, Rf=np.ascontiguousarray(Rf),
             xvw=xvw, Qg=np.eye(3) * 2e-3 ** 2, Qbias=np.eye(3) * 1e-14, Rs=np.eye(3) * 2e-3 ** 2, QKp=5e-6)
    if rf_kind.startswith("pz"):       # ka_problem's Pz = sin^2 Rf + cos^2 Rs with a zero row and column k
        k = int(rf_kind[2:])
        for m in ("Rf", "Rs"):
            d[m][k, :] = 0
            d[m][:, k] = 0
    elif rf_kind.startswith("pp"):     # ka_problem's prior Pp = F P F^T + Q with a zero row and column k
        k = int(rf_kind[2:])
        d["Rot"] = np.eye(3)           # (F's gravity block is Rot^T: the identity keeps the zero row where it is)
        P[k, :] = 0
        P[:, k] = 0
        if k == 0:
            d["QKp"] = 0.0
        elif k < 4:
            d["Qrot"] = np.zeros((3, 3))
            d["Qg"][k - 1, :] = 0
            d["Qg"][:, k - 1] = 0
        else:
            d["Qbias"][k - 4, :] = 0
            d["Qbias"][:, k - 4] = 0
    return d


def _ka_prior(d):
    """est_ka_gmek_bias's Pp = F P F^T + Q, as ka_problem inverts it"""
    F = np.eye(7)
    F[1:4, 1:4] = d["Rot"].T
    g = d["X"][1:4]
    Gx = np.array([[0, g[2], -g[1]], [-g[2], 0, g[0]], [g[1], -g[0], 0]])
    Q = np.zeros((7, 7))
    Q[0, 0] = d["QKp"] / (1 + np.tan(d["X"][0]) ** 2)
    Q[1:4, 1:4] = Gx.T @ d["Qrot"] @ Gx + d["Qg"]
    Q[4:, 4:] = d["Qbias"]
    return F @ d["P"] @ F.T + Q


def _ka_run(fn, d):
    X, P, xv = d["X"].copy(), d["P"].copy(), d["xvw"].copy()
    ge, be = np.zeros(3), np.zeros(3)
    m = {k: np.ascontiguousarray(d[k]) for k in ("Rot", "Qg", "Qrot", "Qbias", "Rs", "Rf", "Wvw")}
    fn.restype = C.c_double
    with np.errstate(all="ignore"):
        k = fn(_p(d["a_s"]), _p(d["a_v"]), C.c_double(1.0), _p(m["Rot"]), _p(X), _p(P), _p(m["Qg"]), _p(m["Qrot"]),
               _p(m["Qbias"]), C.c_double(d["QKp"]), C.c_double(1e10), _p(m["Rs"]), _p(m["Rf"]), _p(ge), _p(be), _p(m["Wvw"]),
               _p(xv), C.c_double(G))
    return dict(K=np.array([k]), X=X, P=P, g_est=ge, b_est=be, Xvw=xv)


# test_cpu_imu_filter.py's bars on finite values: (rtol, atol); P's atol is scaled per entry
KA_BARS = dict(K=(1e-8, 0.0), X=(1e-8, 1e-10), P=(1e-6, 1e-18), g_est=(1e-9, 0.0), b_est=(1e-7, 1e-12), Xvw=(1e-8, 1e-12))
KA_CASES = {"vel_block_zero": ("vel_block_zero", "finite"), "vy_zero": ("vy_zero", "finite"),
            "vel_block_zero_rf_from_w": ("vel_block_zero", "nan"), "rf_nan": ("full", "nan"), "rf_1e50": ("full", "1e50")}
# ka_problem's two inverses at a zero pivot: whatever TooN's inverse keeps finite, its non-finite row multiplies every
# column of the 11 x 11 W products (NaN * 0 = NaN), so JtJ, and then K, X, P and Xvw, are NaN in the reference as well
KA_CASES.update({"pz_zero_%d" % k: ("full", "pz%d" % k) for k in range(3)})
KA_CASES.update({"pp_zero_%d" % k: ("full", "pp%d" % k) for k in range(7)})


@pytest.mark.parametrize("case", list(KA_CASES))
def test_est_ka_gmek_bias(libs, case):
    """imu_filter.h's est_ka_gmek_bias against the reference's ScaleEstimator::estKaGMEKBias, three filter steps, by
    class: K, X, P, g_est, b_est and the bias-corrected Xvw."""
    L, refapi = libs
    R = refapi.lib()
    rng = np.random.default_rng(sum(map(ord, case)))
    wk, rk = KA_CASES[case]
    d = _ka_inputs(rng, wk, rk)
    if wk != "full":   # the case reaches its zero pivot: Wb + Wvw keeps the zero rows of Wvw (Wb is the bias block)
        assert zero_pivot(d["Wvw"]) == {"vel_block_zero": 0, "vy_zero": 1}[wk]
    if rk.startswith("pz"):
        Pz = 0.5 * d["Rf"] + 0.5 * d["Rs"]   # (any angle: both have the zero row)
        assert zero_pivot(Pz) == int(rk[2:])
    if rk.startswith("pp"):
        assert zero_pivot(_ka_prior(d)) == int(rk[2:])
    errs = []
    for step in range(3):
        a, b = _ka_run(L.rb_hostmath_est_ka_gmek_bias, d), _ka_run(R.ref_est_ka_gmek_bias, d)
        for k, (rtol, atol) in KA_BARS.items():
            if k == "P":   # a covariance: each entry against its own scale sqrt(P_ii P_jj)
                dg = np.sqrt(np.abs(np.diag(b["P"])))
                with np.errstate(invalid="ignore"):
                    atol = np.nan_to_num(np.outer(dg, dg) * rtol, nan=0.0, posinf=0.0)
            errs += class_errors("step %d %s" % (step, k), b[k], a[k], rtol, atol)
        fin = {k: int(np.isfinite(b[k]).sum()) for k in b}
        print("%s step %d: finite entries of the reference's %s" % (case, step, fin))
        d.update(X=b["X"], P=b["P"], xvw=b["Xvw"])
        if rk[:2] in ("pz", "pp"):
            assert all(np.isnan(b[k]).all() for k in ("X", "P", "Xvw")), fin
            break
        if rk == "finite":
            # the reference keeps the rotation part of Xvw finite (TooN's stop): the case shows that difference
            assert np.isfinite(b["Xvw"][3:]).all(), b["Xvw"]
            d["xvw"] = np.where(np.isfinite(b["Xvw"]), b["Xvw"], 0.0)
    assert not errs, "\n".join(errs)


# ---- BiasCorrect ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["vel_block_zero", "vy_zero"])
def test_bias_correct(libs, kind):
    """rb_bias_correct against the reference's edge_tracker::BiasCorrect on W_X of a frame without forward matches (a zero
    velocity block) and of one whose edges are all vertical (a zero Vy row and column), by class: X, W_X, the gyro bias
    and its information.  Its Cholesky<6>(Wxb).get_inverse() meets the zero pivot."""
    from rebvo_b200 import capi
    L, refapi = libs
    rng = np.random.default_rng(len(kind))
    A = rng.normal(size=(6, 6))
    Wx = (A @ A.T + np.eye(6) * 50) * 1e4
    if kind == "vel_block_zero":
        Wx[:3, :] = 0
        Wx[:, :3] = 0
    else:
        Wx[1, :] = 0
        Wx[:, 1] = 0
    X, Gb = rng.normal(0, 1e-3, 6), rng.normal(0, 1e-4, 3)
    Wb, Rg, Rb = np.eye(3) * 1e6, np.eye(3) * 1e-6, np.eye(3) * 1e-8
    Wxb = Wx.copy()
    Wxb[3:, 3:] += np.linalg.inv(Rg)   # (the gyro prior only adds to the rotation block: the zero rows stay)
    assert zero_pivot(Wxb) == {"vel_block_zero": 0, "vy_zero": 1}[kind]
    ref = refapi.bias_correct(X, Wx, Gb, Wb, Rg, Rb)
    got = [np.ascontiguousarray(np.array(v, np.float64)) for v in (X, Wx, Gb, Wb)]
    f = capi.lib().rb_bias_correct
    with np.errstate(all="ignore"):
        f(*[_p(a) for a in got], _p(np.ascontiguousarray(Rg)), _p(np.ascontiguousarray(Rb)))
    assert np.isfinite(ref[0][3:]).all(), ref[0]   # TooN keeps the rotation part of X finite
    errs = []
    for name, a, b in zip(("X", "W_X", "Gb", "Wb"), ref, got):
        errs += class_errors(name, a, b, 1e-9, 1e-12)
    assert not errs, "\n".join(errs)

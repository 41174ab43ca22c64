// lm.cuh -- small dense float64 algebra used by the device-resident Levenberg-Marquardt driver and the
// per-frame scalar logic.  __host__ __device__ so that the same code is unit-tested on the CPU
// (tests/test_host_math.py through librebvo_b200's rb_hostmath_* exports) and runs in 1-thread kernels.
//
// Restated from the published algorithms of TooN 2.2 (third-party dependency of the reference, vendored
// there as TooN-2.2.zip): SO3::exp / ln / coerce (so3.h), Cholesky<6> = LDL^T without square roots
// (Cholesky.h), SVD<>::backsub / get_pinv with condition number 1e9 (SVD.h; LAPACK dgesvd_ replaced by
// a cyclic Jacobi eigen-decomposition, valid because every matrix decomposed on this path is symmetric).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define RB_HD __host__ __device__ __forceinline__
#else
#define RB_HD inline
#endif

// ---- SO(3) --------------------------------------------------------------------------------------------
// TooN::SO3<>::exp (so3.h:254-285) with rodrigues_so3_exp (so3.h:219-251); R row-major
RB_HD void so3_exp(const double w[3], double R[9]) {
    const double one_6th = 1.0 / 6.0, one_20th = 1.0 / 20.0;
    double theta_sq = 0;  // w*w : result=0; result+=w[i]*w[i]
    for (int i = 0; i < 3; i++) theta_sq += w[i] * w[i];
    const double theta = sqrt(theta_sq);
    double A, B;
    if (theta_sq < 1e-8) {
        A = 1.0 - one_6th * theta_sq;
        B = 0.5;
    } else if (theta_sq < 1e-6) {
        B = 0.5 - 0.25 * one_6th * theta_sq;
        A = 1.0 - theta_sq * one_6th * (1.0 - one_20th * theta_sq);
    } else {
        const double inv_theta = 1.0 / theta;
        double sn, cs;
        sincos(theta, &sn, &cs);   // one argument reduction for both
        A = sn * inv_theta;
        B = (1 - cs) * (inv_theta * inv_theta);
    }
    const double wx2 = w[0] * w[0], wy2 = w[1] * w[1], wz2 = w[2] * w[2];
    R[0] = 1.0 - B * (wy2 + wz2);
    R[4] = 1.0 - B * (wx2 + wz2);
    R[8] = 1.0 - B * (wx2 + wy2);
    double a = A * w[2], b = B * (w[0] * w[1]);
    R[1] = b - a;
    R[3] = b + a;
    a = A * w[1];
    b = B * (w[0] * w[2]);
    R[2] = b + a;
    R[6] = b - a;
    a = A * w[0];
    b = B * (w[1] * w[2]);
    R[5] = b - a;
    R[7] = b + a;
}

RB_HD double dot3(const double *a, const double *b) {
    double r = 0;
    for (int i = 0; i < 3; i++) r += a[i] * b[i];
    return r;
}

// SO3::coerce (so3.h:110-119): Gram-Schmidt on the rows
RB_HD void so3_coerce(double M[9]) {
    double *r0 = M, *r1 = M + 3, *r2 = M + 6;
    double s = 1 / sqrt(dot3(r0, r0));
    for (int i = 0; i < 3; i++) r0[i] = r0[i] * s;
    double d = dot3(r0, r1);
    for (int i = 0; i < 3; i++) r1[i] -= r0[i] * d;
    s = 1 / sqrt(dot3(r1, r1));
    for (int i = 0; i < 3; i++) r1[i] = r1[i] * s;
    d = dot3(r0, r2);
    for (int i = 0; i < 3; i++) r2[i] -= r0[i] * d;
    d = dot3(r1, r2);
    for (int i = 0; i < 3; i++) r2[i] -= r1[i] * d;
    s = 1 / sqrt(dot3(r2, r2));
    for (int i = 0; i < 3; i++) r2[i] = r2[i] * s;
}

// SO3<>(M).ln() as the reference calls it (rebvo_second_t.cpp:567,571): coerce, then so3.h:288-334
RB_HD void so3_ln_of_matrix(const double Min[9], double out[3]) {
    double m[9];
    for (int i = 0; i < 9; i++) m[i] = Min[i];
    so3_coerce(m);
    const double cos_angle = (m[0] + m[4] + m[8] - 1.0) * 0.5;
    out[0] = (m[7] - m[5]) / 2;
    out[1] = (m[2] - m[6]) / 2;
    out[2] = (m[3] - m[1]) / 2;
    const double sin_angle_abs = sqrt(dot3(out, out));
    const double SQRT1_2 = 0.70710678118654752440;
    if (cos_angle > SQRT1_2) {
        if (sin_angle_abs > 0) {
            const double k = asin(sin_angle_abs) / sin_angle_abs;
            for (int i = 0; i < 3; i++) out[i] *= k;
        }
    } else if (cos_angle > -SQRT1_2) {
        const double k = acos(cos_angle) / sin_angle_abs;
        for (int i = 0; i < 3; i++) out[i] *= k;
    } else {
        const double angle = 3.14159265358979323846 - asin(sin_angle_abs);
        const double d0 = m[0] - cos_angle, d1 = m[4] - cos_angle, d2 = m[8] - cos_angle;
        double r2[3];
        if (d0 * d0 > d1 * d1 && d0 * d0 > d2 * d2) {
            r2[0] = d0;
            r2[1] = (m[3] + m[1]) / 2;
            r2[2] = (m[2] + m[6]) / 2;
        } else if (d1 * d1 > d2 * d2) {
            r2[0] = (m[3] + m[1]) / 2;
            r2[1] = d1;
            r2[2] = (m[7] + m[5]) / 2;
        } else {
            r2[0] = (m[2] + m[6]) / 2;
            r2[1] = (m[7] + m[5]) / 2;
            r2[2] = d2;
        }
        if (dot3(r2, out) < 0)
            for (int i = 0; i < 3; i++) r2[i] *= -1;
        const double s = 1 / sqrt(dot3(r2, r2));
        for (int i = 0; i < 3; i++) out[i] = angle * (r2[i] * s);
    }
}

// ---- 3x3 helpers (TooN operator semantics: dot products accumulate from 0 in index order) ---------------
RB_HD void mat3_mul(const double *A, const double *B, double *C) {  // C = A*B
    double t[9];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += A[r * 3 + k] * B[k * 3 + c];
            t[r * 3 + c] = s;
        }
    for (int i = 0; i < 9; i++) C[i] = t[i];
}
RB_HD void mat3_mul_bt(const double *A, const double *B, double *C) {  // C = A*B^T
    double t[9];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += A[r * 3 + k] * B[c * 3 + k];
            t[r * 3 + c] = s;
        }
    for (int i = 0; i < 9; i++) C[i] = t[i];
}
RB_HD void mat3_vec(const double *A, const double *v, double *o) {
    double t[3];
    for (int r = 0; r < 3; r++) {
        double s = 0;
        for (int k = 0; k < 3; k++) s += A[r * 3 + k] * v[k];
        t[r] = s;
    }
    for (int i = 0; i < 3; i++) o[i] = t[i];
}

// ---- pose-graph measurement (rebvo_second_t.cpp:323-334 and :371-382) ----------------------------------------
// rel = [-Rrel*V ; SO3(Rrel).ln()] and, when W_X is given, Wrel = J^T*W_X*J with J the inverse of
// J_rp_x = [[-Rj, [rel[0:3]]x], [0, -I]].  The reference inverts J_rp_x with TooN's SVD pseudo-inverse; the matrix is block
// upper triangular with orthonormal diagonal blocks, so its inverse is [[-Rj^T, -Rj^T*[t]x], [0, -I]] in closed form, which
// agrees with the pseudo-inverse to rounding.  W_X == nullptr: Wrel = 0.
RB_HD void odom_rel_pose(const double Rrel[9], const double V[3], const double Rj[9], const double *W_X, double rel[6],
                         double Wrel[36]) {
    double t[3];
    mat3_vec(Rrel, V, t);
    for (int i = 0; i < 3; i++) rel[i] = -t[i];
    so3_ln_of_matrix(Rrel, rel + 3);
    if (!W_X) {
        for (int i = 0; i < 36; i++) Wrel[i] = 0;
        return;
    }
    const double cx[9] = {0, -rel[2], rel[1], rel[2], 0, -rel[0], -rel[1], rel[0], 0};   // util::crossMatrix
    double RtC[9];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += Rj[k * 3 + r] * cx[k * 3 + c];
            RtC[r * 3 + c] = s;
        }
    double J[36];
    for (int i = 0; i < 36; i++) J[i] = 0;
    for (int r = 0; r < 3; r++) {
        for (int c = 0; c < 3; c++) {
            J[r * 6 + c] = -Rj[c * 3 + r];
            J[r * 6 + 3 + c] = -RtC[r * 3 + c];
        }
        J[(3 + r) * 6 + 3 + r] = -1;
    }
    // (one thread runs this beside a wide kernel: rolled loops keep J and T out of that kernel's register allocation)
    double T[36];   // J^T * W_X (TooN evaluates the product left to right)
#pragma unroll 1
    for (int r = 0; r < 6; r++)
#pragma unroll 1
        for (int c = 0; c < 6; c++) {
            double s = 0;
            for (int k = 0; k < 6; k++) s += J[k * 6 + r] * W_X[k * 6 + c];
            T[r * 6 + c] = s;
        }
#pragma unroll 1
    for (int r = 0; r < 6; r++)
#pragma unroll 1
        for (int c = 0; c < 6; c++) {
            double s = 0;
            for (int k = 0; k < 6; k++) s += T[r * 6 + k] * J[k * 6 + c];
            Wrel[r * 6 + c] = s;
        }
}

// ---- Cholesky<6> (Cholesky.h do_compute / backsub / get_inverse): L D L^T, no square roots --------------
struct Chol6 {
    double c[36];
    int rank;
};
RB_HD void chol6_compute(const double *M, Chol6 *ch) {
    for (int i = 0; i < 36; i++) ch->c[i] = M[i];
    double *a = ch->c;
    const int n = 6;
#pragma unroll
    for (int col = 0; col < n; col++) {
        double inv_diag = 1;
#pragma unroll
        for (int row = col; row < n; row++) {
            double val = a[row * 6 + col];
#pragma unroll
            for (int col2 = 0; col2 < col; col2++) val -= a[col2 * 6 + col] * a[row * 6 + col2];
            if (row == col) {
                a[row * 6 + col] = val;
                if (val == 0) {
                    ch->rank = row;
                    return;
                }
                inv_diag = 1 / val;
            } else {
                a[col * 6 + row] = val;
                a[row * 6 + col] = val * inv_diag;
            }
        }
    }
    ch->rank = n;
}
RB_HD void chol6_backsub(const Chol6 *ch, const double *v, double *x) {
    const double *a = ch->c;
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        double val = v[i];
#pragma unroll
        for (int j = 0; j < i; j++) val -= a[i * 6 + j] * y[j];
        y[i] = val;
    }
#pragma unroll
    for (int i = 0; i < 6; i++) y[i] /= a[i * 6 + i];
#pragma unroll
    for (int i = 5; i >= 0; i--) {
        double val = y[i];
#pragma unroll
        for (int j = i + 1; j < 6; j++) val -= a[j * 6 + i] * x[j];
        x[i] = val;
    }
}
// get_inverse = backsub(Identity) with the matrix overload (y[i]*=(1/diag))
RB_HD void chol6_inverse(const Chol6 *ch, double *inv) {
    const double *a = ch->c;
    double y[36];
    for (int i = 0; i < 6; i++) {
        double val[6];
        for (int c = 0; c < 6; c++) val[c] = (i == c) ? 1.0 : 0.0;
        for (int j = 0; j < i; j++)
            for (int c = 0; c < 6; c++) val[c] -= a[i * 6 + j] * y[j * 6 + c];
        for (int c = 0; c < 6; c++) y[i * 6 + c] = val[c];
    }
    for (int i = 0; i < 6; i++) {
        const double s = 1 / a[i * 6 + i];
        for (int c = 0; c < 6; c++) y[i * 6 + c] *= s;
    }
    for (int i = 5; i >= 0; i--) {
        double val[6];
        for (int c = 0; c < 6; c++) val[c] = y[i * 6 + c];
        for (int j = i + 1; j < 6; j++)
            for (int c = 0; c < 6; c++) val[c] -= a[j * 6 + i] * inv[j * 6 + c];
        for (int c = 0; c < 6; c++) inv[i * 6 + c] = val[c];
    }
}

// ---- symmetric eigen-decomposition (cyclic Jacobi) standing in for SVD<> of a symmetric matrix ----------
// A (n x n, n <= 6, symmetric) = Q diag(lam) Q^T ; Q row-major, columns are eigenvectors
RB_HD void sym_jacobi(const double *Ain, int n, double *lam, double *Q) {
    double A[36];
    for (int i = 0; i < n * n; i++) A[i] = Ain[i];
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) Q[i * n + j] = (i == j) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; sweep++) {
        double off = 0, diag = 0;
        for (int i = 0; i < n; i++) {
            diag += A[i * n + i] * A[i * n + i];
            for (int j = i + 1; j < n; j++) off += A[i * n + j] * A[i * n + j];
        }
        if (off <= 1e-34 * diag || off == 0) break;
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) {
                const double apq = A[p * n + q];
                if (apq == 0) continue;
                const double app = A[p * n + p], aqq = A[q * n + q];
                const double tau = (aqq - app) / (2 * apq);
                const double t = (tau >= 0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1 + tau * tau));
                const double c = 1 / sqrt(1 + t * t), s = t * c;
                for (int k = 0; k < n; k++) {  // A <- A J
                    const double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s * akq;
                    A[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; k++) {  // A <- J^T A
                    const double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s * aqk;
                    A[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; k++) {
                    const double qkp = Q[k * n + p], qkq = Q[k * n + q];
                    Q[k * n + p] = c * qkp - s * qkq;
                    Q[k * n + q] = s * qkp + c * qkq;
                }
            }
    }
    for (int i = 0; i < n; i++) lam[i] = A[i * n + i];
}

// SVD<>(A).backsub(b) for symmetric A (SVD.h backsub + get_inv_diag, condition_no = 1e9):
// x = V diag(1/s_i or 0) U^T b with s_i = |lam_i|, u_i = sign(lam_i) q_i, v_i = q_i
RB_HD void sym_svd_backsub(const double *A, int n, const double *b, double *x) {
    double lam[6], Q[36];
    sym_jacobi(A, n, lam, Q);
    double smax = 0;
    for (int i = 0; i < n; i++) smax = fmax(smax, fabs(lam[i]));
    for (int i = 0; i < n; i++) x[i] = 0;
    for (int k = 0; k < n; k++) {
        const double s = fabs(lam[k]);
        if (s * 1e9 <= smax) continue;  // get_inv_diag: inv_diag = 0
        double utb = 0;
        for (int i = 0; i < n; i++) utb += Q[i * n + k] * b[i];
        const double coef = utb / lam[k];  // sign(lam) * (1/s)
        for (int i = 0; i < n; i++) x[i] += Q[i * n + k] * coef;
    }
}

// Solve (JtJ + u I) h = rhs the way the init iterations do (SVD<> svdApI(ApI); h = backsub(-JtF),
// global_tracker.cpp:659-661).  ApI is symmetric positive definite here (u = 1e-3 * max(JtJ) bounds the
// condition number far below SVD.h's 1e9 cut), so the pseudo-inverse equals the inverse and the cheap
// LDL^T solve returns the same vector up to rounding; the Jacobi path is kept for rank-deficient input.
RB_HD void solve_sym6_like_svd(const double *ApI, const double *rhs, double *h) {
    Chol6 ch;
    chol6_compute(ApI, &ch);
    bool ok = ch.rank == 6;
    double dmax = 0, dmin = 1e300;
    for (int i = 0; i < 6 && ok; i++) {
        const double d = ch.c[i * 6 + i];
        if (!(d > 0)) ok = false;
        dmax = fmax(dmax, d);
        dmin = fmin(dmin, d);
    }
    if (ok && dmin * 1e7 > dmax) {
        chol6_backsub(&ch, rhs, h);
    } else {
        sym_svd_backsub(ApI, 6, rhs, h);
    }
}

// TooN::determinant of a 3x3 (TooN/determinant.h:91-146, determinant_gaussian_elimination): partial pivoting, running
// product of the pivots -- not the cofactor expansion, and the last bits differ
RB_HD double det3_toon(const double *Ain) {
    double A[3][3];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) A[i][j] = Ain[i * 3 + j];
    double det = 1;
    for (int i = 0; i < 3; i++) {
        int argmax = i;
        double maxval = fabs(A[i][i]);
        for (int ii = i + 1; ii < 3; ii++) {
            const double v = fabs(A[ii][i]);
            if (v > maxval) {
                maxval = v;
                argmax = ii;
            }
        }
        const double pivot = A[argmax][i];
        if (argmax != i) {
            det *= -1;
            for (int j = i; j < 3; j++) {
                const double t = A[i][j];
                A[i][j] = A[argmax][j];
                A[argmax][j] = t;
            }
        }
        det *= A[i][i];
        if (det == 0) return 0;
        for (int u = i + 1; u < 3; u++) {
            const double factor = A[u][i] / pivot;
            for (int j = i + 1; j < 3; j++) A[u][j] = A[u][j] - factor * A[i][j];
        }
    }
    return det;
}
// util::Matrix3x3Inv (include/UtilLib/toon_util.h:32-41): cofactors / TooN::determinant
RB_HD void mat3_inv(const double *A, double *B) {
    double t[9];
    t[0] = A[8] * A[4] - A[7] * A[5];
    t[1] = -(A[8] * A[1] - A[7] * A[2]);
    t[2] = A[5] * A[1] - A[4] * A[2];
    t[3] = -(A[8] * A[3] - A[6] * A[5]);
    t[4] = A[8] * A[0] - A[6] * A[2];
    t[5] = -(A[5] * A[0] - A[3] * A[2]);
    t[6] = A[7] * A[3] - A[6] * A[4];
    t[7] = -(A[7] * A[0] - A[6] * A[1]);
    t[8] = A[4] * A[0] - A[3] * A[1];
    const double det = det3_toon(A);
    for (int i = 0; i < 9; i++) B[i] = t[i] / det;
}

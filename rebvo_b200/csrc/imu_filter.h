// imu_filter.h -- host-side filter chain of the IMU mode (config 3), plain C++ on row-major double arrays:
//   ImuGrabber::SeachByTimeStamp / GrabAndIntegrate   src/UtilLib/imugrabber.cpp:171-253   (inter-frame gyro integration)
//   ScaleEstimator::EstAcelLsq4 / MeanAcel4           src/mtracklib/scaleestimator.cpp:37-110
//   ScaleEstimator::estKaGMEKBias + Problem_KaGMEKBias + FunT_KaGMEKBias   scaleestimator.cpp:117-318
//   Minimizer<7,11,..>::GaussNewton (problem form)     include/UtilLib/minimizer.h:86-116
// This is small serial algebra (7 x 7, 11 x 11) once per frame; it stays on the host like in the reference and feeds
// the device stages through the stage-level entry points.  The reference's function-static histories (EstAcelLsq4's
// V..V3 / T / Dt, MeanAcel4's A..A2) live in ImuFilterHist, one per pipeline.  TooN's LAPACK-backed SVD<7> of the
// Gauss-Newton step is replaced by a Jacobi pseudo-inverse (sym_svd_backsub<7>, lm.cuh): the matrix is symmetric.  Its
// Cholesky<3/6/7>::get_inverse calls are lm.cuh's ldlt_inverse; the bias-corrected Xvw's stops at a zero pivot as TooN's
// does (lm.cuh says why the others need not).
// Agreement with the reference: rounding level (tests/test_cpu_imu_filter.py, rel 1e-9 on the filter state).
#pragma once
#include <math.h>
#include <string.h>

#include "lm.cuh"

namespace rbimu {

// ---- tiny dense helpers (row-major) -------------------------------------------------------------------------------------
inline void matmul(const double *A, const double *B, double *C, int n, int k, int m) {   // C[n x m] = A[n x k] * B[k x m]
    for (int i = 0; i < n; i++)
        for (int j = 0; j < m; j++) {
            double s = 0;
            for (int q = 0; q < k; q++) s += A[i * k + q] * B[q * m + j];
            C[i * m + j] = s;
        }
}
inline void transpose(const double *A, double *T, int n, int m) {   // T[m x n] = A[n x m]^T
    for (int i = 0; i < n; i++)
        for (int j = 0; j < m; j++) T[j * n + i] = A[i * m + j];
}
inline void matvec(const double *A, const double *x, double *y, int n, int m) {
    for (int i = 0; i < n; i++) {
        double s = 0;
        for (int j = 0; j < m; j++) s += A[i * m + j] * x[j];
        y[i] = s;
    }
}
inline double dot(const double *a, const double *b, int n) {
    double s = 0;
    for (int i = 0; i < n; i++) s += a[i] * b[i];
    return s;
}
// TooN::SO3<>(a, b): the rotation that takes the direction of a onto the direction of b (so3.h:118-134)
inline void so3_from_two(const double *a, const double *b, double *R) {
    double n[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};   // n = a ^ b
    const double nn = dot(n, n, 3);
    if (nn == 0) {
        for (int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
        return;
    }
    const double s = 1 / sqrt(nn);
    for (int i = 0; i < 3; i++) n[i] *= s;
    double Ra[9], Rb[9];   // R1 rows: a_hat, n, n ^ a_hat ; M rows: b_hat, n, n ^ b_hat ; result = M^T * R1
    const double sa = 1 / sqrt(dot(a, a, 3)), sb = 1 / sqrt(dot(b, b, 3));
    for (int i = 0; i < 3; i++) {
        Ra[i] = a[i] * sa;
        Rb[i] = b[i] * sb;
        Ra[3 + i] = n[i];
        Rb[3 + i] = n[i];
    }
    Ra[6] = n[1] * Ra[2] - n[2] * Ra[1];
    Ra[7] = n[2] * Ra[0] - n[0] * Ra[2];
    Ra[8] = n[0] * Ra[1] - n[1] * Ra[0];
    Rb[6] = n[1] * Rb[2] - n[2] * Rb[1];
    Rb[7] = n[2] * Rb[0] - n[0] * Rb[2];
    Rb[8] = n[0] * Rb[1] - n[1] * Rb[0];
    double RbT[9];
    transpose(Rb, RbT, 3, 3);
    matmul(RbT, Ra, R, 3, 3, 3);
}

// ---- ImuGrabber (dataset mode, ImuMode=2, and live mode, ImuMode=1) ---------------------------------------------------------
struct ImuSample {
    double t, giro[3], acel[3];
};
struct ImuIntegral {   // IntegratedImuData (include/UtilLib/imugrabber.h:56-67)
    int n;
    double dt, Rot[9], giro[3], acel[3], dgiro[3], cacel[3];
};
// The circular list of ImuGrabber.  Both forms have one slot more than they can hold and share search / grab; they differ
// only in who owns the samples and where writing starts:
//   dataset  ImuGrabber(const std::vector<ImuData>&) (imugrabber.cpp:47-68): the caller's count samples, already written,
//            tsample = their mean spacing
//   live     ImuGrabber(list_size, tsamp) (imugrabber.cpp:34-40): list_size + 1 slots of the caller's, empty, filled by push
//            (PushData); tsample = the configured SampleTime
struct ImuBuffer {
    const ImuSample *s;
    ImuSample *ring;   // live form: the writable slots (== s); nullptr in the dataset form
    int n, size, write_inx, read_inx;
    double tsample, Rc2i[9], Tc2i[3];
    void init(const ImuSample *samples, int count, const double *R, const double *T) {
        s = samples;
        ring = nullptr;
        n = count;
        size = count + 1;
        write_inx = count % size;
        read_inx = size - 1;
        tsample = count > 1 ? (samples[count - 1].t - samples[0].t) / (count - 1) : 0;
        set_se3(R, T);
    }
    void init_live(ImuSample *slots, int list_size, double tsamp, const double *R, const double *T) {
        s = ring = slots;
        n = 0;
        size = list_size + 1;
        write_inx = 0;
        read_inx = size - 1;
        tsample = tsamp;
        set_se3(R, T);
    }
    void set_se3(const double *R, const double *T) {
        for (int i = 0; i < 9; i++) Rc2i[i] = R ? R[i] : (i % 4 == 0 ? 1.0 : 0.0);
        for (int i = 0; i < 3; i++) Tc2i[i] = T ? T[i] : 0.0;
    }
    // slots PushData can still fill before it meets read_inx (the slot of the last sample grabbed stays taken)
    int free_slots() const { return (read_inx - write_inx + size) % size; }
    // PushData (imugrabber.cpp:258-269) of count samples: all of them, or none when they do not fit (the reference stores
    // the samples that fit and throws overflow_error at the first one that does not)
    bool push(const ImuSample *in, int count) {
        if (!ring || count > free_slots()) return false;
        for (int i = 0; i < count; i++) {
            ring[write_inx] = in[i];
            write_inx = (write_inx + 1) % size;
        }
        n += count;
        return true;
    }
    // SeachByTimeStamp (imugrabber.cpp:171-210): [begin, end) of the samples with tstart < t <= tend
    bool search(double tstart, double tend, int *begin, int *end) const {
        int inx = read_inx;
        do {
            inx = (inx + 1) % size;
            if (inx == write_inx) return false;
        } while (s[inx].t <= tstart);
        const int b = inx;
        do {
            inx = (inx + 1) % size;
            if (inx == write_inx) return false;
        } while (s[inx].t < tend);
        if (s[inx].t - tend < 1e-12) inx = (inx + 1) % size;
        *begin = b;
        *end = inx;
        return true;
    }
    // the read position grab(tstart, tend) leaves, without the integration; false (and no change) where grab finds no sample
    bool release(double tstart, double tend) {
        int b = 0, e = 0;
        if (!search(tstart, tend, &b, &e)) return false;
        read_inx = (e - 1 + size) % size;
        return true;
    }
    // GrabAndIntegrate (imugrabber.cpp:217-253)
    ImuIntegral grab(double tstart, double tend) {
        ImuIntegral d;
        memset(&d, 0, sizeof(d));
        d.Rot[0] = d.Rot[4] = d.Rot[8] = 1;
        int b = 0, e = 0;
        if (!search(tstart, tend, &b, &e)) return d;
        double RT[9], comp_dummy[3];
        (void)comp_dummy;
        transpose(Rc2i, RT, 3, 3);
        for (int i = b; i != e; i = (i + 1) % size) {
            double g[3], a[3], w[3], E[9], R2[9];
            matvec(RT, s[i].giro, g, 3, 3);
            matvec(RT, s[i].acel, a, 3, 3);
            for (int k = 0; k < 3; k++) {
                d.giro[k] += g[k];
                d.acel[k] += a[k];
                w[k] = g[k] * tsample;
            }
            so3_exp(w, E);
            matmul(d.Rot, E, R2, 3, 3, 3);
            memcpy(d.Rot, R2, sizeof(R2));
            d.n++;
        }
        d.dt = d.n * tsample;
        if (d.n > 1) {
            for (int k = 0; k < 3; k++) {
                d.giro[k] /= d.n;
                d.acel[k] /= d.n;
            }
            const int last = (e - 1 + size) % size;
            double dg[3] = {s[last].giro[0] - s[b].giro[0], s[last].giro[1] - s[b].giro[1], s[last].giro[2] - s[b].giro[2]};
            matvec(RT, dg, d.dgiro, 3, 3);
            for (int k = 0; k < 3; k++) d.dgiro[k] /= d.dt;
        }
        double tn[3], mt[3];
        matvec(RT, Tc2i, tn, 3, 3);
        for (int k = 0; k < 3; k++) mt[k] = -tn[k];
        // cacel = acel + (dgiro ^ (-(R^T T)))
        d.cacel[0] = d.acel[0] + (d.dgiro[1] * mt[2] - d.dgiro[2] * mt[1]);
        d.cacel[1] = d.acel[1] + (d.dgiro[2] * mt[0] - d.dgiro[0] * mt[2]);
        d.cacel[2] = d.acel[2] + (d.dgiro[0] * mt[1] - d.dgiro[1] * mt[0]);
        read_inx = (e - 1 + size) % size;
        return d;
    }
};

// ---- ScaleEstimator ---------------------------------------------------------------------------------------------------------
struct ImuFilterHist {
    double V[3], V0[3], V1[3], V2[3], V3[3], T[5], Dt[4];   // EstAcelLsq4's statics
    double A[3], A0[3], A1[3], A2[3];                         // MeanAcel4's statics
};
inline void rt_vec(const double *R, const double *v, double *o) {   // o = R^T * v
    for (int i = 0; i < 3; i++) o[i] = R[0 * 3 + i] * v[0] + R[1 * 3 + i] * v[1] + R[2 * 3 + i] * v[2];
}
// scaleestimator.cpp:37-91.  The reference's mean uses V[3] (one past the end of V) for the fifth term; the mean cancels
// out of the least-squares slope (the time offsets sum to zero), so the term only moves the last bits: V3 is used here.
inline void est_acel_lsq4(ImuFilterHist &h, const double *vel, double *acel, const double *R, double dt) {
    double t[3];
    rt_vec(R, h.V2, t);
    memcpy(h.V3, t, sizeof(t));
    rt_vec(R, h.V1, t);
    memcpy(h.V2, t, sizeof(t));
    rt_vec(R, h.V0, t);
    memcpy(h.V1, t, sizeof(t));
    rt_vec(R, h.V, t);
    memcpy(h.V0, t, sizeof(t));
    memcpy(h.V, vel, sizeof(t));
    for (int i = 0; i < 3; i++) h.Dt[i] = h.Dt[i + 1];
    h.Dt[3] = dt;
    h.T[0] = 0;
    double mt = 0;
    for (int i = 0; i < 4; i++) {
        h.T[i + 1] = h.T[i] + h.Dt[i];
        mt += h.T[i + 1];
    }
    mt /= 5;
    double den = 0;
    for (int i = 0; i < 5; i++) den += (h.T[i] - mt) * (h.T[i] - mt);
    for (int i = 0; i < 3; i++) {
        const double vm = (h.V[i] + h.V0[i] + h.V1[i] + h.V2[i] + h.V3[i]) / 5.0;
        double num = (h.V[i] - vm) * (h.T[4] - mt);
        num += (h.V0[i] - vm) * (h.T[3] - mt);
        num += (h.V1[i] - vm) * (h.T[2] - mt);
        num += (h.V2[i] - vm) * (h.T[1] - mt);
        num += (h.V3[i] - vm) * (h.T[0] - mt);
        if (den > 0) acel[i] = num / den;
    }
}
inline void mean_acel4(ImuFilterHist &h, const double *s_acel, double *acel, const double *R) {   // :93-110
    double t[3];
    rt_vec(R, h.A1, t);
    memcpy(h.A2, t, sizeof(t));
    rt_vec(R, h.A0, t);
    memcpy(h.A1, t, sizeof(t));
    rt_vec(R, h.A, t);
    memcpy(h.A0, t, sizeof(t));
    memcpy(h.A, s_acel, sizeof(t));
    for (int i = 0; i < 3; i++) acel[i] = (h.A[i] + h.A0[i] + h.A1[i] + h.A2[i]) / 4;
}

struct KaParams {   // FunParams_KaGMEKBias (:117-126)
    double a_v[3], a_s[3], G, x_p[7], Rv[9], Rs[9], Rg, Pp[49];
};
// Problem_KaGMEKBias (:128-203): JtJ (7 x 7), JtF (7) of the posterior at x
inline void ka_problem(double *JtJ, double *JtF, const double *x, const KaParams &p) {
    const double a = x[0];
    const double *g = x + 1, *b = x + 4;
    const double ca = cos(a), sa = sin(a);
    double F[11] = {0};
    for (int i = 0; i < 3; i++) F[i] = (p.a_s[i] + g[i]) * ca - p.a_v[i] * sa;
    F[3] = dot(g, g, 3) - p.G * p.G;
    F[4] = x[0] - p.x_p[0];
    if (F[4] > M_PI) F[4] -= 2 * M_PI;
    else if (F[4] < -M_PI) F[4] += 2 * M_PI;
    double Rb[9], Rgv[3];
    so3_exp(b, Rb);
    matvec(Rb, g, Rgv, 3, 3);
    for (int i = 0; i < 3; i++) {
        F[5 + i] = Rgv[i] - p.x_p[1 + i];
        F[8 + i] = b[i] - p.x_p[4 + i];
    }
    double dFda[11] = {0};
    for (int i = 0; i < 3; i++) dFda[i] = -(p.a_s[i] + g[i]) * sa - p.a_v[i] * ca;
    dFda[4] = 1;
    const double Gx[9] = {0, Rgv[2], -Rgv[1], -Rgv[2], 0, Rgv[0], Rgv[1], -Rgv[0], 0};
    double dFdx1[11 * 6] = {0};
    for (int i = 0; i < 3; i++) {
        dFdx1[i * 6 + i] = ca;                    // dF(0:2)/dG
        dFdx1[3 * 6 + i] = 2 * g[i];              // dF(3)/dG
        for (int j = 0; j < 3; j++) {
            dFdx1[(5 + i) * 6 + j] = Rb[i * 3 + j];        // dF(5:7)/dG
            dFdx1[(5 + i) * 6 + 3 + j] = Gx[i * 3 + j];    // dF(5:7)/db
        }
        dFdx1[(8 + i) * 6 + 3 + i] = 1;           // dF(8:10)/db
    }
    double Pz[9];
    for (int i = 0; i < 9; i++) Pz[i] = sa * sa * p.Rv[i] + ca * ca * p.Rs[i];
    double P[121] = {0}, W[121] = {0}, dPda[121] = {0};
    double iPz[9], iPp[49];
    ldlt_inverse<3, false>(Pz, iPz);   // a zero pivot here makes W, and so JtJ, NaN either way
    ldlt_inverse<7, false>(p.Pp, iPp);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            P[i * 11 + j] = Pz[i * 3 + j];
            W[i * 11 + j] = iPz[i * 3 + j];
            dPda[i * 11 + j] = 2 * sa * ca * (p.Rv[i * 3 + j] - p.Rs[i * 3 + j]);
        }
    P[3 * 11 + 3] = p.Rg;
    W[3 * 11 + 3] = 1 / p.Rg;
    for (int i = 0; i < 7; i++)
        for (int j = 0; j < 7; j++) {
            P[(4 + i) * 11 + 4 + j] = p.Pp[i * 7 + j];
            W[(4 + i) * 11 + 4 + j] = iPp[i * 7 + j];
        }
    double t1[121], dWda[121];
    matmul(W, dPda, t1, 11, 11, 11);
    matmul(t1, W, dWda, 11, 11, 11);
    for (int i = 0; i < 121; i++) dWda[i] = -dWda[i];
    // JtJ(0,0) = 0.25*F*dWda*P*dWda*F + dFda*dWda*F + dFda*W*dFda
    double v1[11], v2[11], v3[11];
    matvec(dWda, F, v1, 11, 11);          // dWda*F
    matvec(P, v1, v2, 11, 11);            // P*dWda*F
    matvec(dWda, v2, v3, 11, 11);         // dWda*P*dWda*F
    double WdFda[11];
    matvec(W, dFda, WdFda, 11, 11);
    JtJ[0] = 0.25 * dot(F, v3, 11) + dot(dFda, v1, 11) + dot(dFda, WdFda, 11);
    // JtJ(1:6,0) = 0.5*dFdx1^T*dWda*F + dFdx1^T*W*dFda
    double dT[6 * 11];
    transpose(dFdx1, dT, 11, 6);
    double c1[6], c2[6];
    matvec(dT, v1, c1, 6, 11);
    matvec(dT, WdFda, c2, 6, 11);
    for (int i = 0; i < 6; i++) {
        const double v = 0.5 * c1[i] + c2[i];
        JtJ[(1 + i) * 7 + 0] = v;
        JtJ[0 * 7 + 1 + i] = v;
    }
    double WD[11 * 6], DWD[36];
    matmul(W, dFdx1, WD, 11, 11, 6);
    matmul(dT, WD, DWD, 6, 11, 6);
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) JtJ[(1 + i) * 7 + 1 + j] = DWD[i * 6 + j];
    double WF[11];
    matvec(W, F, WF, 11, 11);
    JtF[0] = 0.5 * dot(F, v1, 11) + dot(dFda, WF, 11);
    double c3[6];
    matvec(dT, WF, c3, 6, 11);
    for (int i = 0; i < 6; i++) JtF[1 + i] = c3[i];
}
inline double saturate(double v, double lim) { return v > lim ? lim : (v < -lim ? -lim : v); }   // util::saturate
// estKaGMEKBias (:213-318); returns the scale K = tan(X[0]) (0 when negative / NaN / inf)
inline double est_ka_gmek_bias(const double *s_acel, const double *f_acel, double kP, const double *Rot, double *X, double *P,
                               const double *Qg, const double *Qrot, const double *Qbias, double QKp, double Rg, const double *Rs,
                               const double *Rf, double *g_est, double *b_est, const double *Wvw, double *Xvw, double g_gravit) {
    double F[49] = {0};
    F[0] = kP;
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) F[(1 + i) * 7 + 1 + j] = Rot[j * 3 + i];   // Rot.T()
        F[(4 + i) * 7 + 4 + i] = 1;
    }
    const double G[3] = {X[1], X[2], X[3]};
    const double GProd[9] = {0, G[2], -G[1], -G[2], 0, G[0], G[1], -G[0], 0};
    double Q[49] = {0};
    const double tx = tan(X[0]);
    Q[0] = QKp / (1 + tx * tx);
    double GT[9], t9[9], q3[9];
    transpose(GProd, GT, 3, 3);
    matmul(GT, Qrot, t9, 3, 3, 3);
    matmul(t9, GProd, q3, 3, 3, 3);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            Q[(1 + i) * 7 + 1 + j] = q3[i * 3 + j] + Qg[i * 3 + j];
            Q[(4 + i) * 7 + 4 + j] = Qbias[i * 3 + j];
        }
    double Xn[7];
    matvec(F, X, Xn, 7, 7);
    memcpy(X, Xn, sizeof(Xn));
    double FT[49], t49[49], Pp[49];
    transpose(F, FT, 7, 7);
    matmul(F, P, t49, 7, 7, 7);
    matmul(t49, FT, Pp, 7, 7, 7);
    for (int i = 0; i < 49; i++) Pp[i] += Q[i];
    KaParams prm;
    memcpy(prm.a_s, s_acel, sizeof(prm.a_s));
    memcpy(prm.a_v, f_acel, sizeof(prm.a_v));
    memcpy(prm.Rs, Rs, sizeof(prm.Rs));
    memcpy(prm.Rv, Rf, sizeof(prm.Rv));
    memcpy(prm.Pp, Pp, sizeof(prm.Pp));
    prm.Rg = Rg;
    prm.G = g_gravit;
    memcpy(prm.x_p, X, sizeof(prm.x_p));
    double JtJ[49], JtF[7];
    for (int it = 0; it < 20; it++) {   // Minimizer<7,11,..>::GaussNewton(X, Problem, &params, 20, FunT): tolerances 0 -> 20 steps
        ka_problem(JtJ, JtF, X, prm);
        double rhs[7], h[7];
        for (int i = 0; i < 7; i++) rhs[i] = -JtF[i];
        sym_svd_backsub<7>(JtJ, rhs, h);
        for (int i = 0; i < 7; i++) X[i] += h[i];
        X[0] = atan2(sin(X[0]), cos(X[0]));   // FunT_KaGMEKBias (:205-209)
        for (int i = 4; i < 7; i++) X[i] = saturate(X[i], 5e-1 / 25);
    }
    ka_problem(JtJ, JtF, X, prm);
    ldlt_inverse<7, false>(JtJ, *(double (*)[49])P);   // J^T W J, J of full rank: no zero pivot
    double k = tan(X[0]);
    if (k < 0 || isnan(k) || isinf(k)) k = 0;
    for (int i = 0; i < 3; i++) {
        g_est[i] = X[1 + i];
        b_est[i] = X[4 + i];
    }
    // correct the visual measurement with the bias estimate (:296-309)
    double WVBias[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) WVBias[i * 3 + j] = JtJ[(4 + i) * 7 + 4 + j];
    double Wb[36] = {0}, Wsum[36], iW[36];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) Wb[(3 + i) * 6 + 3 + j] = WVBias[i * 3 + j];
    for (int i = 0; i < 36; i++) Wsum[i] = Wb[i] + Wvw[i];
    const double wc[3] = {Xvw[3] - b_est[0], Xvw[4] - b_est[1], Xvw[5] - b_est[2]};
    double WXc[6] = {0}, w3[3], rhs6[6], Xc[6];
    matvec(WVBias, wc, w3, 3, 3);
    for (int i = 0; i < 3; i++) WXc[3 + i] = w3[i];
    matvec(Wvw, Xvw, rhs6, 6, 6);
    for (int i = 0; i < 6; i++) rhs6[i] += WXc[i];
    ldlt_inverse<6, true>(Wsum, iW);   // a frame without forward matches: zero velocity block
    matvec(iW, rhs6, Xc, 6, 6);
    memcpy(Xvw, Xc, sizeof(Xc));
    return k;
}

}   // namespace rbimu

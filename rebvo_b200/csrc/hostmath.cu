// hostmath.cu -- C exports of the host/device algebra in lm.cuh so that the CPU test-suite can check it without a GPU
// against the reference's TooN results and numpy: SO3 exp/ln, and the solver instances the minimiser, the IMU stages and the
// IMU filter run (the LDL^T of lm.cuh with and without TooN's zero-pivot stop, its pivot rule, the Jacobi pseudo-inverse).
#include "lm.cuh"
#include "imu_filter.h"
#include <vector>

template <int N>
static const double (&arr(const double *p))[N] { return *(const double (*)[N])p; }
template <int N>
static double (&arr(double *p))[N] { return *(double (*)[N])p; }

extern "C" {
void rb_hostmath_so3_exp(const double *w, double *R) { so3_exp(w, R); }
void rb_hostmath_so3_ln(const double *R, double *w) { so3_ln_of_matrix(R, w); }
// the minimiser's solve (mc_solve): x = A^-1 b without the zero-pivot stop; piv = {smallest, largest} pivot
void rb_hostmath_ldlt6_solve(const double *A, const double *b, double *x, double *piv) {
    double a[36];
    ldlt_factor<6, false>(arr<36>(A), a, piv[0], piv[1]);
    ldlt_backsub<6>(a, arr<6>(b), arr<6>(x));
}
// get_inverse without the zero-pivot stop and with it (TooN's: every get_inverse site of the product), N = 3, 6, 7
void rb_hostmath_ldlt3_inverse(const double *A, double *inv) { ldlt_inverse<3, false>(arr<9>(A), arr<9>(inv)); }
void rb_hostmath_ldlt6_inverse(const double *A, double *inv) { ldlt_inverse<6, false>(arr<36>(A), arr<36>(inv)); }
void rb_hostmath_ldlt7_inverse(const double *A, double *inv) { ldlt_inverse<7, false>(arr<49>(A), arr<49>(inv)); }
void rb_hostmath_ldlt3_inverse_stop(const double *A, double *inv) { ldlt_inverse<3, true>(arr<9>(A), arr<9>(inv)); }
void rb_hostmath_ldlt6_inverse_stop(const double *A, double *inv) { ldlt_inverse<6, true>(arr<36>(A), arr<36>(inv)); }
void rb_hostmath_ldlt7_inverse_stop(const double *A, double *inv) { ldlt_inverse<7, true>(arr<49>(A), arr<49>(inv)); }
int rb_hostmath_ldlt_solves_like_svd(double dmin, double dmax) { return ldlt_solves_like_svd(dmin, dmax) ? 1 : 0; }
void rb_hostmath_sym_svd_backsub6(const double *A, const double *b, double *x) {
    sym_svd_backsub<6>(arr<36>(A), arr<6>(b), arr<6>(x));
}
void rb_hostmath_sym_svd_backsub7(const double *A, const double *b, double *x) {
    sym_svd_backsub<7>(arr<49>(A), arr<7>(b), arr<7>(x));
}
void rb_hostmath_mat3_inv(const double *A, double *B) { mat3_inv(A, B); }

// IMU-mode host filter chain (imu_filter.h) for the CPU parity test against the reference's ScaleEstimator / ImuGrabber
void *rb_hostmath_imu_hist_new() {
    rbimu::ImuFilterHist *h = new rbimu::ImuFilterHist;
    memset(h, 0, sizeof(*h));
    return h;
}
void rb_hostmath_imu_hist_free(void *h) { delete (rbimu::ImuFilterHist *)h; }
void rb_hostmath_est_acel_lsq4(void *h, const double *vel, double *acel, const double *R, double dt) {
    rbimu::est_acel_lsq4(*(rbimu::ImuFilterHist *)h, vel, acel, R, dt);
}
void rb_hostmath_mean_acel4(void *h, const double *s_acel, double *acel, const double *R) {
    rbimu::mean_acel4(*(rbimu::ImuFilterHist *)h, s_acel, acel, R);
}
double rb_hostmath_est_ka_gmek_bias(const double *s_acel, const double *f_acel, double kP, const double *Rot, double *X, double *P,
                                    const double *Qg, const double *Qrot, const double *Qbias, double QKp, double Rg,
                                    const double *Rs, const double *Rf, double *g_est, double *b_est, const double *Wvw,
                                    double *Xvw, double g_gravit) {
    return rbimu::est_ka_gmek_bias(s_acel, f_acel, kP, Rot, X, P, Qg, Qrot, Qbias, QKp, Rg, Rs, Rf, g_est, b_est, Wvw, Xvw, g_gravit);
}
// ImuGrabber dataset mode: integrate the samples (n x 7: t, gyro, accel) over consecutive frame intervals ts[0..nf-1]
// (first interval starts at 0 like FirstThr's t0); out: nf x 20 {n, dt, Rot[9], giro[3], acel[3], cacel[3]}
int rb_hostmath_imu_integrate(const double *samples, int n, const double *ts, int nf, double *out) {
    std::vector<rbimu::ImuSample> s(n);
    for (int i = 0; i < n; i++) {
        s[i].t = samples[i * 7];
        for (int k = 0; k < 3; k++) {
            s[i].giro[k] = samples[i * 7 + 1 + k];
            s[i].acel[k] = samples[i * 7 + 4 + k];
        }
    }
    rbimu::ImuBuffer b;
    b.init(s.data(), n, nullptr, nullptr);
    double t0 = 0;
    for (int f = 0; f < nf; f++) {
        const rbimu::ImuIntegral d = b.grab(t0, ts[f]);
        double *o = out + f * 20;
        o[0] = d.n;
        o[1] = d.dt;
        for (int k = 0; k < 9; k++) o[2 + k] = d.Rot[k];
        for (int k = 0; k < 3; k++) {
            o[11 + k] = d.giro[k];
            o[14 + k] = d.acel[k];
            o[17 + k] = d.cacel[k];
        }
        t0 = ts[f];
    }
    return 0;
}
// ImuGrabber live mode: the ring of rb_pipeline_set_imu_live (list_size samples, integration step tsample)
struct HostImuRing {
    std::vector<rbimu::ImuSample> slots;
    rbimu::ImuBuffer b;
};
void *rb_hostmath_imu_ring_new(int list_size, double tsample) {
    HostImuRing *r = new HostImuRing;
    r->slots.resize((size_t)list_size + 1);
    r->b.init_live(r->slots.data(), list_size, tsample, nullptr, nullptr);
    return r;
}
void rb_hostmath_imu_ring_free(void *r) { delete (HostImuRing *)r; }
// n rows {t, gyro, accel}: 1 when stored, 0 (nothing stored) when they do not fit
int rb_hostmath_imu_ring_push(void *r, const double *rows, int n) {
    std::vector<rbimu::ImuSample> s(n);
    for (int i = 0; i < n; i++) {
        s[i].t = rows[i * 7];
        for (int k = 0; k < 3; k++) {
            s[i].giro[k] = rows[i * 7 + 1 + k];
            s[i].acel[k] = rows[i * 7 + 4 + k];
        }
    }
    return ((HostImuRing *)r)->b.push(s.data(), n) ? 1 : 0;
}
// whether grab(tstart, tend) finds samples, without changing the ring (the check of a live-mode frame push)
int rb_hostmath_imu_ring_covers(void *r, double tstart, double tend) {
    rbimu::ImuBuffer probe = ((HostImuRing *)r)->b;
    return probe.release(tstart, tend) ? 1 : 0;
}
// out: 20 doubles as rb_hostmath_imu_integrate's, plus dgiro[3] at 20..22
void rb_hostmath_imu_ring_grab(void *r, double tstart, double tend, double *out) {
    const rbimu::ImuIntegral d = ((HostImuRing *)r)->b.grab(tstart, tend);
    out[0] = d.n;
    out[1] = d.dt;
    for (int k = 0; k < 9; k++) out[2 + k] = d.Rot[k];
    for (int k = 0; k < 3; k++) {
        out[11 + k] = d.giro[k];
        out[14 + k] = d.acel[k];
        out[17 + k] = d.cacel[k];
        out[20 + k] = d.dgiro[k];
    }
}
// {write_inx, read_inx, size, free slots}
void rb_hostmath_imu_ring_state(const void *r, int *out) {
    const rbimu::ImuBuffer &b = ((const HostImuRing *)r)->b;
    out[0] = b.write_inx;
    out[1] = b.read_inx;
    out[2] = b.size;
    out[3] = b.free_slots();
}
}

// TEST INFRASTRUCTURE ONLY -- never linked into, imported by or executed from the product path.
//
// ref_shim.cpp: a thin extern "C" window onto the UNMODIFIED reference classes so that the
// parity tests (ctypes) can drive the reference's own mtracklib stage by stage.  It is compiled
// by oracle/build_ref.py together with the reference translation units *where they lie* under
// /root/reference (no reference source is copied into this repository) into
// oracle/_ref/libref_mtrack.so.
//
// The call order mirrors src/rebvo/rebvo_first_t.cpp:259-272 (detector) and
// src/rebvo/rebvo_second_t.cpp:172-487 (tracker + mapper).
//
// global_tracker.cpp is #included (compiled in place) instead of linked so that the
// implicit template instantiations of TryVelRot<> are reachable for single-evaluation tests.

#include "mtracklib/global_tracker.cpp"  // resolved through -I<reference>/src by oracle/build_ref.py

#include "mtracklib/edge_tracker.h"
#include "mtracklib/sspace.h"
#include <cstring>

using namespace rebvo;
using namespace TooN;

struct RefMap {
    cam_model cam;
    sspace *ss;
    edge_tracker *ef;
    global_tracker *gt;
    Image<float> *img;
};

static Matrix<3, 3> M3(const double *m) {
    Matrix<3, 3> r;
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) r(i, j) = m[i * 3 + j];
    return r;
}
static void M3out(const Matrix<3, 3> &r, double *m) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) m[i * 3 + j] = r(i, j);
}

#include "CommLib/net_keypoint.h"
extern "C" {

int ref_sizeof_keyline() { return (int)sizeof(KeyLine); }

// rebvo.cpp:297-312: one sspace / edge_tracker(cam,255*3) / global_tracker per ring slot
void *ref_map_create(int w, int h, float ppx, float ppy, float zfx, float zfy, double sigma0,
                     double ksigma) {
    RefMap *m = new RefMap;
    cam_model::rad_tan_distortion kc = {0, 0, 0, 0, 0};
    m->cam = cam_model({ppx, ppy}, {zfx, zfy}, kc, {(uint)w, (uint)h});
    m->ss = new sspace(sigma0, ksigma, m->cam.sz, 3);
    m->ef = new edge_tracker(m->cam, 255 * 3);
    m->gt = new global_tracker(m->cam);
    m->img = new Image<float>(m->cam.sz);
    return m;
}
void ref_map_destroy(void *p) {
    RefMap *m = (RefMap *)p;
    delete m->ss;
    delete m->ef;
    delete m->gt;
    delete m->img;
    delete m;
}

// Image<float>::ConvertRGB2BW (image.h:197-203)
void ref_rgb2bw(void *p, const unsigned char *rgb) {
    RefMap *m = (RefMap *)p;
    Image<RGB24Pixel> c((RGB24Pixel *)rgb, m->cam.sz);
    Image<float>::ConvertRGB2BW(*m->img, c);
}
void ref_set_gray(void *p, const float *g) {
    RefMap *m = (RefMap *)p;
    memcpy(m->img->Data(), g, sizeof(float) * m->img->bSize());
}
// sspace::build (sspace.cpp:52-60)
void ref_build(void *p) {
    RefMap *m = (RefMap *)p;
    m->ss->build(*m->img);
}
// which: 0 img0, 1 img1, 2 dog, 3 dx, 4 dy, 5 gray
void ref_get_plane(void *p, int which, float *out) {
    RefMap *m = (RefMap *)p;
    Image<float> *im = which == 0   ? &m->ss->Img(0)
                       : which == 1 ? &m->ss->Img(1)
                       : which == 2 ? &m->ss->ImgDOG()
                       : which == 3 ? &m->ss->ImgDx()
                       : which == 4 ? &m->ss->ImgDy()
                                    : m->img;
    memcpy(out, im->Data(), sizeof(float) * im->bSize());
}
// edge_finder::detect (edge_finder.cpp:342-365)
int ref_detect(void *p, int plane_fit, double pos_neg, double dog_thresh, int kl_max, double *tresh,
               int *l_kl_num, int kl_ref, double gain, double tmax, double tmin) {
    RefMap *m = (RefMap *)p;
    m->ef->detect(m->ss, plane_fit, pos_neg, dog_thresh, kl_max, *tresh, *l_kl_num, kl_ref, gain,
                  tmax, tmin);
    return m->ef->KNum();
}
// edge_finder::reEstimateThresh (edge_finder.cpp:373-405); returns the int cast the reference returns,
// *out gets the float it stores (getThresh()).
int ref_reestimate(void *p, int knum, int n, float *out) {
    RefMap *m = (RefMap *)p;
    int r = m->ef->reEstimateThresh(knum, n);
    *out = m->ef->getThresh();
    return r;
}
int ref_knum(void *p) { return ((RefMap *)p)->ef->KNum(); }
void ref_get_keylines(void *p, void *out) {
    RefMap *m = (RefMap *)p;
    if (m->ef->KNum() > 0) memcpy(out, &(*m->ef)[0], sizeof(KeyLine) * m->ef->KNum());
}
void ref_set_keylines(void *p, const void *in, int n) {
    RefMap *m = (RefMap *)p;
    if (n > 0) memcpy(&(*m->ef)[0], in, sizeof(KeyLine) * n);
}
// mask lives in a protected member; reach it through a derived accessor
struct MaskPeek : public edge_tracker {
    using edge_tracker::edge_tracker;
    Image<int> &mask() { return img_mask_kl; }
    int &knref() { return kn; }
};
void ref_get_mask(void *p, int *out) {
    RefMap *m = (RefMap *)p;
    MaskPeek *mp = (MaskPeek *)m->ef;
    memcpy(out, mp->mask().Data(), sizeof(int) * mp->mask().bSize());
}
void ref_set_mask(void *p, const int *in, int kn) {
    RefMap *m = (RefMap *)p;
    MaskPeek *mp = (MaskPeek *)m->ef;
    memcpy(mp->mask().Data(), in, sizeof(int) * mp->mask().bSize());
    mp->knref() = kn;
}
// edge_tracker::EstimateQuantile (edge_tracker.cpp:1148-1186)
double ref_quantile(void *p, double smin, double smax, double perc, int n) {
    return ((RefMap *)p)->ef->EstimateQuantile(smin, smax, perc, n);
}
// global_tracker::build_field (global_tracker.cpp:61-105)
void ref_build_field(void *p, int radius, float min_mod) {
    RefMap *m = (RefMap *)p;
    m->gt->build_field(*m->ef, radius, min_mod);
}
struct FieldPeek {  // same layout as global_tracker's leading members (global_tracker.h:42-44)
    Image<gt_field_data> field;
};
void ref_get_field(void *p, int *out) {  // out: 2*N ints {dist, ikl}
    RefMap *m = (RefMap *)p;
    FieldPeek *fp = (FieldPeek *)m->gt;
    memcpy(out, fp->field.Data(), sizeof(gt_field_data) * fp->field.bSize());
}
// global_tracker::Minimizer_RV<double> (global_tracker.cpp:578-819); pn = map providing the field (new),
// po = old map whose keylines are moved.
double ref_minimizer_rv(void *pn, void *po, double *V, double *W, double *RVel, double *RW0,
                        double match_thresh, int iter_max, int init_type, double reweight,
                        double *rel_err, double *rel_err_score, double max_s_rho,
                        unsigned match_num_thresh, double init_iter, double *W_X) {
    RefMap *mn = (RefMap *)pn, *mo = (RefMap *)po;
    Vector<3> v = makeVector(V[0], V[1], V[2]), w = makeVector(W[0], W[1], W[2]);
    Matrix<3, 3> rv = M3(RVel), rw = M3(RW0);
    Matrix<6, 6, double> wx = Zeros;
    double F = mn->gt->Minimizer_RV<double>(v, w, rv, rw, *mo->ef, match_thresh, iter_max, init_type,
                                            reweight, *rel_err, *rel_err_score, max_s_rho,
                                            match_num_thresh, init_iter, wx);
    for (int i = 0; i < 3; i++) {
        V[i] = v[i];
        W[i] = w[i];
    }
    M3out(rv, RVel);
    M3out(rw, RW0);
    for (int i = 0; i < 6; i++)
        for (int j = 0; j < 6; j++) W_X[i * 6 + j] = wx(i, j);
    return F;
}
// one global_tracker::TryVelRot<double,ReWeight,ProcJF,false> evaluation (global_tracker.cpp:285-543)
// res_in/res_out have pnum = (K0+3)&~3 entries.
double ref_try_vel_rot(void *pn, void *po, const double *X, int reweight, int procjf,
                       double match_thresh, double s_rho_min, unsigned match_num_thresh,
                       double k_huber, double *res_in, double *res_out, double *JtJ, double *JtF) {
    RefMap *mn = (RefMap *)pn, *mo = (RefMap *)po;
    edge_tracker &klist = *mo->ef;
    int pnum = (klist.KNum() + 3) & ~3;
    std::vector<double> P0Im(pnum * 3), P0m(pnum * 3);
    KltoI3PMatrix<double>(klist, pnum, P0Im.data());
    Ne10::ProyI3Pto3PMatrix<double>(P0m.data(), P0Im.data(), mn->cam.zfm, pnum);
    Matrix<6, 6, double> jtj = Zeros;
    Vector<6, double> jtf = Zeros, x;
    for (int i = 0; i < 6; i++) x[i] = X[i];
    Vector<3> z3 = Zeros;
    Matrix<3, 3> i3 = Identity;
    double s;
#define TVR(RW, PJ)                                                                               \
    s = mn->gt->TryVelRot<double, RW, PJ, false>(jtj, jtf, x, z3, i3, z3, i3, klist, P0m.data(),  \
                                                  pnum, match_thresh, s_rho_min, match_num_thresh, \
                                                  k_huber, res_in, res_out)
    if (reweight && procjf) TVR(true, true);
    else if (reweight) TVR(true, false);
    else if (procjf) TVR(false, true);
    else TVR(false, false);
#undef TVR
    for (int i = 0; i < 6; i++) {
        JtF[i] = jtf[i];
        for (int j = 0; j < 6; j++) JtJ[i * 6 + j] = jtj(i, j);
    }
    return s;
}
// edge_tracker::FordwardMatch (edge_tracker.cpp:380-436)
int ref_forward_match(void *po, void *pn) {
    return ((RefMap *)po)->ef->FordwardMatch(((RefMap *)pn)->ef);
}
// edge_tracker::rotate_keylines (edge_tracker.cpp:42-76)
void ref_rotate(void *p, const double *R) { ((RefMap *)p)->ef->rotate_keylines(M3(R)); }
// edge_tracker::directed_matching (edge_tracker.cpp:302-374)
int ref_directed_matching(void *pn, void *po, const double *V, const double *RVel,
                          const double *BackRot, int *kf_matchs, double thr_mod, double thr_ang,
                          double max_radius, double loc_unc) {
    RefMap *mn = (RefMap *)pn, *mo = (RefMap *)po;
    return mn->ef->directed_matching(makeVector(V[0], V[1], V[2]), M3(RVel), M3(BackRot), mo->ef,
                                     *kf_matchs, thr_mod, thr_ang, max_radius, loc_unc, false);
}
// copy_net_keyline + copy_net_keyline_nextid (src/CommLib/net_keypoint.cpp:29-107), monocular; out: 15 bytes per record
int ref_pack_net(void *p, unsigned char *out, int kl_size, double k_prof) {
    RefMap *m = (RefMap *)p;
    const int n = copy_net_keyline(*m->ef, nullptr, (net_keyline *)out, kl_size, k_prof);
    copy_net_keyline_nextid(*m->ef, (net_keyline *)out, kl_size);
    return n;
}
int ref_sizeof_net_keyline() { return (int)sizeof(net_keyline); }
int ref_num_matches(void *p) { return ((RefMap *)p)->ef->NumMatches(); }
// edge_tracker::Regularize_1_iter (edge_tracker.cpp:87-148)
int ref_regularize(void *p, double thresh) { return ((RefMap *)p)->ef->Regularize_1_iter(thresh); }
// edge_tracker::UpdateInverseDepthKalman (edge_tracker.cpp:695-724, 954-1055)
void ref_ekf(void *p, const double *V, const double *RVel, const double *RW0, double qabs,
             double qrel, double loc_unc) {
    ((RefMap *)p)
        ->ef->UpdateInverseDepthKalman(makeVector(V[0], V[1], V[2]), M3(RVel), M3(RW0), qabs, qrel,
                                       loc_unc);
}
// edge_tracker::EstimateReScalingOpt (edge_tracker.cpp:1104-1140)
double ref_rescale(void *p, double *RKp, double s_rho_min, unsigned match_num_min, int re_escale) {
    return ((RefMap *)p)->ef->EstimateReScalingOpt(*RKp, s_rho_min, match_num_min, re_escale != 0);
}
// TooN SO3 exp / ln as used at rebvo_second_t.cpp:360-361,567
void ref_so3_exp(const double *w, double *R) {
    SO3<> r(makeVector(w[0], w[1], w[2]));
    M3out(r.get_matrix(), R);
}
void ref_so3_ln(const double *R, double *w) {
    SO3<> r(M3(R));
    Vector<3> l = r.ln();
    for (int i = 0; i < 3; i++) w[i] = l[i];
}
}  // extern "C"

// ---- TooN::Cholesky<N> (Cholesky.h): x = backsub(b) and inv = get_inverse(), for the sizes the product solves ------------
#include <TooN/Cholesky.h>
template <int N>
static void ref_cholesky(const double *A, const double *b, double *x, double *inv) {
    Matrix<N, N> m;
    Vector<N> v;
    for (int i = 0; i < N; i++) {
        v[i] = b[i];
        for (int j = 0; j < N; j++) m(i, j) = A[i * N + j];
    }
    Cholesky<N> ch(m);
    const Vector<N> r = ch.backsub(v);
    const Matrix<N, N> mi = ch.get_inverse();
    for (int i = 0; i < N; i++) {
        x[i] = r[i];
        for (int j = 0; j < N; j++) inv[i * N + j] = mi(i, j);
    }
}
extern "C" {
void ref_cholesky3(const double *A, const double *b, double *x, double *inv) { ref_cholesky<3>(A, b, x, inv); }
void ref_cholesky6(const double *A, const double *b, double *x, double *inv) { ref_cholesky<6>(A, b, x, inv); }
void ref_cholesky7(const double *A, const double *b, double *x, double *inv) { ref_cholesky<7>(A, b, x, inv); }
}

// ---- image_undistort (SURVEY.md 8(f) rank 1): reference undistort<true> on RGB24 -------------------------
#include "VideoLib/image_undistort.h"
extern "C" void ref_undistort_rgb(int w, int h, float ppx, float ppy, float zfx, float zfy, const double *kc,
                                  const unsigned char *in, unsigned char *out) {
    cam_model::rad_tan_distortion d = {kc[0], kc[1], kc[2], kc[3], kc[4]};
    cam_model cam({ppx, ppy}, {zfx, zfy}, d, {(uint)w, (uint)h});
    image_undistort und(cam);
    Image<RGB24Pixel> i((RGB24Pixel *)in, cam.sz), o((RGB24Pixel *)out, cam.sz);
    und.undistort<true>(o, i);
}

// ---- IMU-mode rows (SURVEY.md 8(a) K6, K13) ------------------------------------------------------------------
extern "C" {
// global_tracker::TryVel<double> (global_tracker.cpp:829-934); residuals: K0 doubles, updated in place
double ref_try_vel(void *pn, void *po, const double *V, double match_thresh, double s_rho_min, unsigned mnt,
                   double *residuals, double rw_dist, float min_mod, double *JtJ, double *JtF) {
    RefMap *mn = (RefMap *)pn, *mo = (RefMap *)po;
    Matrix<3, 3> jtj;
    Vector<3> jtf;
    double s = mn->gt->TryVel<double>(jtj, jtf, makeVector(V[0], V[1], V[2]), *mo->ef, match_thresh, s_rho_min, mnt,
                                      residuals, rw_dist, min_mod);
    M3out(jtj, JtJ);
    for (int i = 0; i < 3; i++) JtF[i] = jtf[i];
    return s;
}
// global_tracker::Minimizer_V<double> (global_tracker.cpp:1036-1093)
double ref_minimizer_v(void *pn, void *po, double *V, double *RVel, double match_thresh, int iter_max, double s_rho_min,
                       unsigned mnt, double rw_dist, float min_mod) {
    RefMap *mn = (RefMap *)pn, *mo = (RefMap *)po;
    Vector<3> v = makeVector(V[0], V[1], V[2]);
    Matrix<3, 3> rv = Zeros;
    double F = mn->gt->Minimizer_V<double>(v, rv, *mo->ef, match_thresh, iter_max, s_rho_min, mnt, rw_dist, min_mod);
    for (int i = 0; i < 3; i++) V[i] = v[i];
    M3out(rv, RVel);
    return F;
}
// edge_tracker::ExtRotVel(vel, Wx, Rx, X, LocUncert, HubReweigth) (edge_tracker.cpp:1207-1301)
int ref_ext_rot_vel(void *p, const double *V, double *Wx, double *Rx, double *X, double loc_unc, double hub) {
    RefMap *m = (RefMap *)p;
    Matrix<6, 6> wx = Zeros, rx = Zeros;
    Vector<6> x = Zeros;
    bool ok = m->ef->ExtRotVel(makeVector(V[0], V[1], V[2]), wx, rx, x, loc_unc, hub);
    for (int i = 0; i < 6; i++) {
        X[i] = x[i];
        for (int j = 0; j < 6; j++) {
            Wx[i * 6 + j] = wx(i, j);
            Rx[i * 6 + j] = rx(i, j);
        }
    }
    return ok ? 1 : 0;
}
// edge_tracker::BiasCorrect (edge_tracker.cpp:1308-1338)
void ref_bias_correct(double *X, double *Wx, double *Gb, double *Wb, const double *Rg, const double *Rb) {
    Vector<6> x;
    Matrix<6, 6> wx;
    for (int i = 0; i < 6; i++) {
        x[i] = X[i];
        for (int j = 0; j < 6; j++) wx(i, j) = Wx[i * 6 + j];
    }
    Vector<3> gb = makeVector(Gb[0], Gb[1], Gb[2]);
    Matrix<3, 3> wb = M3(Wb);
    edge_tracker::BiasCorrect(x, wx, gb, wb, M3(Rg), M3(Rb));
    for (int i = 0; i < 6; i++) {
        X[i] = x[i];
        for (int j = 0; j < 6; j++) Wx[i * 6 + j] = wx(i, j);
    }
    for (int i = 0; i < 3; i++) Gb[i] = gb[i];
    M3out(wb, Wb);
}
}

// ---- IMU-mode host filter chain (config 3): ScaleEstimator (src/mtracklib/scaleestimator.cpp) and ImuGrabber's dataset
// integration (src/UtilLib/imugrabber.cpp), for tests/test_cpu_imu_filter.py -------------------------------------------------
#include "mtracklib/scaleestimator.h"
#include "UtilLib/imugrabber.h"
extern "C" {
void ref_est_acel_lsq4(const double *vel, double *acel, const double *R, double dt) {
    Vector<3> v = makeVector(vel[0], vel[1], vel[2]), a = makeVector(acel[0], acel[1], acel[2]);
    ScaleEstimator::EstAcelLsq4(v, a, M3(R), dt);
    for (int i = 0; i < 3; i++) acel[i] = a[i];
}
void ref_mean_acel4(const double *s_acel, double *acel, const double *R) {
    Vector<3> s = makeVector(s_acel[0], s_acel[1], s_acel[2]), a = Zeros;
    ScaleEstimator::MeanAcel4(s, a, M3(R));
    for (int i = 0; i < 3; i++) acel[i] = a[i];
}
static Matrix<3, 3> M3c(const double *m) { return M3(m); }
double ref_est_ka_gmek_bias(const double *s_acel, const double *f_acel, double kP, const double *Rot, double *X, double *P,
                            const double *Qg, const double *Qrot, const double *Qbias, double QKp, double Rg, const double *Rs,
                            const double *Rf, double *g_est, double *b_est, const double *Wvw, double *Xvw, double g_gravit) {
    Vector<3> sa = makeVector(s_acel[0], s_acel[1], s_acel[2]), fa = makeVector(f_acel[0], f_acel[1], f_acel[2]), ge = Zeros, be = Zeros;
    Vector<7> x;
    Matrix<7, 7> p;
    for (int i = 0; i < 7; i++) {
        x[i] = X[i];
        for (int j = 0; j < 7; j++) p(i, j) = P[i * 7 + j];
    }
    Matrix<6, 6> wvw;
    Vector<6> xvw;
    for (int i = 0; i < 6; i++) {
        xvw[i] = Xvw[i];
        for (int j = 0; j < 6; j++) wvw(i, j) = Wvw[i * 6 + j];
    }
    const double k = ScaleEstimator::estKaGMEKBias(sa, fa, kP, M3c(Rot), x, p, M3c(Qg), M3c(Qrot), M3c(Qbias), QKp, Rg, M3c(Rs),
                                                   M3c(Rf), ge, be, wvw, xvw, g_gravit);
    for (int i = 0; i < 7; i++) {
        X[i] = x[i];
        for (int j = 0; j < 7; j++) P[i * 7 + j] = p(i, j);
    }
    for (int i = 0; i < 3; i++) {
        g_est[i] = ge[i];
        b_est[i] = be[i];
    }
    for (int i = 0; i < 6; i++) Xvw[i] = xvw[i];
    return k;
}
int ref_imu_integrate(const double *samples, int n, const double *ts, int nf, double *out) {
    std::vector<ImuData> v(n);
    for (int i = 0; i < n; i++) {
        v[i].tstamp = samples[i * 7];
        v[i].giro = makeVector(samples[i * 7 + 1], samples[i * 7 + 2], samples[i * 7 + 3]);
        v[i].acel = makeVector(samples[i * 7 + 4], samples[i * 7 + 5], samples[i * 7 + 6]);
        v[i].comp = Zeros;
    }
    ImuGrabber g(v);
    double t0 = 0;
    for (int f = 0; f < nf; f++) {
        IntegratedImuData d = g.GrabAndIntegrate(t0, ts[f]);
        double *o = out + f * 20;
        o[0] = d.n;
        o[1] = d.dt;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) o[2 + i * 3 + j] = d.Rot(i, j);
        for (int k = 0; k < 3; k++) {
            o[11 + k] = d.giro[k];
            o[14 + k] = d.acel[k];
            o[17 + k] = d.cacel[k];
        }
        t0 = ts[f];
    }
    return 0;
}
}

// imu_track.cu -- the IMU-mode rows of SURVEY.md section 8(a) (config 3, ImuMode>0):
//   K6  global_tracker::TryVel / Minimizer_V<double>   (src/mtracklib/global_tracker.cpp:829-934, 1036-1093)
//   K13 edge_tracker::ExtRotVel + BiasCorrect           (src/mtracklib/edge_tracker.cpp:1207-1338)
// TryVel is the translation-only counterpart of TryVelRot (3x3 normal equations, residuals divided by s_rho, in-place
// residual buffer); ExtRotVel builds one linearised 6-DoF system over the forward matches.  The per-keyline terms are
// evaluated in the reference's float/double mix; the sums over keylines use the library's fixed-order reduction
// (rel. difference vs the reference's sequential sums ~1e-15, tests allow 1e-10).  The 3x3 / 6x6 solves run on the
// host (they are O(1) work between evaluations): Minimizer_V's LM loop is host-driven because the IMU path is not the
// replay hot loop (rebvo_second_t.cpp:182-336 interleaves it with host-side IMU filtering anyway).
#include <math.h>

#include "common.cuh"
#include "lm.cuh"
#include "tracker.cuh"
#include "stage_reduce.cuh"

// One TryVel evaluation.  partials[k][block], k = 0..9: JtJ(0,0),(1,1),(2,2),(0,1),(0,2),(1,2), JtF[0..2], score.
__global__ void __launch_bounds__(STAGE_T) k_tv_eval(KLSoA old, const MapState *__restrict__ old_st,
                                                     const unsigned long long *__restrict__ field,
                                                     const float4 *__restrict__ fpack, const MapState *__restrict__ f_st,
                                                     const double *__restrict__ velp, double *__restrict__ res,
                                                     double *__restrict__ partials, int *blk_has, double *blk_last,
                                                     double zfm, float ppx, float ppy, int w, int h, double max_r,
                                                     double match_thresh, double s_rho_min, unsigned int mnt_arg,
                                                     double rw_dist, float min_mod) {
    __shared__ double s_part[10][STAGE_T / 32];
    __shared__ StaleSmem sm;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int i = blockIdx.x * STAGE_T + tid;
    const int K0 = old_st->kn;
    const double V0 = velp[0], V1 = velp[1], V2 = velp[2];
    const unsigned int fc = f_st->frame_count;
    const unsigned int mnt = mnt_arg < fc ? mnt_arg : fc;   // std::min(MatchNumThresh,FrameCount)
    double acc[10];
#pragma unroll
    for (int k = 0; k < 10; k++) acc[k] = 0;
    bool matched = false, need = false;
    double fi_own = 0;
    if (i < K0) {
        int mid_f = -1;
        const float n_m = old.n_m[i];
        const double rho = old.rho[i], s_rho = old.s_rho[i];
        const bool skip = (min_mod > 0 && n_m < min_mod) || s_rho > s_rho_min || (unsigned int)old.m_num[i] < mnt;
        if (!skip) {
            const float2 pm = old.p_m[i];
            const double r_prev = res[i];
            double weight = 1;
            if (r_prev > rw_dist) weight = rw_dist / r_prev;                        // :860-862
            const double z_p = 1.0 / rho + V2;
            double f;
            if (z_p <= 0) {
                f = (1 / (s_rho)) * max_r * weight;                                 // :867-871
                acc[9] = f * f;
            } else {
                const double rho_p = 1.0 / z_p;
                const double pjx = rho_p * (V0 * zfm - V2 * (double)pm.x) + (double)pm.x;   // :874-875
                const double pjy = rho_p * (V1 * zfm - V2 * (double)pm.y) + (double)pm.y;
                const double pix = pjx + (double)ppx, piy = pjy + (double)ppy;      // Hom2Img
                const int x = (int)(pix + 0.5), y = (int)(piy + 0.5);
                if (x < 1 || y < 1 || x >= w - 1 || y >= h - 1) {
                    f = (1 / (s_rho)) * max_r * weight;                             // :883-887
                    acc[9] = f * f;
                } else {
                    double df_dx = 0, df_dy = 0;
                    f = max_r / s_rho;                                               // Calc_f_J miss (:190-203)
                    const unsigned long long key = field[(size_t)y * w + x];
                    bool hit = false;
                    if (key != ~0ull) {
                        const int ikl = (int)(0xFFFFFFFFu - (unsigned int)(key & 0xFFFFFFFFull));
                        const float4 a = fpack[2 * ikl], b = fpack[2 * ikl + 1];
                        const float2 m = old.m_m[i];
                        const double p_n2 = (double)(n_m * n_m);                   // Test_f_k
                        const double p_esc = (double)(m.x * a.x + m.y * a.y);
                        if (!(fabs(p_esc - p_n2) > match_thresh * p_n2)) {
                            const double dx = pix - (double)a.z, dy = piy - (double)a.w;
                            const double fi = dx * (double)b.x + dy * (double)b.y;
                            df_dx = (double)b.x / s_rho;
                            df_dy = (double)b.y / s_rho;
                            f = fi / s_rho;
                            matched = true;
                            fi_own = fi;
                            mid_f = ikl;
                            hit = true;
                        }
                    }
                    if (!hit) need = true;
                    f *= weight;
                    const double jx = rho_p * zfm * df_dx * weight;                  // :899-901
                    const double jy = rho_p * zfm * df_dy * weight;
                    const double jz = -rho_p * (pjx * df_dx + pjy * df_dy) * weight;
                    acc[0] = jx * jx;
                    acc[1] = jy * jy;
                    acc[2] = jz * jz;
                    acc[3] = jx * jy;
                    acc[4] = jx * jz;
                    acc[5] = jy * jz;
                    acc[6] = jx * f;
                    acc[7] = jy * f;
                    acc[8] = jz * f;
                    acc[9] = f * f;
                }
            }
        }
        old.m_id_f[i] = mid_f;
    }
    // Residuals[ikl]=fabs(fi), fi of the last match on a miss (:836)
    const double stale = block_stale_fi(matched, fi_own, true, sm, blk_has, blk_last, lane, wid);
    if (matched) res[i] = fabs(fi_own);
    else if (need) res[i] = stale;
    block_sum_to<10>(acc, s_part, lane, wid, partials + blockIdx.x, STAGE_T);
}

static int tv_eval(rb_ctx *c, rb_map *fmap, rb_map *old, const double vel[3], double match_thresh, double s_rho_min,
                   unsigned int mnt, double rw_dist, float min_mod, double JtJ[9], double JtF[3], double *score) {
    double *args = (double *)((char *)c->dev_small + RB_DS_ARGS), *pin = (double *)((char *)c->pinned + RB_DS_ARGS);
    memcpy(pin, vel, sizeof(double) * 3);
    RB_CUDA(cudaMemcpyAsync(args, pin, sizeof(double) * 3, cudaMemcpyHostToDevice, c->stream));
    const int nb = fmap->ts_host.nblk;
    k_tv_eval<<<nb, STAGE_T, 0, c->stream>>>(old->kl, old->st, fmap->field, fmap->kl.pack, fmap->st, args, fmap->res[0],
                                             fmap->ts_host.partials, fmap->ts_host.blk_has, fmap->ts_host.blk_last_fi, c->zfm,
                                             c->ppx, c->ppy, c->w, c->h, (double)fmap->field_radius, match_thresh, s_rho_min,
                                             mnt, rw_dist, min_mod);
    RB_LAUNCH_CHECK();
    k_blocks_finish<10><<<nb, STAGE_T, 0, c->stream>>>(fmap->ts_host.partials, nb, args + 8, fmap->res[0],
                                                       fmap->ts_host.blk_has, fmap->ts_host.blk_last_fi, old->st, true);
    RB_LAUNCH_CHECK();
    RB_CUDA(cudaMemcpyAsync(pin + 8, args + 8, sizeof(double) * 10, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    const double *s = pin + 8;
    JtJ[0] = s[0];
    JtJ[4] = s[1];
    JtJ[8] = s[2];
    JtJ[1] = JtJ[3] = s[3];
    JtJ[2] = JtJ[6] = s[4];
    JtJ[5] = JtJ[7] = s[5];
    JtF[0] = s[6];
    JtF[1] = s[7];
    JtF[2] = s[8];
    *score = s[9];
    return RB_OK;
}

// global_tracker::TryVel<double> -- one evaluation; residuals (|fi| per old keyline) are read and updated in place
extern "C" int rb_try_vel(rb_map *fmap, rb_map *old, const double Vel[3], double match_thresh, double s_rho_min,
                          uint32_t match_num_thresh, double *residuals, double reweigth_distance, float min_mod,
                          double JtJ[9], double JtF[3], double *score) {
    if (!fmap || !old) return RB_ERR_ARG;
    RB_ENTER(fmap->c);
    rb_ctx *c = fmap->c;
    if (fmap->field_radius <= 0) return RB_ERR_STATE;
    MapState so;
    int r = rb_read_map_state(old, &so);
    if (r) return r;
    if (residuals && so.kn > 0)
        RB_CUDA(cudaMemcpyAsync(fmap->res[0], residuals, sizeof(double) * so.kn, cudaMemcpyHostToDevice, c->stream));
    if ((r = tv_eval(c, fmap, old, Vel, match_thresh, s_rho_min, match_num_thresh, reweigth_distance, min_mod, JtJ, JtF,
                     score)))
        return r;
    if (residuals && so.kn > 0) {
        RB_CUDA(cudaMemcpyAsync(residuals, fmap->res[0], sizeof(double) * so.kn, cudaMemcpyDeviceToHost, c->stream));
        RB_CUDA(cudaStreamSynchronize(c->stream));
    }
    return RB_OK;
}

// global_tracker::Minimizer_V<double> (global_tracker.cpp:1036-1093)
extern "C" int rb_minimizer_v(rb_map *fmap, rb_map *old, double Vel[3], double RVel[9], double match_thresh, int iter_max,
                              double s_rho_min, uint32_t match_num_thresh, double reweigth_distance, float min_mod,
                              double *score) {
    if (!fmap || !old) return RB_ERR_ARG;
    RB_ENTER(fmap->c);
    rb_ctx *c = fmap->c;
    if (fmap->field_radius <= 0) return RB_ERR_STATE;
    int r;
    RB_CUDA(cudaMemsetAsync(fmap->res[0], 0, sizeof(double) * (size_t)c->kcap, c->stream));   // residuals[i]=0
    double JtJ[9], JtF[3], JtJn[9], JtFn[3], ApI[9], inv[9], h[3], Vnew[3], F, Fnew;
    if ((r = tv_eval(c, fmap, old, Vel, match_thresh, s_rho_min, match_num_thresh, reweigth_distance, min_mod, JtJ, JtF, &F)))
        return r;
    double v = 2, tau = 1e-3, mx = JtJ[0];
    for (int i = 1; i < 9; i++)
        if (JtJ[i] > mx) mx = JtJ[i];
    double u = tau * mx, gain;
    for (int it = 0; it < iter_max; it++) {
        for (int i = 0; i < 9; i++) ApI[i] = JtJ[i];
        for (int i = 0; i < 3; i++) ApI[i * 3 + i] = JtJ[i * 3 + i] + u;
        mat3_inv(ApI, inv);                                     // h=util::Matrix3x3Inv(ApI)*(-JtF)
        double nf[3] = {-JtF[0], -JtF[1], -JtF[2]};
        mat3_vec(inv, nf, h);
        for (int i = 0; i < 3; i++) Vnew[i] = Vel[i] + h[i];
        if ((r = tv_eval(c, fmap, old, Vnew, match_thresh, s_rho_min, match_num_thresh, reweigth_distance, min_mod, JtJn, JtFn,
                         &Fnew)))
            return r;
        double den = 0;
        for (int i = 0; i < 3; i++) den += (0.5 * h[i]) * (u * h[i] - JtF[i]);
        gain = (F - Fnew) / den;
        if (gain > 0) {
            F = Fnew;
            for (int i = 0; i < 3; i++) Vel[i] = Vnew[i];
            for (int i = 0; i < 9; i++) JtJ[i] = JtJn[i];
            for (int i = 0; i < 3; i++) JtF[i] = JtFn[i];
            const double g = 2 * gain - 1, f = 1 - (g * g * g);
            u *= (0.33 > f ? 0.33 : f);
            v = 2;
        } else {
            u *= v;
            v *= 2;
        }
    }
    mat3_inv(JtJ, RVel);
    if (score) *score = F;
    return RB_OK;
}

// ---- ExtRotVel (edge_tracker.cpp:1207-1301): sums of Phi^T Phi (21) and Phi^T Y (6) over the matched keylines ------
__global__ void __launch_bounds__(STAGE_T) k_extrotvel(KLSoA kl, const MapState *__restrict__ st,
                                                       const double *__restrict__ velp, double *__restrict__ partials,
                                                       double zf, double loc_unc, double hub) {
    __shared__ double s_part[27][STAGE_T / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int i = blockIdx.x * STAGE_T + tid;
    double acc[27];
#pragma unroll
    for (int k = 0; k < 27; k++) acc[k] = 0;
    if (i < st->kn && kl.m_id[i] >= 0) {
        const double vel0 = velp[0], vel1 = velp[1], vel2 = velp[2];
        const float2 u = kl.u_m[i], pm = kl.p_m[i], pm0 = kl.p_m_0[i];
        const float u_x = u.x, u_y = u.y;
        const double rho = kl.rho[i], s_rho = kl.s_rho[i];
        const double rho_t = 1 / (1 / rho + vel2);
        const float qt_x = (float)((double)pm0.x + rho_t * (vel0 * zf - vel2 * (double)pm0.x));
        const float qt_y = (float)((double)pm0.y + rho_t * (vel1 * zf - vel2 * (double)pm0.y));
        const float q_x = pm.x, q_y = pm.y;
        double P[6];
        P[0] = (double)u_x * rho_t * zf;
        P[1] = (double)u_y * rho_t * zf;
        P[2] = (double)u_x * (-rho_t * (double)q_x) + (double)u_y * (-rho_t * (double)q_y);
        P[3] = (double)(-u_x * q_x * q_y) / zf - (double)u_y * (zf + (double)(q_y * q_y) / zf);
        P[4] = (double)(+u_y * q_x * q_y) / zf + (double)u_x * (zf + (double)(q_x * q_x) / zf);
        P[5] = (double)(-u_x * q_y + u_y * q_x);
        double Y = (double)(u_x * (pm.x - qt_x) + u_y * (pm.y - qt_y));
        const float dqvel = (float)((double)u_x * (vel0 * zf - vel2 * (double)pm0.x) + (double)u_y * (vel1 * zf - vel2 * (double)pm0.y));
        const float s_y = (float)sqrt(s_rho * s_rho * (double)dqvel * (double)dqvel + loc_unc * loc_unc);
        double weigth = 1;
        if (fabs(Y) > hub) weigth = fabs(Y) / hub;
        const double div = (double)s_y * weigth;
#pragma unroll
        for (int k = 0; k < 6; k++) P[k] /= div;
        Y /= div;
        int k = 0;
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = a; b < 6; b++) acc[k++] = P[a] * P[b];
#pragma unroll
        for (int a = 0; a < 6; a++) acc[21 + a] = P[a] * Y;
    }
    block_sum_to<27>(acc, s_part, lane, wid, partials + blockIdx.x, STAGE_T);
}

// edge_tracker::ExtRotVel(vel, Wx, Rx, X, LocUncert, HubReweigth); returns *ok = 0 when the estimate is NaN (the reference
// returns false, edge_tracker.cpp:1294-1297)
extern "C" int rb_ext_rot_vel(rb_map *m, const double vel[3], double Wx[36], double Rx[36], double X[6],
                              double loc_uncertainty, double hub_reweight, int *ok) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    double *args = (double *)((char *)c->dev_small + RB_DS_ARGS), *pin = (double *)((char *)c->pinned + RB_DS_ARGS);
    memcpy(pin, vel, sizeof(double) * 3);
    RB_CUDA(cudaMemcpyAsync(args, pin, sizeof(double) * 3, cudaMemcpyHostToDevice, c->stream));
    const int nb = m->ts_host.nblk;
    k_extrotvel<<<nb, STAGE_T, 0, c->stream>>>(m->kl, m->st, args, m->ts_host.partials, c->zfm, loc_uncertainty, hub_reweight);
    RB_LAUNCH_CHECK();
    k_blocks_finish<27><<<1, 32, 0, c->stream>>>(m->ts_host.partials, nb, args + 8, nullptr, nullptr, nullptr, nullptr,
                                                 false);
    RB_LAUNCH_CHECK();
    RB_CUDA(cudaMemcpyAsync(pin + 8, args + 8, sizeof(double) * 27, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    const double *s = pin + 8;
    double JtJ[36], JtF[6];
    int k = 0;
    for (int a = 0; a < 6; a++)
        for (int b = a; b < 6; b++) {
            JtJ[a * 6 + b] = s[k];
            JtJ[b * 6 + a] = s[k];
            k++;
        }
    for (int a = 0; a < 6; a++) JtF[a] = s[21 + a];
    // SVD<> SVDpTp(JtJ); X=backsub(JtF); Rx=get_pinv(); Wx=JtJ  -- symmetric input: Jacobi eigen-decomposition
    sym_svd_backsub(JtJ, 6, JtF, X);
    for (int col = 0; col < 6; col++) {
        double e[6] = {0, 0, 0, 0, 0, 0}, x[6];
        e[col] = 1;
        sym_svd_backsub(JtJ, 6, e, x);
        for (int row = 0; row < 6; row++) Rx[row * 6 + col] = x[row];
    }
    for (int i = 0; i < 36; i++) Wx[i] = JtJ[i];
    bool nan = false;
    for (int i = 0; i < 36; i++) nan = nan || isnan(Rx[i]);
    for (int i = 0; i < 6; i++) nan = nan || isnan(X[i]);
    if (ok) *ok = nan ? 0 : 1;
    return RB_OK;
}

// edge_tracker::BiasCorrect (edge_tracker.cpp:1308-1338): gyro-prior fusion, pure 3x3 / 6x6 host algebra
extern "C" int rb_bias_correct(double X[6], double Wx[36], double Gb[3], double Wb[9], const double Rg[9],
                               const double Rb[9]) {
    double Wg[9], t[9], t2[9], iWgWb[9];
    mat3_inv(Rg, Wg);                                   // Wg = inv(Rg)
    mat3_inv(Wb, t);                                    // Wb = inv(inv(Wb)+Rb)
    for (int i = 0; i < 9; i++) t[i] = t[i] + Rb[i];
    mat3_inv(t, Wb);
    double Wxb[36];
    for (int i = 0; i < 36; i++) Wxb[i] = Wx[i];
    for (int i = 0; i < 9; i++) t[i] = Wg[i] + Wb[i];
    mat3_inv(t, iWgWb);                                 // iWgWb = inv(Wg+Wb)
    mat3_mul(iWgWb, Wg, t);                             // Wg*(Identity - iWgWb*Wg)
    for (int i = 0; i < 9; i++) t[i] = ((i % 4 == 0) ? 1.0 : 0.0) - t[i];
    mat3_mul(Wg, t, t2);
    for (int r = 0; r < 3; r++)
        for (int cc = 0; cc < 3; cc++) Wxb[(r + 3) * 6 + cc + 3] += t2[r * 3 + cc];
    double X1[6];
    for (int r = 0; r < 6; r++) {                       // X1 = Wx*X
        double s = 0;
        for (int k = 0; k < 6; k++) s += Wx[r * 6 + k] * X[k];
        X1[r] = s;
    }
    double v3[3], w3[3];
    mat3_mul(Wg, iWgWb, t);                             // X1.slice<3,3>() += Wg*iWgWb*Wb*Gb
    mat3_mul(t, Wb, t2);
    mat3_vec(t2, Gb, v3);
    for (int i = 0; i < 3; i++) X1[3 + i] += v3[i];
    Chol6 ch;                                           // X = Cholesky<6>(Wxb).get_inverse()*X1
    chol6_compute(Wxb, &ch);
    double inv[36];
    chol6_inverse(&ch, inv);
    for (int r = 0; r < 6; r++) {
        double s = 0;
        for (int k = 0; k < 6; k++) s += inv[r * 6 + k] * X1[k];
        X[r] = s;
    }
    mat3_vec(Wg, X + 3, v3);                            // Gb = iWgWb*(Wg*X.slice<3,3>() + Wb*Gb)
    mat3_vec(Wb, Gb, w3);
    for (int i = 0; i < 3; i++) v3[i] = v3[i] + w3[i];
    mat3_vec(iWgWb, v3, Gb);
    for (int i = 0; i < 9; i++) Wb[i] = Wg[i] + Wb[i];  // Wb = Wg+Wb
    for (int r = 0; r < 3; r++)
        for (int cc = 0; cc < 3; cc++) Wx[(r + 3) * 6 + cc + 3] += Wg[r * 3 + cc];   // Wx.slice<3,3,3,3>() += Wg
    return RB_OK;
}

// imu_flow.cuh -- the IMU-mode loop body of REBVO::SecondThread (src/rebvo/rebvo_second_t.cpp:146-600 with ImuMode > 0)
// on top of the stage-level entry points.  Included by pipeline.cu.
//
// In IMU mode the per-frame chain contains host algebra between its device stages that the vision-only flow does not
// have (gyro-prior BiasCorrect on 6 x 6 systems, the 7-state scale / gravity / bias filter with its 20 Gauss-Newton steps on
// 11 x 11 matrices): like the reference, that algebra runs on the host (imu_filter.h), so a frame is a sequence of
// stage calls with read-backs, not a captured graph.  The scale space of a push is still built as one batch.
#pragma once
#include <vector>

#include "imu_filter.h"

// the session part of the IMU flow: plain data, which a state blob carries as it is (rb_pipeline_save_state)
struct ImuSession {
    rbimu::ImuFilterHist hist;
    // SecondThread locals (:57-90)
    double V[3], W[3], Pos[3], R[9], Pose[9], Rgva[9], P_V[9], P_W[9];
    double K, Kp, P_Kp;
    long long n_frame;
    double t_prev_grab;   // FirstThr's t0 (:89,296-307)
    // IMUState (include/rebvo/rebvo.h:239-290)
    double Vg[3], P_Vg[9], Bg[3], W_Bg[9], RGiro[9], RGBias[9], Av[3], As[3], X[7], P[49], Qg[9], Qbias[9], Rs[9], g_est[3],
        u_est[3], b_est[3], Posgv[3];
    double Rg;
    bool init;
    int n_giro_init;
    double giro_init[3], g_init[3];
};
struct ImuFlow : ImuSession {
    rb_imu_params ip;
    std::vector<rbimu::ImuSample> samples;   // dataset mode: every sample; live mode: the ring's slots
    rbimu::ImuBuffer buf;
    bool enabled;
    bool live;            // ImuMode=1 (rb_pipeline_set_imu_live): samples arrive through rb_pipeline_push_imu
    double t_last;        // live mode: timestamp of the last sample pushed (-inf before the first)
};

// n rows {t, gyro xyz, accel xyz} of the C interface -> samples
static void imu_rows(const double *rows, int n, rbimu::ImuSample *out) {
    for (int i = 0; i < n; i++) {
        out[i].t = rows[i * 7];
        for (int k = 0; k < 3; k++) {
            out[i].giro[k] = rows[i * 7 + 1 + k];
            out[i].acel[k] = rows[i * 7 + 4 + k];
        }
    }
}

static void imu_eye(double *M, double v) {
    for (int i = 0; i < 9; i++) M[i] = (i % 4 == 0) ? v : 0.0;
}

static void imu_flow_reset(ImuFlow &f) {
    const rb_imu_params &p = f.ip;
    memset(&f.hist, 0, sizeof(f.hist));
    for (int i = 0; i < 3; i++) f.V[i] = f.W[i] = f.Pos[i] = f.Vg[i] = f.Bg[i] = f.Av[i] = f.As[i] = f.Posgv[i] = 0;
    imu_eye(f.R, 1);
    imu_eye(f.Pose, 1);
    imu_eye(f.Rgva, 1);
    imu_eye(f.P_V, 1e50);
    imu_eye(f.P_W, 1e-10);
    f.K = 1;
    f.Kp = 1;
    f.P_Kp = 5e-6;
    f.n_frame = 0;
    f.t_prev_grab = 0;
    imu_eye(f.P_Vg, 1e50);
    imu_eye(f.RGiro, 1);
    imu_eye(f.RGBias, 1);
    imu_eye(f.W_Bg, 1);
    {   // istate.W_Bg=util::Matrix3x3Inv(istate.RGBias*100)  (:70)
        double t[9];
        for (int i = 0; i < 9; i++) t[i] = f.RGBias[i] * 100;
        mat3_inv(t, f.W_Bg);
    }
    imu_eye(f.Qg, p.g_uncert * p.g_uncert);
    f.Rg = p.g_module_uncer * p.g_module_uncer;
    imu_eye(f.Rs, p.AcelMeasStdDev * p.AcelMeasStdDev);
    imu_eye(f.Qbias, p.VBiasStdDev * p.VBiasStdDev);
    const double x0[7] = {M_PI / 4, 0, p.g_module, 0, 0, 0, 0};
    memcpy(f.X, x0, sizeof(x0));
    memset(f.P, 0, sizeof(f.P));
    f.P[0] = p.ScaleStdDevInit * p.ScaleStdDevInit;
    f.P[1 * 7 + 1] = f.P[2 * 7 + 2] = f.P[3 * 7 + 3] = 100;
    f.P[4 * 7 + 4] = f.P[5 * 7 + 5] = f.P[6 * 7 + 6] = p.VBiasStdDev * p.VBiasStdDev * 1e1;
    f.u_est[0] = 1;
    f.u_est[1] = f.u_est[2] = 0;
    for (int i = 0; i < 3; i++) f.g_est[i] = f.b_est[i] = f.giro_init[i] = f.g_init[i] = 0;
    f.init = false;
    f.n_giro_init = 0;
    // (live mode: the ring keeps the samples it has not released and its read position, so the next frame still finds them)
    if (!f.live && !f.samples.empty())
        f.buf.init(f.samples.data(), (int)f.samples.size(), p.use_se3 ? p.Rc2i : nullptr, p.use_se3 ? p.Tc2i : nullptr);
}

// one tracked frame: new = maps[fr % 3] (detected), old = maps[(fr-1) % 3]; returns the nav record and, with odom, the
// odometry record
static int imu_track_frame(rb_pipeline *pl, ImuFlow &f, rb_map *neu, rb_map *old, double t, double dt_frame,
                           const rbimu::ImuIntegral &imu, rb_nav *nav, rb_odometry *odom) {
    rb_ctx *c = pl->c;
    const rb_params &p = pl->p;
    const rb_imu_params &ip = f.ip;
    int r;
    bool est_ok = true;
    int klm_num = 0, fwd = 0;
    // :167-169
    imu_eye(f.P_V, 1e50);
    imu_eye(f.P_W, 1e50);
    imu_eye(f.R, 1);
    double s_rho_q = 1e3;
    if ((r = rb_map_quantile(old, RB_RHO_MIN, RB_RHO_MAX, p.QCutOffQuantile, p.QCutOffNumBins, &s_rho_q))) return r;   // :172
    MapState ns, os;
    if ((r = rb_read_map_state(neu, &ns)) || (r = rb_read_map_state(old, &os))) return r;
    if ((r = rb_map_build_field(neu, p.SearchRange, ns.retuned))) return r;                                            // :177
    // ---- IMU branch (:182-336) --------------------------------------------------------------------------------------------
    if (!f.init && f.n_frame > 0) {
        if (ip.InitBias > 0) {
            for (int i = 0; i < 3; i++) {
                f.giro_init[i] += imu.giro[i] * imu.dt;
                f.g_init[i] -= imu.cacel[i];
            }
            if (++f.n_giro_init > ip.InitBiasFrameNum) {
                for (int i = 0; i < 3; i++) f.Bg[i] = f.giro_init[i] / f.n_giro_init;
                f.init = true;
                double t9[9];
                for (int i = 0; i < 9; i++) t9[i] = f.RGBias[i] * 1e2;
                mat3_inv(t9, f.W_Bg);
                for (int i = 0; i < 3; i++) f.X[1 + i] = f.g_init[i] / f.n_giro_init;
            }
        } else {
            f.init = true;
            for (int i = 0; i < 3; i++) f.Bg[i] = ip.BiasInitGuess[i] * imu.dt;
        }
    }
    memcpy(f.R, imu.Rot, sizeof(f.R));                       // R=new_buf.imu.Rot
    double E[9], RT[9], t9[9];
    so3_exp(f.Bg, E);                                        // R.T()=SO3<>(Bg)*R.T()
    rbimu::transpose(f.R, RT, 3, 3);
    mat3_mul(E, RT, t9);
    rbimu::transpose(t9, f.R, 3, 3);
    rbimu::transpose(f.R, RT, 3, 3);
    if ((r = rb_map_rotate_keylines(old, RT))) return r;     // old_buf.ef->rotate_keylines(R.T())
    if (p.TrackerInitType == 0)
        for (int i = 0; i < 3; i++) f.Vg[i] = 0;
    double score = 0;
    // On an empty old map the reference's Minimizer_V runs iter_max rejected NaN steps: Vel stays as it is and P_Vg
    // becomes NaN.  P_Vg is never read (rebvo_second_t.cpp only writes it), so skipping the call gives the same frame.
    if (os.kn > 0)
        if ((r = rb_minimizer_v(neu, old, f.Vg, f.P_Vg, p.TrackerMatchThresh, p.TrackerIterNum, s_rho_q, p.MatchNumThresh,
                                p.ReweigthDistance, os.retuned, &score)))
            return r;
    if ((r = rb_forward_match(old, neu, &fwd))) return r;
    double W_Xv[36], R_Xv[36], Xv[6];
    int ok = 0;
    if ((r = rb_ext_rot_vel(neu, f.Vg, W_Xv, R_Xv, Xv, p.LocationUncertainty, p.ReweigthDistance, &ok))) return r;
    est_ok = est_ok && ok != 0;
    double Xgv[6], W_Xgv[36];
    memcpy(Xgv, Xv, sizeof(Xgv));
    memcpy(W_Xgv, W_Xv, sizeof(W_Xgv));
    imu_eye(f.RGBias, ip.GiroBiasStdDev * ip.GiroBiasStdDev * dt_frame * dt_frame);
    imu_eye(f.RGiro, ip.GiroMeasStdDev * ip.GiroMeasStdDev * dt_frame * dt_frame);
    double dgbias[3] = {0, 0, 0};
    rb_bias_correct(Xgv, W_Xgv, dgbias, f.W_Bg, f.RGiro, f.RGBias);
    for (int i = 0; i < 3; i++) f.Bg[i] += dgbias[i];
    const double *dVgv = Xgv, *dWgv = Xgv + 3;
    memcpy(f.Rgva, f.R, sizeof(f.R));                        // Rgva=R
    double R0[9];
    so3_exp(dWgv, R0);                                       // SO3<> R0(dWgv); R.T()=R0*R.T()
    rbimu::transpose(f.R, RT, 3, 3);
    mat3_mul(R0, RT, t9);
    rbimu::transpose(t9, f.R, 3, 3);
    double Vgv[3];
    mat3_vec(R0, f.Vg, Vgv);                                 // Vgv=R0*Vg+dVgv
    for (int i = 0; i < 3; i++) Vgv[i] += dVgv[i];
    memcpy(f.V, Vgv, sizeof(Vgv));
    double R_Xgv[36];
    ldlt_inverse<6, false>(W_Xgv, R_Xgv);                    // R_Xgv=Cholesky<6>(W_Xgv).get_inverse(), no zero-pivot stop
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            f.P_V[i * 3 + j] = R_Xgv[i * 6 + j];
            f.P_W[i * 3 + j] = R_Xgv[(3 + i) * 6 + 3 + j];
        }
    // scale / gravity / bias filter (:280-318)
    double vel[3];
    for (int i = 0; i < 3; i++) vel[i] = -Vgv[i] / dt_frame;
    rbimu::est_acel_lsq4(f.hist, vel, f.Av, f.R, dt_frame);
    rbimu::mean_acel4(f.hist, imu.cacel, f.As, f.R);
    double Xgva[6];
    memcpy(Xgva, Xgv, sizeof(Xgva));
    double Rv[9];
    const double dt4 = dt_frame * dt_frame * dt_frame * dt_frame;
    for (int i = 0; i < 9; i++) Rv[i] = f.P_V[i] / dt4;
    double Vgva[3], dWgva[3];
    const double QKp = f.P_Kp;                               // istate.QKp=P_Kp
    if (f.n_frame > 4 + ip.InitBiasFrameNum) {
        f.K = rbimu::est_ka_gmek_bias(f.As, f.Av, 1, f.R, f.X, f.P, f.Qg, f.P_W, f.Qbias, f.P_Kp, f.Rg, f.Rs, Rv, f.g_est,
                                      f.b_est, W_Xgv, Xgva, ip.g_module);
        for (int i = 0; i < 3; i++) dWgva[i] = Xgva[3 + i];
        double R0gva[9];
        so3_exp(dWgva, R0gva);
        rbimu::transpose(f.Rgva, RT, 3, 3);
        mat3_mul(R0gva, RT, t9);
        rbimu::transpose(t9, f.Rgva, 3, 3);
        mat3_vec(R0gva, f.Vg, Vgva);
        for (int i = 0; i < 3; i++) Vgva[i] += Xgva[i];
    } else {
        memcpy(f.Rgva, f.R, sizeof(f.R));
        memcpy(Vgva, Vgv, sizeof(Vgv));
    }
    if ((r = rb_map_rotate_keylines(old, R0))) return r;     // old_buf.ef->rotate_keylines(R0.get_matrix())
    if (odom) {   // :320-334 cf->poses.addFrameMeas(...): relPose from Rgva / Vgva, J_rp_x from R, W_Xgv as BiasCorrect left it
        rb_odometry &o = *odom;
        memset(&o, 0, sizeof(o));
        odom_rel_pose(f.Rgva, Vgva, f.R, W_Xgv, o.relPosPose, o.WrelPosPose);
        for (int i = 0; i < 3; i++) {
            o.AcelMeas[i] = f.As[i];
            o.VisualMeas[i] = f.Av[i];
            o.GMeas[i] = f.g_est[i];
        }
        for (int i = 0; i < 9; i++) {
            o.Rs[i] = f.Rs[i];
            o.Rv[i] = Rv[i];
            o.Rg[i] = f.P[(1 + i / 3) * 7 + 1 + i % 3];   // istate.P.slice<1,1,3,3>()
        }
        o.K = f.K;
        o.WK = 1 / f.P[0];
        o.QK = QKp;
        o.KF_ID = -1;   // cf->kf_list.size()-1 without keyframes (:598)
        o.tracked = 1;
    }
    // ---- common part (:387-487) ---------------------------------------------------------------------------------------------
    bool nan = false;
    for (int i = 0; i < 3; i++) nan = nan || isnan(f.V[i]) || isnan(f.W[i]);
    if (nan) {
        imu_eye(f.P_V, 1e50);
        for (int i = 0; i < 3; i++) f.V[i] = 0;
        f.Kp = 1;
        f.P_Kp = 1e50;
        est_ok = false;
    } else {
        if ((r = rb_directed_matching(neu, old, f.V, f.P_V, f.R, p.MatchThreshModule, p.MatchThreshAngle, (double)p.SearchRange,
                                      p.LocationUncertaintyMatch, &klm_num)))
            return r;
        if (klm_num < p.MatchThreshold) {
            imu_eye(f.P_V, 1e50);
            for (int i = 0; i < 3; i++) f.V[i] = 0;
            f.Kp = 1;
            f.P_Kp = 10;
            est_ok = false;
        } else {
            int rn = 0;
            if ((r = rb_map_regularize(neu, p.RegularizeThresh, &rn))) return r;
            if ((r = rb_map_ekf_update(neu, f.V, p.ReshapeQAbsolute, p.LocationUncertainty))) return r;
            if ((r = rb_map_rescale_opt(neu, RB_RHO_MAX, 1, p.DoReScaling > 0 ? 1 : 0, &f.Kp, &f.P_Kp))) return r;
        }
    }
    // ---- pose (:521-551, IMU variant) ----------------------------------------------------------------------------------------------
    if (f.n_frame > 4 + ip.InitBiasFrameNum) {
        double u[3];
        rbimu::rt_vec(f.Rgva, f.u_est, u);                   // u_est=Rgva.T()*u_est
        const double s = rbimu::dot(u, f.g_est, 3) / rbimu::dot(f.g_est, f.g_est, 3);
        for (int i = 0; i < 3; i++) u[i] = u[i] - s * f.g_est[i];
        const double nu = sqrt(rbimu::dot(u, u, 3));
        for (int i = 0; i < 3; i++) f.u_est[i] = u[i] / nu;
        double P1[9], P2[9], pu[3];
        const double ey[3] = {0, 1, 0}, ex[3] = {1, 0, 0};
        rbimu::so3_from_two(f.g_est, ey, P1);
        mat3_vec(P1, f.u_est, pu);
        rbimu::so3_from_two(pu, ex, P2);
        mat3_mul(P2, P1, f.Pose);                            // Pose=PoseP2*PoseP1
        double pv[3];
        mat3_vec(f.Pose, Vgva, pv);
        for (int i = 0; i < 3; i++) f.Pos[i] += -pv[i] * f.K;
        mat3_vec(f.Pose, Vgv, pv);
        for (int i = 0; i < 3; i++) f.Posgv[i] += -pv[i] * f.K;
    }
    for (int i = 0; i < 9; i++) f.P_V[i] /= dt_frame * dt_frame;
    rb_nav o;
    memset(&o, 0, sizeof(o));
    o.t = t;
    o.dt = dt_frame;
    for (int i = 0; i < 9; i++) {
        o.Rot[i] = f.R[i];
        o.Pose[i] = f.Pose[i];
    }
    so3_ln_of_matrix(f.R, o.RotLie);
    so3_ln_of_matrix(f.Pose, o.PoseLie);
    for (int i = 0; i < 3; i++) {
        o.Vel[i] = (-f.V[i]) * f.K / dt_frame;
        o.Pos[i] = f.Pos[i];
        o.V[i] = f.V[i];
        o.W[i] = f.W[i];
    }
    o.K = f.K;
    o.Kp = f.Kp;
    o.RKp = f.P_Kp;
    o.s_rho_p = s_rho_q;
    o.score = score;
    o.kn = ns.kn;
    o.matches = klm_num;
    o.fwd_matches = fwd;
    o.estimation_ok = est_ok ? 1 : 0;
    o.thresh = ns.thresh_used;
    o.retuned_thresh = ns.retuned;
    *nav = o;
    f.n_frame++;
    return RB_OK;
}

// live mode, before a push enqueues anything: every frame's window (t_prev + TimeDesinc, t + TimeDesinc] must hold a sample
// and end at or before the newest sample, replayed on a copy of the ring.  Where the reference's FirstThr sleeps and grabs again
// (rebvo_first_t.cpp:293-302), the push fails with RB_ERR_STATE and changes nothing; the caller pushes more samples and repeats
// it.  (The reference's failed GrabAndIntegrate also releases the samples before the window; this one releases none.)
static int imu_live_check(rb_pipeline *pl, const ImuFlow &f, const double *ts, int n) {
    rbimu::ImuBuffer probe = f.buf;
    double t0 = f.t_prev_grab;
    for (int i = 0; i < n; i++) {
        if (!probe.release(t0 + f.ip.TimeDesinc, ts[i] + f.ip.TimeDesinc)) {
            snprintf(pl->c->err, sizeof(pl->c->err),
                     "IMU live mode: the samples pushed do not cover frame %d of the push (t=%.6f): push more samples and "
                     "push the frames again", i, ts[i]);
            return RB_ERR_STATE;
        }
        t0 = ts[i];
    }
    return RB_OK;
}

// a push in IMU mode: batched scale space, then frame by frame detect (device chain) + host-driven IMU tracking
// (rgb, frames, fmt as push_impl's)
static int imu_push(rb_pipeline *pl, ImuFlow &f, const uint8_t *rgb, const rb_frame *frames, int fmt, bool on_device,
                    const double *ts, int n, rb_nav *nav_out, rb_odometry *odom_out) {
    rb_ctx *c = pl->c;
    const rb_params &p = pl->p;
    int r;
    if (!on_device && (r = stage_host_frames(pl, rgb, frames, fmt, 0, n, c->stream))) return r;
    if (in_strided(fmt) && (r = write_frame_table(pl, frames, n))) return r;
    pl->sb_pin[0].src = on_device ? (const void *)rgb : (const void *)pl->ws.rgb;
    RB_CUDA(cudaMemcpyAsync(pl->sb_dev, pl->sb_pin, sizeof(SubBatchPtrs), cudaMemcpyHostToDevice, c->stream));
    if ((r = rb_gray_enqueue(c, &pl->ws, pl->und, in_mono(fmt), &pl->sb_dev->src, in_strided(fmt) ? pl->frames_dev : nullptr,
                             n)))
        return r;
    if ((r = rb_dog_build_batch(c, &pl->ws, n))) return r;
    for (int i = 0; i < n; i++) {
        const long long fr = pl->n_pushed + i;
        rb_map *neu = pl->maps[fr % RB_NMAPS], *old = pl->maps[(fr + RB_NMAPS - 1) % RB_NMAPS];
        const float *img0 = pl->ws.img0 + (size_t)i * c->NP, *dog = pl->ws.dog + (size_t)i * c->NP;
        if ((r = rb_detect_enqueue(c, neu, img0, dog, &p.det, pl->chain))) return r;
        if ((r = rb_reestimate_enqueue(c, neu, p.TrackPoints, p.QCutOffNumBins))) return r;
        // FirstThr :296: the gyro / accelerometer samples between the previous frame and this one
        const rbimu::ImuIntegral imu = f.buf.grab(f.t_prev_grab + f.ip.TimeDesinc, ts[i] + f.ip.TimeDesinc);
        if (imu.n <= 0) {
            snprintf(c->err, sizeof(c->err), "IMU mode: no inertial samples between t=%.6f and t=%.6f", f.t_prev_grab, ts[i]);
            return RB_ERR_STATE;
        }
        f.t_prev_grab = ts[i];
        rb_nav *no = nav_out ? nav_out + i : pl->nav_pin + i;
        if (fr == 0) {
            MapState ns;
            if ((r = rb_read_map_state(neu, &ns))) return r;
            memset(no, 0, sizeof(*no));
            no->t = ts[i];
            for (int k = 0; k < 9; k++) no->Rot[k] = no->Pose[k] = (k % 4 == 0) ? 1 : 0;
            no->K = f.K;
            no->Kp = f.Kp;
            no->RKp = f.P_Kp;
            no->kn = ns.kn;
            no->thresh = ns.thresh_used;
            no->retuned_thresh = ns.retuned;
            if (odom_out) memset(odom_out + i, 0, sizeof(rb_odometry));   // tracked = 0
        } else {
            double dt = ts[i] - (i == 0 ? pl->t_prev : ts[i - 1]);
            if (dt < 0.001) dt = 1 / p.config_fps;
            if ((r = imu_track_frame(pl, f, neu, old, ts[i], dt, imu, no, odom_out ? odom_out + i : nullptr))) return r;
        }
    }
    pl->t_prev = ts[n - 1];
    pl->n_pushed += n;
    pl->restored = false;
    return RB_OK;
}

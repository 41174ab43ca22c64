// frame.cuh -- per-frame state of the SecondThread loop (src/rebvo/rebvo_second_t.cpp) kept in device memory, and the
// scalar glue between its stages as device functions, so that they can run either as one-thread kernels or folded
// into the neighbouring kernel's first / last block (each fold removes one launch from the per-frame dependency chain).
#pragma once
#include "common.cuh"
#include "tracker.cuh"
#include "lm.cuh"

struct FrameState {
    double V[3], W[3], Pos[3];
    double R[9], Pose[9];
    double P_V[9], P_W[9];
    double Kp, K, P_Kp;
    double VW[6];       // minimiser priors (V, W of the previous frame)
    double R0[9];       // forward rotation exp(W)
    DMatchArgs dm;
    int do_match, do_map, est_ok;
    int klm_num;
    int n_frame;
    int pose_done;      // d_frame_pose already integrated this frame's pose (cleared by d_frame_finish)
    double RotLie[3], PoseLie[3];   // its logarithms for the nav record
};

__device__ __forceinline__ void d_eye(double *M, double v) {
    for (int i = 0; i < 9; i++) M[i] = 0;
    M[0] = M[4] = M[8] = v;
}

// per-frame scalars that change from push to push; kept in device memory so that the kernel arguments of a batch
// are constant and the whole batch can be replayed as one CUDA graph
struct FrameArgs {
    double t, dt;
    unsigned int frame_count;   // global_tracker::FrameCount of the reference ring slot serving this frame
    unsigned int next_frame_count;   // ... and of the slot serving the NEXT frame (its loop-body start may be folded into this
                                     // frame's last kernel, before the next push's arguments exist)
};

// start of the SecondThread loop body (:167-169) + minimiser priors
__device__ __forceinline__ void d_frame_pre(FrameState *fs, unsigned int frame_count, MapState *nst) {
    nst->frame_count = frame_count;
    nst->fwd_match = 0;   // counters of FordwardMatch / directed_matching / Regularize_1_iter
    nst->nmatch = 0;
    nst->reg_num = 0;
    d_eye(fs->P_V, 1e50);
    d_eye(fs->P_W, 1e50);
    d_eye(fs->R, 1);
    for (int i = 0; i < 3; i++) {
        fs->VW[i] = fs->V[i];
        fs->VW[3 + i] = fs->W[i];
    }
    fs->est_ok = 1;
    fs->do_match = 0;
    fs->do_map = 0;
    fs->klm_num = 0;
}

// after Minimizer_RV (:346-398): outputs, R0 = exp(W), R.T() = R0*R.T(), NaN guard, directed-matching args.  Two parts:
// the first needs only Vel / W0, so the cluster minimiser runs it beside lm_finalize_cov; the second needs RVel / RW0.
__device__ __forceinline__ void d_frame_post_min_pose(FrameState *fs, const LMState &lm) {
    if (!lm.no_keylines) {                  // (an empty old map leaves V, W, P_V, P_W as they were, global_tracker.cpp:601)
        for (int i = 0; i < 3; i++) {
            fs->V[i] = lm.Vel[i];
            fs->W[i] = lm.W0[i];
        }
    }
    so3_exp(fs->W, fs->R0);                 // SO3<> R0(W)
    double Rt[9], RtT[9];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) RtT[r * 3 + c] = fs->R[c * 3 + r];
    mat3_mul(fs->R0, RtT, Rt);              // R.T() = R0*R.T()
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) fs->R[r * 3 + c] = Rt[c * 3 + r];
    bool nan = false;
    for (int i = 0; i < 3; i++) nan = nan || isnan(fs->V[i]) || isnan(fs->W[i]);
    if (nan) {                              // :387-398 (P_V=1e50 in the second part)
        for (int i = 0; i < 3; i++) fs->V[i] = 0;
        fs->Kp = 1;
        fs->P_Kp = 1e50;
        fs->est_ok = 0;
        fs->do_match = 0;
    } else {
        fs->do_match = 1;
        // directed_matching prologue (edge_tracker.cpp:324-325): Vel=BackRot*Vel (RVel in the second part)
        mat3_vec(fs->R, fs->V, fs->dm.Vel);
        for (int i = 0; i < 9; i++) fs->dm.BackRot[i] = fs->R[i];
    }
}
// reads what the first part wrote: R, and do_match = no NaN
__device__ __forceinline__ void d_frame_post_min_cov(FrameState *fs, const LMState &lm) {
    if (!lm.no_keylines)
        for (int i = 0; i < 9; i++) {
            fs->P_V[i] = lm.RVel[i];
            fs->P_W[i] = lm.RW0[i];
        }
    if (!fs->do_match) {
        d_eye(fs->P_V, 1e50);
    } else {   // RVel=BackRot*RVel*BackRot.T()
        double t[9];
        mat3_mul(fs->R, fs->P_V, t);
        mat3_mul_bt(t, fs->R, fs->dm.RVel);
    }
}
__device__ __forceinline__ void d_frame_post_min(FrameState *fs, const LMState &lm) {
    d_frame_post_min_pose(fs, lm);
    d_frame_post_min_cov(fs, lm);
}

// after directed_matching (:410-423)
__device__ __forceinline__ void d_frame_post_match(FrameState *fs, const MapState *nst, int match_threshold) {
    if (!fs->do_match) {
        fs->do_map = 0;
        return;
    }
    fs->klm_num = nst->nmatch;
    if (fs->klm_num < match_threshold) {
        d_eye(fs->P_V, 1e50);
        for (int i = 0; i < 3; i++) fs->V[i] = 0;
        fs->Kp = 1;
        fs->P_Kp = 10;
        fs->est_ok = 0;
        fs->do_map = 0;
    } else {
        fs->do_map = 1;
    }
}

// pose integration + NavData (:545-585)
// pose integration of the frame (:545-551: Pose=Pose*R, Pos+=-Pose*V*K) and the two matrix logarithms of the nav record: the
// serial part of d_frame_finish that needs nothing of the map update.  The pipeline runs it in a spare thread of the
// regularise / EKF kernel (after the match-count gate has fixed V), so that the map-update kernel's one-thread tail is short.
__device__ __forceinline__ void d_frame_pose(FrameState *fs) {
    const double K = fs->K;
    double Pose[9];
    mat3_mul(fs->Pose, fs->R, Pose);          // Pose=Pose*R
    for (int i = 0; i < 9; i++) fs->Pose[i] = Pose[i];
    double nP[9], pv[3];
    for (int i = 0; i < 9; i++) nP[i] = -Pose[i];
    mat3_vec(nP, fs->V, pv);                  // Pos+=-Pose*V*K
    for (int i = 0; i < 3; i++) fs->Pos[i] = fs->Pos[i] + pv[i] * K;
    so3_ln_of_matrix(fs->R, fs->RotLie);
    so3_ln_of_matrix(fs->Pose, fs->PoseLie);
    fs->pose_done = 1;
}

// rescaled = false: the map's EstimateReScalingOpt has not run yet.  With DoReScaling=0 its Kp / RKp reach nothing but this
// record (every frame sets Kp afresh: NaN guard, match-count restart or rescaling), so the pipeline runs it on a side
// stream, which fills in the record's Kp / RKp when do_map is set; FrameState keeps the value of the last restart.
__device__ __forceinline__ void d_frame_finish(FrameState *fs, const MapState *nst, const MapState *ost,
                                               double lm_score, rb_nav *nav, const FrameArgs *fa, bool rescaled) {
    const double t = fa->t, dt_frame = fa->dt;
    if (rescaled && fs->do_map) {
        fs->Kp = nst->Kp;      // Kp=EstimateReScalingOpt(P_Kp,...)
        fs->P_Kp = nst->RKp;
    }
    const double K = fs->K;
    if (!fs->pose_done) d_frame_pose(fs);
    fs->pose_done = 0;
    rb_nav o;
    o.t = t;
    o.dt = dt_frame;
    for (int i = 0; i < 9; i++) {
        o.Rot[i] = fs->R[i];
        o.Pose[i] = fs->Pose[i];
    }
    for (int i = 0; i < 3; i++) {
        o.RotLie[i] = fs->RotLie[i];
        o.PoseLie[i] = fs->PoseLie[i];
        o.Vel[i] = (-fs->V[i]) * K / dt_frame;
        o.Pos[i] = fs->Pos[i];
        o.V[i] = fs->V[i];
        o.W[i] = fs->W[i];
    }
    o.K = K;
    o.Kp = fs->Kp;
    o.RKp = fs->P_Kp;
    o.s_rho_p = ost->s_rho_q;
    o.score = lm_score;
    o.kn = nst->kn;
    o.matches = fs->klm_num;
    o.fwd_matches = nst->fwd_match;
    o.estimation_ok = fs->est_ok;
    o.thresh = nst->thresh_used;
    o.retuned_thresh = nst->retuned;
    *nav = o;
    for (int i = 0; i < 9; i++) fs->P_V[i] = fs->P_V[i] / (dt_frame * dt_frame);   // P_V/=dt_frame*dt_frame
    fs->n_frame++;
}


// capi_track.cu -- stage-level C ABI of the tracker / mapper (include/rebvo_b200.h): thin synchronous
// wrappers that stage scalar arguments in device memory, enqueue the kernels of tracker.cu and read the
// scalar results back.  The per-frame flow (pipeline.cu) calls the *_enqueue functions directly and never
// synchronises between stages.
#include <math.h>

#include "common.cuh"
#include "tracker.cuh"
#include "frame.cuh"

int rb_try_vel_rot_enqueue(rb_ctx *c, rb_map *fmap, rb_map *old, const double X[6], int reweight, int procjf,
                           double match_thresh, double s_rho_min, unsigned int mnt, unsigned int fc, double k_huber,
                           double *tot_dev);

static double *args_dev(rb_ctx *c) { return (double *)((char *)c->dev_small + RB_DS_ARGS); }
static double *args_pin(rb_ctx *c) { return (double *)((char *)c->pinned + RB_DS_ARGS); }

static int stage_in(rb_ctx *c, const double *src, int n, int off) {
    memcpy(args_pin(c) + off, src, sizeof(double) * n);
    RB_CUDA(cudaMemcpyAsync(args_dev(c) + off, args_pin(c) + off, sizeof(double) * n, cudaMemcpyHostToDevice,
                            c->stream));
    return RB_OK;
}

extern "C" int rb_map_quantile(rb_map *m, double s_rho_min, double s_rho_max, double percentile, int nbins,
                               double *out) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    int r = rb_quantile_enqueue(m->c, m, s_rho_min, s_rho_max, percentile, nbins);
    if (r) return r;
    MapState s;
    if ((r = rb_read_map_state(m, &s))) return r;
    if (out) *out = s.s_rho_q;
    return RB_OK;
}

extern "C" int rb_map_build_field(rb_map *m, int radius, float min_mod) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    int r = rb_build_field_enqueue(m->c, m, radius, min_mod, false);
    if (r) return r;
    return rb_ctx_sync(m->c);
}

__global__ void k_field_unpack(const unsigned long long *__restrict__ f, int2 *__restrict__ out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = f[i];
    int2 o;
    if (k == ~0ull) {
        o.x = 0;
        o.y = -1;
    } else {
        o.x = (int)(k >> 32);
        o.y = (int)(0xFFFFFFFFu - (unsigned int)(k & 0xFFFFFFFFull));
    }
    out[i] = o;
}

extern "C" int rb_map_get_field(rb_map *m, int32_t *out) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    int2 *tmp = nullptr;
    RB_CUDA(cudaMalloc(&tmp, sizeof(int2) * (size_t)c->N));
    k_field_unpack<<<(unsigned)((c->N + 255) / 256), 256, 0, c->stream>>>(m->field, tmp, (size_t)c->N);
    c->launches++;
    cudaError_t e = cudaMemcpyAsync(out, tmp, sizeof(int2) * (size_t)c->N, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    cudaFree(tmp);
    if (e != cudaSuccess) {
        snprintf(c->err, sizeof(c->err), "get_field: %s", cudaGetErrorString(e));
        return RB_ERR_CUDA;
    }
    return RB_OK;
}

extern "C" int rb_map_set_frame_count(rb_map *m, uint32_t fc) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    RB_CUDA(cudaMemcpyAsync(&m->st->frame_count, &fc, sizeof(fc), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

extern "C" int rb_try_vel_rot(rb_map *fmap, rb_map *old, const double X[6], int reweight, int procjf,
                              double match_thresh, double s_rho_min, uint32_t match_num_thresh, double k_huber,
                              const double *res_in, double *res_out, double JtJ[36], double JtF[6], double *score) {
    if (!fmap || !old) return RB_ERR_ARG;
    RB_ENTER(fmap->c);
    rb_ctx *c = fmap->c;
    MapState so, sf;
    int r;
    if ((r = rb_read_map_state(old, &so))) return r;
    if ((r = rb_read_map_state(fmap, &sf))) return r;
    if (res_in && so.kn > 0)
        RB_CUDA(cudaMemcpyAsync(fmap->res[0], res_in, sizeof(double) * so.kn, cudaMemcpyHostToDevice, c->stream));
    else
        RB_CUDA(cudaMemsetAsync(fmap->res[0], 0, sizeof(double) * (size_t)c->kcap, c->stream));
    if ((r = rb_try_vel_rot_enqueue(c, fmap, old, X, reweight, procjf, match_thresh, s_rho_min, match_num_thresh,
                                    sf.frame_count, k_huber, args_dev(c))))
        return r;
    RB_CUDA(cudaMemcpyAsync(args_pin(c), args_dev(c), sizeof(double) * 28, cudaMemcpyDeviceToHost, c->stream));
    if (res_out && so.kn > 0)
        RB_CUDA(cudaMemcpyAsync(res_out, fmap->res[1], sizeof(double) * so.kn, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    const double *s = args_pin(c);
    if (procjf) {   // JtJ upper triangle and JtF, their sign fix-ups and the symmetric fill (:484-490, :492-496)
        double J[36], F[6];
        int k = 0;
        for (int a = 0; a < 6; a++)
            for (int b = a; b < 6; b++) J[a * 6 + b] = s[k++];
        for (int a = 0; a < 6; a++) F[a] = s[21 + a];
        for (int a = 0; a < 2; a++) {
            F[a + 2] = -F[a + 2];
            for (int b = 0; b < 2; b++) {
                J[(a + 0) * 6 + (b + 2)] = -J[(a + 0) * 6 + (b + 2)];
                J[(a + 2) * 6 + (b + 4)] = -J[(a + 2) * 6 + (b + 4)];
            }
        }
        for (int a = 0; a < 6; a++)
            for (int b = a + 1; b < 6; b++) J[b * 6 + a] = J[a * 6 + b];
        if (JtJ) memcpy(JtJ, J, sizeof(J));
        if (JtF) memcpy(JtF, F, sizeof(F));
    }
    if (score) *score = s[27];
    return RB_OK;
}

// Minimizer_RV; forward: as the per-frame pipeline runs it, with a scratch FrameState (so that the last evaluation offers
// the old keylines to fmap's FordwardMatch arg-max), then FordwardMatch's apply
static int minimizer_rv(rb_map *fmap, rb_map *old, double V[3], double W[3], double RVel[9], double RW0[9],
                        double match_thresh, int iter_max, int init_type, double reweight_distance, double *rel_error,
                        double *rel_error_score, double max_s_rho, uint32_t match_num_thresh, int init_iter,
                        double W_X[36], double *score, bool forward, int *fwd_nmatch) {
    if (!fmap || !old) return RB_ERR_ARG;
    RB_ENTER(fmap->c);
    rb_ctx *c = fmap->c;
    int r;
    double vw[6] = {V[0], V[1], V[2], W[0], W[1], W[2]};
    if ((r = stage_in(c, vw, 6, 0))) return r;
    rb_minimizer_args a;
    a.match_thresh = match_thresh;
    a.iter_max = iter_max;
    a.init_type = init_type;
    a.init_iter = init_iter;
    a.reweight_distance = reweight_distance;
    a.match_num_thresh = match_num_thresh;
    FrameState *fs = nullptr;
    if (forward) {   // the frame state as the loop-body start (d_frame_pre) leaves it
        FrameState h;
        memset(&h, 0, sizeof(h));
        for (int i = 0; i < 9; i += 4) {
            h.R[i] = 1;
            h.P_V[i] = h.P_W[i] = 1e50;
        }
        memcpy(h.VW, vw, sizeof(vw));
        h.est_ok = 1;
        RB_CUDA(cudaMalloc(&fs, sizeof(FrameState)));
        cudaError_t e = cudaMemcpy(fs, &h, sizeof(h), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemsetAsync(&fmap->st->fwd_match, 0, sizeof(int), c->stream);
        if (e != cudaSuccess) {
            cudaFree(fs);
            snprintf(c->err, sizeof(c->err), "minimizer_rv_forward: %s", cudaGetErrorString(e));
            return RB_ERR_CUDA;
        }
        r = rb_forward_match_init_enqueue(c, fmap);
    }
    // operands staged as the per-frame pipeline stages them (REBVO_B200_MIN_EARLY, default on): the copy of V / W above is
    // the stream's last operation, so no kernel that writes the old map can still be running when they are read
    c->min_early = getenv("REBVO_B200_MIN_EARLY") ? atoi(getenv("REBVO_B200_MIN_EARLY")) != 0 : true;
    if (!r) r = rb_minimizer_enqueue(c, fmap, old, args_dev(c), &a, max_s_rho, false, 0, true, fs);
    c->min_early = false;
    if (!r && forward) r = rb_forward_match_apply_enqueue(c, old, fmap);
    LMState *lmh = (LMState *)((char *)c->pinned + 4096);
    if (!r) {
        const cudaError_t e = cudaMemcpyAsync(lmh, &fmap->ts->lm, sizeof(LMState), cudaMemcpyDeviceToHost, c->stream);
        if (e != cudaSuccess) {
            snprintf(c->err, sizeof(c->err), "minimizer_rv: %s", cudaGetErrorString(e));
            r = RB_ERR_CUDA;
        }
    }
    if (!r) r = rb_minimizer_check_abort(c, fmap);   // (synchronises)
    if (fs) cudaFree(fs);
    if (r) return r;
    if (forward) {
        MapState s;
        if ((r = rb_read_map_state(fmap, &s))) return r;
        if (fwd_nmatch) *fwd_nmatch = s.fwd_match;
    }
    if (lmh->no_keylines) {   // "if(klist.KNum()<=0) return 0;": every output keeps the caller's value
        if (score) *score = 0;
        return RB_OK;
    }
    memcpy(V, lmh->Vel, sizeof(double) * 3);
    memcpy(W, lmh->W0, sizeof(double) * 3);
    if (RVel) memcpy(RVel, lmh->RVel, sizeof(double) * 9);
    if (RW0) memcpy(RW0, lmh->RW0, sizeof(double) * 9);
    if (W_X) memcpy(W_X, lmh->W_X, sizeof(double) * 36);
    if (rel_error) *rel_error = lmh->rel_error;
    if (rel_error_score) *rel_error_score = lmh->rel_error_score;
    if (score) *score = lmh->score;
    return RB_OK;
}

extern "C" int rb_minimizer_rv(rb_map *fmap, rb_map *old, double V[3], double W[3], double RVel[9], double RW0[9],
                               double match_thresh, int iter_max, int init_type, double reweight_distance,
                               double *rel_error, double *rel_error_score, double max_s_rho,
                               uint32_t match_num_thresh, int init_iter, double W_X[36], double *score) {
    return minimizer_rv(fmap, old, V, W, RVel, RW0, match_thresh, iter_max, init_type, reweight_distance, rel_error,
                        rel_error_score, max_s_rho, match_num_thresh, init_iter, W_X, score, false, nullptr);
}

extern "C" int rb_minimizer_rv_forward(rb_map *fmap, rb_map *old, double V[3], double W[3], double RVel[9],
                                       double RW0[9], double match_thresh, int iter_max, int init_type,
                                       double reweight_distance, double *rel_error, double *rel_error_score,
                                       double max_s_rho, uint32_t match_num_thresh, int init_iter, double W_X[36],
                                       double *score, int *fwd_nmatch) {
    return minimizer_rv(fmap, old, V, W, RVel, RW0, match_thresh, iter_max, init_type, reweight_distance, rel_error,
                        rel_error_score, max_s_rho, match_num_thresh, init_iter, W_X, score, true, fwd_nmatch);
}

extern "C" int rb_forward_match(rb_map *old, rb_map *neu, int *nmatch) {
    if (!old || !neu) return RB_ERR_ARG;
    RB_ENTER(old->c);
    // *nmatch counts this call's matches: a pipeline context leaves the counter to its per-frame kernel, which the IMU
    // flow (the caller inside a pipeline) does not run, so the count would add up over the frames that reuse neu
    rb_ctx *c = old->c;
    RB_CUDA(cudaMemsetAsync(&neu->st->fwd_match, 0, sizeof(int), c->stream));
    int r = rb_forward_match_enqueue(c, old, neu);
    if (r) return r;
    MapState s;
    if ((r = rb_read_map_state(neu, &s))) return r;
    if (nmatch) *nmatch = s.fwd_match;
    return RB_OK;
}

extern "C" int rb_map_rotate_keylines(rb_map *m, const double R[9]) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    int r;
    if ((r = stage_in(c, R, 9, 16))) return r;
    if ((r = rb_rotate_enqueue(c, m, args_dev(c) + 16))) return r;
    return rb_ctx_sync(c);
}

// directed_matching's prologue (edge_tracker.cpp:324-325): Vel=BackRot*Vel; RVel=BackRot*RVel*BackRot.T(), TooN dot order
static void dm_args(const double Vel[3], const double RVel[9], const double BackRot[9], DMatchArgs &a) {
    for (int i = 0; i < 3; i++) {
        double s = 0;
        for (int k = 0; k < 3; k++) s += BackRot[i * 3 + k] * Vel[k];
        a.Vel[i] = s;
    }
    double t[9];
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += BackRot[i * 3 + k] * RVel[k * 3 + j];
            t[i * 3 + j] = s;
        }
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double s = 0;
            for (int k = 0; k < 3; k++) s += t[i * 3 + k] * BackRot[j * 3 + k];
            a.RVel[i * 3 + j] = s;
        }
    memcpy(a.BackRot, BackRot, sizeof(double) * 9);
}

extern "C" int rb_directed_matching(rb_map *neu, rb_map *old, const double Vel[3], const double RVel[9],
                                    const double BackRot[9], double min_thr_mod, double min_thr_ang,
                                    double max_radius, double loc_uncertainty, int *nmatch) {
    if (!neu || !old) return RB_ERR_ARG;
    RB_ENTER(neu->c);
    rb_ctx *c = neu->c;
    DMatchArgs a;
    dm_args(Vel, RVel, BackRot, a);
    int r;
    if ((r = stage_in(c, (const double *)&a, sizeof(a) / sizeof(double), 32))) return r;
    if ((r = rb_directed_matching_enqueue(c, neu, old, (const DMatchArgs *)(args_dev(c) + 32), min_thr_mod,
                                          min_thr_ang, max_radius, loc_uncertainty, nullptr)))
        return r;
    MapState s;
    if ((r = rb_read_map_state(neu, &s))) return r;
    if (nmatch) *nmatch = s.nmatch;
    return RB_OK;
}

extern "C" int rb_map_regularize(rb_map *m, double thresh, int *r_num) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    int r = rb_regularize_enqueue(m->c, m, thresh, nullptr);
    if (r) return r;
    MapState s;
    if ((r = rb_read_map_state(m, &s))) return r;
    if (r_num) *r_num = s.reg_num;
    return RB_OK;
}

extern "C" int rb_map_ekf_update(rb_map *m, const double vel[3], double reshape_q_abs, double loc_uncertainty) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    int r;
    if ((r = stage_in(c, vel, 3, 64))) return r;
    if ((r = rb_ekf_enqueue(c, m, args_dev(c) + 64, reshape_q_abs, loc_uncertainty, nullptr))) return r;
    return rb_ctx_sync(c);
}

extern "C" int rb_map_rescale_opt(rb_map *m, double s_rho_min, uint32_t match_num_min, int re_escale, double *Kp,
                                  double *RKp) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    int r = rb_rescale_enqueue(m->c, m, s_rho_min, match_num_min, re_escale, nullptr);
    if (r) return r;
    MapState s;
    if ((r = rb_read_map_state(m, &s))) return r;
    if (Kp) *Kp = s.Kp;
    if (RKp) *RKp = s.RKp;
    return RB_OK;
}

extern "C" int rb_map_match_update(rb_map *neu, rb_map *old, const double V[3], const double P_V[9],
                                   const double BackRot[9], const double R0[9], int do_match, double min_thr_mod,
                                   double min_thr_ang, double max_radius, double loc_uncertainty_match,
                                   int match_threshold, double reg_thresh, double reshape_q_abs, double loc_uncertainty,
                                   double Pose_io[9], double Pos_io[3], double K, rb_match_update_out *out) {
    if (!neu || !old || !out) return RB_ERR_ARG;
    RB_ENTER(neu->c);
    rb_ctx *c = neu->c;
    // the frame state the pipeline's chain reads: directed_matching's arguments, R0, the gate's inputs and the pose
    FrameState h;
    memset(&h, 0, sizeof(h));
    dm_args(V, P_V, BackRot, h.dm);
    memcpy(h.V, V, sizeof(double) * 3);
    memcpy(h.P_V, P_V, sizeof(double) * 9);
    memcpy(h.R, BackRot, sizeof(double) * 9);
    memcpy(h.R0, R0, sizeof(double) * 9);
    memcpy(h.Pose, Pose_io, sizeof(double) * 9);
    memcpy(h.Pos, Pos_io, sizeof(double) * 3);
    h.K = K;
    h.do_match = do_match ? 1 : 0;
    h.est_ok = 1;
    FrameState *fs = nullptr;
    RB_CUDA(cudaMalloc(&fs, sizeof(FrameState)));
    int r = RB_OK;
    cudaError_t e = cudaMemcpy(fs, &h, sizeof(h), cudaMemcpyHostToDevice);
    // the counters the pipeline's loop-body start (d_frame_pre) zeroes
    if (e == cudaSuccess) e = cudaMemsetAsync(&neu->st->nmatch, 0, 3 * sizeof(int), c->stream);
    if (e != cudaSuccess) r = RB_ERR_CUDA;
    // FordwardMatch's arg-max over old's m_id_f (in the pipeline: the minimiser's last evaluation)
    if (!r) r = rb_forward_match_init_enqueue(c, neu);
    if (!r) r = rb_forward_match_argmax_enqueue(c, old, neu);
    if (!r)
        r = rb_match_enqueue(c, neu, old, &fs->dm, fs->R0, min_thr_mod, min_thr_ang, max_radius, loc_uncertainty_match,
                             &fs->do_match);
    if (!r)
        r = rb_reg_ekf_enqueue(c, neu, old, reg_thresh, fs, match_threshold, reshape_q_abs, loc_uncertainty, fs->R0,
                               nullptr, nullptr, nullptr);
    if (!r) {
        e = cudaMemcpyAsync(&h, fs, sizeof(h), cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) r = RB_ERR_CUDA;
    }
    cudaFree(fs);
    if (e != cudaSuccess) snprintf(c->err, sizeof(c->err), "map_match_update: %s", cudaGetErrorString(e));
    if (r) return r;
    MapState s;
    if ((r = rb_read_map_state(neu, &s))) return r;
    out->nmatch = s.nmatch;
    out->fwd_match = s.fwd_match;
    out->reg_num = s.reg_num;
    out->do_map = h.do_map;
    out->est_ok = h.est_ok;
    out->klm_num = h.klm_num;
    memcpy(out->V, h.V, sizeof(out->V));
    out->Kp = h.Kp;
    out->P_Kp = h.P_Kp;
    memcpy(out->P_V, h.P_V, sizeof(out->P_V));
    memcpy(out->Pose, h.Pose, sizeof(out->Pose));
    memcpy(out->Pos, h.Pos, sizeof(out->Pos));
    memcpy(out->RotLie, h.RotLie, sizeof(out->RotLie));
    memcpy(out->PoseLie, h.PoseLie, sizeof(out->PoseLie));
    memcpy(Pose_io, h.Pose, sizeof(double) * 9);
    memcpy(Pos_io, h.Pos, sizeof(double) * 3);
    return RB_OK;
}

// tracker.cuh -- device-resident state of global_tracker::Minimizer_RV and entry points of tracker.cu
#pragma once
#include "common.cuh"

enum LMStep {
    STEP_NONE = 0,
    STEP_INIT_FIRST_ZERO,   // first evaluation of the zero-initialised try   (global_tracker.cpp:651-653)
    STEP_INIT_ITER_ZERO,    // an init iteration that still needs Jacobians  (:657-683)
    STEP_INIT_LAST_ZERO,    // last init iteration, score only; then set up the prior-initialised try (:686-700)
    STEP_INIT_FIRST_PRIOR,  // (:700-704)
    STEP_INIT_ITER_PRIOR,   // (:706-732)
    STEP_INIT_LAST_PRIOR,   // + pick the better start and swap the residual buffers (:734-747)
    STEP_MAIN_FIRST,        // first re-weighted evaluation (:755-757)
    STEP_MAIN_ITER,         // LM iteration with Cholesky solve (:760-791)
    STEP_MAIN_LAST          // last iteration + uncertainties / outputs (:793-816)
};

// control block of the cluster Minimizer_RV kernel (min_cluster.cuh), one per TrackState, in device memory
struct MinCtl {
    unsigned int gen;              // base of the slot sequence numbers of the next minimisation
    int abort;                     // an exchange timed out (results are NaN); read and cleared by rb_minimizer_check_abort
};

// FordwardMatch's arg-max record of one new keyline: the lexicographic maximum of (dbl_key(rho), index) over the old
// keylines that matched it; {0, -1} = none (written by rb_forward_match_init_enqueue)
struct __align__(16) FmBest {
    unsigned long long key;
    long long idx;
};

int rb_minimizer_cluster_setup(rb_ctx *c);
// reads (and clears) the abort flag of a map's minimiser; returns RB_ERR_CUDA with a message when it was set.  Synchronises.
int rb_minimizer_check_abort(rb_ctx *c, rb_map *fmap);
int rb_track_state_alloc(rb_ctx *c, rb_map *m);
void rb_track_state_free(rb_map *m);

struct rb_minimizer_args {
    double match_thresh;
    int iter_max, init_type, init_iter;
    double reweight_distance;
    unsigned int match_num_thresh;
};

// Enqueue the whole Minimizer_RV on c->stream.  Vel/W0 priors are read from dev pointers VW_dev[6]
// (V then W); max_s_rho is read from old->st->s_rho_q when s_rho_from_state, else from the argument.
// The optional FrameState / FrameArgs / rb_nav arguments below belong to the per-frame pipeline (frame.cuh): when given,
// the one-thread glue stage next to the kernel runs inside it instead of as its own launch.
// rb_minimizer_enqueue with post_fs: the stage after the minimiser (d_frame_post_min) and FordwardMatch's arg-max of old
// into fmap (its scratch cleared before by rb_forward_match_init_enqueue) run inside it.
struct FrameState;
struct FrameArgs;
int rb_minimizer_enqueue(rb_ctx *c, rb_map *fmap, rb_map *old, const double *VW_dev,
                         const rb_minimizer_args *a, double max_s_rho, bool s_rho_from_state,
                         unsigned int frame_count, bool frame_count_from_state, FrameState *post_fs = nullptr);
int rb_quantile_enqueue(rb_ctx *c, rb_map *m, double smin, double smax, double perc, int nbins,
                        FrameState *fs = nullptr, const unsigned int *frame_count_dev = nullptr, MapState *nst = nullptr);
int rb_build_field_enqueue(rb_ctx *c, rb_map *m, int radius, float min_mod, bool min_mod_from_state);
// FordwardMatch = init (clears neu's arg-max scratch) -> arg-max (m_id_f of old) -> apply (copies each winner into neu);
// rb_forward_match_enqueue is the whole stage.
int rb_forward_match_init_enqueue(rb_ctx *c, rb_map *neu);
int rb_forward_match_argmax_enqueue(rb_ctx *c, rb_map *old, rb_map *neu);
int rb_forward_match_apply_enqueue(rb_ctx *c, rb_map *old, rb_map *neu);
int rb_forward_match_enqueue(rb_ctx *c, rb_map *old, rb_map *neu);
int rb_rotate_enqueue(rb_ctx *c, rb_map *m, const double *R_dev);
struct DMatchArgs {       // device-resident arguments of directed_matching (after the back-rotation)
    double Vel[3];        // BackRot*Vel
    double RVel[9];       // BackRot*RVel*BackRot^T
    double BackRot[9];
};
int rb_directed_matching_enqueue(rb_ctx *c, rb_map *neu, rb_map *old, const DMatchArgs *args_dev,
                                 double min_thr_mod, double min_thr_ang, double max_radius,
                                 double loc_uncertainty, const int *enable_dev);
int rb_regularize_enqueue(rb_ctx *c, rb_map *m, double thresh, const int *enable_dev);
struct rb_nav;
// The per-frame map chain of two kernels, with the old map rotated last.  rb_match_enqueue: FordwardMatch's apply (the
// arg-max of neu is complete) and directed_matching against the unrotated old map, each probed keyline rotated by R_dev;
// the matched (rho, s_rho) of every keyline go to neu's regularisation scratch.  rb_reg_ekf_enqueue: the match-count
// gate, Regularize_1_iter from that scratch, the EKF, rotate_keylines(R_dev) of old, and with nav the frame's nav record
// (except Kp / RKp of a mapped frame, which rb_rescale_enqueue fills in); with odom the frame's odometry record (d_frame_odometry).
int rb_match_enqueue(rb_ctx *c, rb_map *neu, rb_map *old, const DMatchArgs *args_dev, const double *R_dev,
                     double min_thr_mod, double min_thr_ang, double max_radius, double loc_uncertainty,
                     const int *do_match_dev);
int rb_reg_ekf_enqueue(rb_ctx *c, rb_map *m, rb_map *old, double thresh, FrameState *fs, int match_threshold,
                       double q_abs, double loc_unc, const double *R_dev, rb_nav *nav, const FrameArgs *fa,
                       rb_odometry *odom);
int rb_map_update_enqueue(rb_ctx *c, rb_map *m, double s_rho_min, unsigned int match_num_min, int re_escale, FrameState *fs,
                          const MapState *ost, rb_nav *nav, const FrameArgs *fa);
int rb_ekf_enqueue(rb_ctx *c, rb_map *m, const double *vel_dev, double q_abs, double loc_unc,
                   const int *enable_dev);
int rb_rescale_enqueue(rb_ctx *c, rb_map *m, double s_rho_min, unsigned int match_num_min, int re_escale,
                       const int *enable_dev, rb_nav *kp_nav = nullptr);
int rb_read_map_state(rb_map *m, MapState *host);

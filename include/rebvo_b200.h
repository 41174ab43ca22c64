/* rebvo_b200.h -- C ABI of librebvo_b200.so: the H100 (sm_90a) implementation of REBVO's per-frame
 * edge pipeline (DoG edge detector + keyline extraction, edge-map tracker / SE(3) minimiser, per-keyline
 * inverse-depth EKF).
 *
 * The reference (JuanTarrio/rebvo) has no FFI: its hot path is a set of C++ classes called directly by
 * REBVO::FirstThr (src/rebvo/rebvo_first_t.cpp:259-272) and REBVO::SecondThread
 * (src/rebvo/rebvo_second_t.cpp:172-487).  Each entry point below replaces one of those calls; the
 * comment on each cites the reference method it stands for.  Host shim classes with the reference's own
 * names/signatures (include/rebvo_b200_shim.hpp) forward to these functions, see INTEGRATION.md.
 *
 * Conventions: every function returns 0 on success, a negative rb_status otherwise, and never throws.
 * A CUDA failure is sticky per context (rb_last_error()).  Pointers are plain host pointers unless the
 * name says dev.  Images are row-major without stride (Image<T>, include/VideoLib/image.h:42-217), except the rb_frame
 * ones of rb_pipeline_push_frames, which have a row step.
 * All calls on one context are ordered on the context's CUDA stream; functions that return values to
 * host memory synchronise that stream before returning.
 */
#ifndef REBVO_B200_H
#define REBVO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct rb_ctx rb_ctx; /* device, stream, camera model, DoG filter plan, scratch */
typedef struct rb_map rb_map; /* one ring slot: sspace + edge_tracker + global_tracker (rebvo.cpp:297-312) */
typedef struct rb_pipeline rb_pipeline; /* FirstThr + SecondThread per-frame flow, device resident */

enum rb_status {
    RB_OK = 0,
    RB_ERR_CUDA = -1,
    RB_ERR_ARG = -2,
    RB_ERR_NO_DEVICE = -3,
    RB_ERR_STATE = -4
};

/* struct KeyLine (include/mtracklib/edge_finder.h:45-91): 168-byte AoS record produced for host
 * consumers by rb_map_sync_host_keylines(); field names and offsets are the reference's. */
typedef struct rb_keyline {
    int32_t p_inx;
    float m_m[2], u_m[2], n_m, score, c_p[2];
    int32_t _pad0;
    double rho, s_rho, rho_nr, s_rho_nr, rho0, s_rho0;
    float p_m[2], p_m_0[2];
    int32_t m_id, m_id_f, m_id_kf, m_num;
    float m_m0[2];
    double n_m0;
    int32_t p_id, n_id, net_id, stereo_m_id;
    double stereo_rho, stereo_s_rho;
} rb_keyline;

/* cam_model (include/UtilLib/cam_model.h:32-50): pinhole part used by the hot path.  Any w >= 32, h >= 32 (KITTI's
 * 1241x376 and 1226x370 included): the push calls take packed frames (3*w*h or w*h bytes, no row stride), and
 * rb_pipeline_push_frames / rb_pipeline_push_frames_dev take frames with a row step, one buffer per frame; the device keeps
 * the scale-space planes in rows padded to a multiple of 4 floats, which no interface exposes. */
typedef struct rb_camera {
    int32_t w, h;
    float ppx, ppy, zfx, zfy;
} rb_camera;

/* arguments of edge_finder::detect (edge_finder.cpp:342-365) */
typedef struct rb_detect_params {
    int32_t plane_fit_size; /* DetectorPlaneFitSize 1..4: a 3x3 to 9x9 plane-fit window (other values: RB_ERR_ARG) */
    double pos_neg_thresh;  /* DetectorPosNegThresh */
    double dog_thresh;      /* DetectorDoGThresh */
    int32_t kl_max;         /* MaxPoints */
    int32_t kl_ref;         /* ReferencePoints */
    double gain;            /* DetectorAutoGain (0 = fixed threshold) */
    double thresh_max, thresh_min;
} rb_detect_params;

/* the REBVOParameters subset (include/rebvo/rebvo.h:64-235) the edge pipeline reads */
typedef struct rb_params {
    rb_camera cam;
    double Sigma0, KSigma;
    rb_detect_params det;
    double DetectorThresh;
    int32_t TrackPoints;
    int32_t QCutOffNumBins;
    double QCutOffQuantile;
    int32_t SearchRange;
    int32_t TrackerIterNum, TrackerInitIterNum, TrackerInitType;
    double TrackerMatchThresh;
    double LocationUncertaintyMatch, MatchThreshModule, MatchThreshAngle;
    double ReweigthDistance;
    uint32_t MatchNumThresh;
    int32_t MatchThreshold; /* GlobalMatchThreshold */
    double RegularizeThresh, ReshapeQAbsolute, ReshapeQRelative, LocationUncertainty;
    double DoReScaling;
    double config_fps;
    int32_t kl_capacity; /* KEYLINE_MAX of the build (<= 50000) */
} rb_params;

/* NavData subset + per-frame scalars REBVO hands to the output callback (rebvo.h:292-351) */
typedef struct rb_nav {
    double t, dt;
    double Rot[9], RotLie[3], Vel[3];
    double Pose[9], PoseLie[3], Pos[3];
    double V[3], W[3]; /* raw minimiser output (translation, rotation) */
    double K, Kp, RKp, s_rho_p;
    double score;   /* Minimizer_RV return value */
    int32_t kn;     /* keylines in this edge map */
    int32_t matches; /* directed_matching() return */
    int32_t fwd_matches; /* distinct new keylines matched by FordwardMatch (see rb_forward_match) */
    int32_t estimation_ok;
    float thresh;   /* detector threshold used for this frame */
    float retuned_thresh;
} rb_nav;

/* On-disk formats of the third thread (host code, no device work).  rb_nav_format_trajectory: the lines of the reference's
 * TrayFile (rebvo_third_t.cpp:311: t / ImuTimeScale, Pos, util::LieRot2Quaternion(PoseLie), std::scientific with 18 digits,
 * TooN vector streaming), one per record.  rb_nav_format_log: the pose / map records of its m-file LogFile
 * (rebvo_third_t.cpp:265-281: Kp, RKp, Rot, Vel, t, dt, i, Pose, Pos, K, KLN), a_log_inx counted from first_index, p_id from
 * frame_id0.  Both write at most cap bytes (no terminator) and report the length needed in *written; RB_ERR_ARG if it did
 * not fit. */
int rb_nav_format_trajectory(const rb_nav *nav, int n, double time_scale, char *buf, size_t cap, size_t *written);
int rb_nav_format_log(const rb_nav *nav, int n, long long first_index, long long frame_id0, char *buf, size_t cap,
                      size_t *written);

/* struct OdometryMeas (include/mtracklib/pose_graph.h:31-52): the relative motion of one tracked frame with its information
 * matrix, as SecondThread appends it to REBVO::poses (rebvo_second_t.cpp:323-334 in IMU mode, :371-382 otherwise).  Fields in
 * the order OdometryMeas::dumpToFile writes them.
 *   relPosPose   [0:3] -R*V (translation), [3:6] SO3(R).ln(), with R the backward rotation and V the minimiser's
 *                translation before the NaN guard (IMU mode: Rgva, Vgva)
 *   WrelPosPose  J^T * W_X * J (row-major), J the inverse of J_rp_x = [[-R, [relPosPose[0:3]]x], [0, -I]] (the reference
 *                takes TooN's SVD pseudo-inverse; the closed-form inverse used here agrees to rounding).  W_X: the minimiser's
 *                JtJ (IMU mode: W_Xgv after BiasCorrect).  Deviation: after an empty old map the reference's W_X is an
 *                uninitialised matrix (rebvo_second_t.cpp:345, Minimizer_RV returns at once); the pipeline writes zeros.
 *   AcelMeas     the frame's mean accelerometer reading (zero without an IMU); IMU mode: As
 *   VisualMeas, GMeas, Rs, Rv, Rg   zero without an IMU; IMU mode: Av, g_est, Rs, P_V / dt^4, P[1:4, 1:4]
 *   K, WK, QK    1, 0 and P_Kp as the frame found it (the previous frame's RKp); IMU mode: K, 1 / P(0, 0), P_Kp
 *   KF_ID        -1 (TrackKeyFrames is not supported) */
typedef struct rb_odometry {
    double relPosPose[6];
    double WrelPosPose[36];
    double AcelMeas[3], VisualMeas[3], GMeas[3];
    double Rs[9], Rv[9], Rg[9];
    double K, WK, QK;
    int32_t KF_ID;   /* kf_list.size()-1 (rebvo_second_t.cpp:598): -1, keyframes are not tracked */
    int32_t tracked; /* 0 for a frame SecondThread never tracked (the first frame of a sequence): not part of the pose graph */
} rb_odometry;
/* pose_graph::saveToFile (pose_graph.cpp:32-40, util::dumpElement / dumpVector / dumpMatrix of toon_util.h): a uint32 record
 * count, then per record 6 + 36 + 3 * 3 + 3 * 9 + 3 raw doubles and one int32 (652 bytes); records with tracked == 0 are
 * skipped.  Writes at most cap bytes and reports the size needed in *written; RB_ERR_ARG if it did not fit. */
int rb_odometry_format_pose_graph(const rb_odometry *r, int n, void *buf, size_t cap, size_t *written);

/* ---- context ---------------------------------------------------------------------------------- */
/* RB_ERR_ARG for cam->w < 32, cam->h < 32, kl_capacity < 1 or kl_capacity > 50000 (the reference's KEYLINE_MAX); every
 * other frame size is accepted.  RB_ERR_CUDA, with the reason in rb_last_error, when the device cannot run Minimizer_RV's
 * 16-CTA thread-block cluster. */
int rb_ctx_create(rb_ctx **out, int device, const rb_camera *cam, double sigma0, double ksigma,
                  int kl_capacity);
void rb_ctx_destroy(rb_ctx *c);
const char *rb_last_error(const rb_ctx *c);
int rb_ctx_sync(rb_ctx *c);
/* iigauss::iigauss box plan (iigauss.cpp:43-81): out_d[6] = box widths filter0[3], filter1[3];
 * out_sigma_r[2] = achieved sigmas */
int rb_ctx_box_plan(const rb_ctx *c, int *out_d, double *out_sigma_r);
/* kernels launched on this context so far (bench.py's gpu_launches) */
int64_t rb_ctx_launch_count(const rb_ctx *c);
/* thread-block clusters of one Minimizer_RV launch: REBVO_B200_MIN_G (default 4) when all fit, else 1 */
int rb_ctx_minimizer_clusters(const rb_ctx *c);

/* ---- edge map (ring slot) ---------------------------------------------------------------------- */
int rb_map_create(rb_ctx *c, rb_map **out);
void rb_map_destroy(rb_map *m);
/* edge_finder(const edge_finder&) + global_tracker(const global_tracker&) (edge_finder.cpp:42-52,
 * global_tracker.cpp:42-47; used by keyframe, keyframe.cpp:28-35): a new map holding a device-side copy of the
 * keylines, id mask, match field (+ radius) and FrameCount of src */
int rb_map_clone(const rb_map *src, rb_map **out);

/* Image<float>::ConvertRGB2BW (image.h:197-203) after the H2D copy of the RGB24 frame */
int rb_map_upload_rgb(rb_map *m, const uint8_t *rgb);
/* the same for an 8-bit grayscale frame (w*h bytes): it stands for the RGB24 frame (m, m, m), so the gray plane
 * (rb_map_get_plane 5) is float(3*v), bit-identical to rb_map_upload_rgb's on the replicated frame */
int rb_map_upload_mono(rb_map *m, const uint8_t *mono);
int rb_map_upload_gray(rb_map *m, const float *gray);
/* sspace::build (sspace.cpp:52-60): bit-exact float32 integral-image DoG */
int rb_map_dog_build(rb_map *m);
/* which: 0 Img(0), 1 Img(1), 2 ImgDOG, 3 ImgDx, 4 ImgDy, 5 gray.  Img(1), dx, dy are materialised on
 * demand (the detector computes them on the fly). */
int rb_map_get_plane(rb_map *m, int which, float *out);
/* edge_finder::detect (edge_finder.cpp:342-365): UpdateThresh + build_mask + join_edges.
 * tresh / l_kl_num are the caller-held feedback state of FirstThr (rebvo_first_t.cpp:92-94). */
int rb_map_detect(rb_map *m, const rb_detect_params *p, double *tresh, int *l_kl_num, int *kn_out);
/* same, reading the scale space of another ring object (the reference passes `sspace *ss` to detect()) */
int rb_map_detect_ss(rb_map *m, rb_map *ss, const rb_detect_params *p, double *tresh, int *l_kl_num,
                     int *kn_out);
/* rb_map_detect_ss with a detection mask: w x h bytes of host memory with a row step (step >= w); a zero byte at (x, y)
 * keeps pixel (x, y) from being a keyline candidate, as rb_pipeline_set_detect_mask does in the pipeline.  The mask is
 * copied to the device for this call.  RB_ERR_ARG for a NULL mask or a step < w. */
int rb_map_detect_masked(rb_map *m, rb_map *ss, const rb_detect_params *p, const uint8_t *mask, int64_t step,
                         double *tresh, int *l_kl_num, int *kn_out);
/* edge_finder::reEstimateThresh (edge_finder.cpp:373-405) */
int rb_map_reestimate_thresh(rb_map *m, int knum, int nbins, float *out_thresh);
int rb_map_knum(rb_map *m, int *kn);
/* the matching counters of the frame that built this map: out = {fwd_match, nmatch, reg_num} (FordwardMatch winners,
 * directed_matching hits, keylines Regularize_1_iter smoothed) */
int rb_map_counters(rb_map *m, int out[3]);
/* AoS mirror for host consumers (callback / net packer): kn records of 168 bytes */
int rb_map_sync_host_keylines(rb_map *m, rb_keyline *dst, int capacity, int *kn);
/* test / checkpoint path: load an edge map (keylines + mask) produced elsewhere */
int rb_map_load_keylines(rb_map *m, const rb_keyline *src, int kn, const int32_t *mask);
int rb_map_get_mask(rb_map *m, int32_t *out);

/* edge_tracker::EstimateQuantile (edge_tracker.cpp:1148-1186) */
int rb_map_quantile(rb_map *m, double s_rho_min, double s_rho_max, double percentile, int nbins,
                    double *out);
/* global_tracker::build_field (global_tracker.cpp:61-105) on this map's own keylines */
int rb_map_build_field(rb_map *m, int radius, float min_mod);
/* out: w*h pairs {dist, ikl} as the reference's gt_field_data (global_tracker.h:33-36) */
int rb_map_get_field(rb_map *m, int32_t *out);
/* one global_tracker::TryVelRot<double,ReWeight,ProcJF,false> evaluation (global_tracker.cpp:285-543).
 * fmap holds the field (new map), old is the map being moved.  res_in / res_out: K0 doubles (may be
 * NULL when !reweight / not wanted).  JtJ / JtF are written only when procjf, as the reference leaves them. */
int rb_try_vel_rot(rb_map *fmap, rb_map *old, const double X[6], int reweight, int procjf,
                   double match_thresh, double s_rho_min, uint32_t match_num_thresh, double k_huber,
                   const double *res_in, double *res_out, double JtJ[36], double JtF[6], double *score);
/* global_tracker::Minimizer_RV<double,false> (global_tracker.cpp:578-819), device-resident LM loop */
int rb_minimizer_rv(rb_map *fmap, rb_map *old, double V[3], double W[3], double RVel[9], double RW0[9],
                    double match_thresh, int iter_max, int init_type, double reweight_distance,
                    double *rel_error, double *rel_error_score, double max_s_rho,
                    uint32_t match_num_thresh, int init_iter, double W_X[36], double *score);
/* rb_minimizer_rv as the per-frame pipeline runs it, followed by FordwardMatch of old into fmap: fmap's arg-max scratch
 * cleared, the minimiser with a scratch frame state (so that its last evaluation offers every old keyline to the
 * arg-max), then FordwardMatch's apply.  On return fmap is what Minimizer_RV followed by FordwardMatch leaves; the other
 * outputs are rb_minimizer_rv's.  *fwd_nmatch counts distinct matched new keylines, as rb_forward_match's. */
int rb_minimizer_rv_forward(rb_map *fmap, rb_map *old, double V[3], double W[3], double RVel[9], double RW0[9],
                            double match_thresh, int iter_max, int init_type, double reweight_distance,
                            double *rel_error, double *rel_error_score, double max_s_rho,
                            uint32_t match_num_thresh, int init_iter, double W_X[36], double *score,
                            int *fwd_nmatch);
/* What the per-frame map chain leaves besides the two maps (rb_map_match_update) */
typedef struct rb_match_update_out {
    int32_t nmatch;     /* directed_matching hits */
    int32_t fwd_match;  /* distinct new keylines with a FordwardMatch winner */
    int32_t reg_num;    /* keylines Regularize_1_iter smoothed */
    int32_t do_map, est_ok, klm_num;   /* the match-count gate (rebvo_second_t.cpp:410-423) */
    double V[3], Kp, P_Kp, P_V[9];      /* after the gate; Kp and P_Kp enter as 0 */
    double Pose[9], Pos[3];             /* Pose = Pose*BackRot, Pos += -Pose*V*K (:545-551) */
    double RotLie[3], PoseLie[3];       /* SO3(BackRot).ln(), SO3(Pose).ln() */
} rb_match_update_out;
/* The per-frame map chain of the pipeline on loaded maps: FordwardMatch of old's m_id_f into neu, directed_matching
 * (edge_tracker.cpp:302-374) of neu against old rotated by R0 (rotate_keylines), the match-count gate
 * (do_match && nmatch >= match_threshold), Regularize_1_iter and the EKF when the gate is open, old rotated by R0 in
 * place, and the frame's pose integration.  V / P_V are the minimiser's outputs before directed_matching's
 * back-rotation by BackRot.  Pose_io / Pos_io are updated in place; neu's counters start at 0. */
int rb_map_match_update(rb_map *neu, rb_map *old, const double V[3], const double P_V[9], const double BackRot[9],
                        const double R0[9], int do_match, double min_thr_mod, double min_thr_ang, double max_radius,
                        double loc_uncertainty_match, int match_threshold, double reg_thresh, double reshape_q_abs,
                        double loc_uncertainty, double Pose_io[9], double Pos_io[3], double K, rb_match_update_out *out);
/* edge_tracker::FordwardMatch (edge_tracker.cpp:380-436): old -> new along m_id_f.  The keyline contents follow the
 * reference's sequential rule (arg-max rho, ties -> largest index) bit for bit.  *nmatch counts DISTINCT matched new
 * keylines; the reference's return value also counts the writes that a later old keyline overwrites (its nmatch++ runs
 * per write), so it is larger when several old keylines hit one new keyline.  The count is diagnostic only: the
 * reference overwrites it with directed_matching()'s before anything reads it (rebvo_second_t.cpp:354,410). */
int rb_forward_match(rb_map *old, rb_map *neu, int *nmatch);
/* edge_tracker::rotate_keylines (edge_tracker.cpp:42-76) */
int rb_map_rotate_keylines(rb_map *m, const double R[9]);
/* edge_tracker::directed_matching (edge_tracker.cpp:302-374) */
int rb_directed_matching(rb_map *neu, rb_map *old, const double Vel[3], const double RVel[9],
                         const double BackRot[9], double min_thr_mod, double min_thr_ang,
                         double max_radius, double loc_uncertainty, int *nmatch);
/* edge_tracker::Regularize_1_iter (edge_tracker.cpp:87-148) */
int rb_map_regularize(rb_map *m, double thresh, int *r_num);
/* edge_tracker::UpdateInverseDepthKalman -> ...ARLU (edge_tracker.cpp:695-724, 954-1055) */
int rb_map_ekf_update(rb_map *m, const double vel[3], double reshape_q_abs, double loc_uncertainty);
/* edge_tracker::EstimateReScalingOpt (edge_tracker.cpp:1104-1140) */
int rb_map_rescale_opt(rb_map *m, double s_rho_min, uint32_t match_num_min, int re_escale,
                       double *Kp, double *RKp);
/* global_tracker's FrameCount (global_tracker.cpp:356,816) of this slot */
int rb_map_set_frame_count(rb_map *m, uint32_t fc);

/* ---- IMU-mode tracker rows (SURVEY.md 8(a) K6, K13; config 3) -----------------------------------------
 * global_tracker::TryVel<double> (global_tracker.cpp:829-934): one translation-only evaluation; residuals = K0
 * doubles (|fi| per old keyline) read and updated in place (may be NULL). */
int rb_try_vel(rb_map *fmap, rb_map *old, const double Vel[3], double match_thresh, double s_rho_min,
               uint32_t match_num_thresh, double *residuals, double reweigth_distance, float min_mod,
               double JtJ[9], double JtF[3], double *score);
/* global_tracker::Minimizer_V<double> (global_tracker.cpp:1036-1093) */
int rb_minimizer_v(rb_map *fmap, rb_map *old, double Vel[3], double RVel[9], double match_thresh, int iter_max,
                   double s_rho_min, uint32_t match_num_thresh, double reweigth_distance, float min_mod,
                   double *score);
/* edge_tracker::ExtRotVel(vel, Wx, Rx, X, LocUncert, HubReweigth) (edge_tracker.cpp:1207-1301); *ok = 0 when the
 * reference would return false (NaN estimate) */
int rb_ext_rot_vel(rb_map *m, const double vel[3], double Wx[36], double Rx[36], double X[6],
                   double loc_uncertainty, double hub_reweight, int *ok);
/* edge_tracker::BiasCorrect (edge_tracker.cpp:1308-1338), host algebra, all arguments in/out like the reference */
int rb_bias_correct(double X[6], double Wx[36], double Gb[3], double Wb[9], const double Rg[9],
                    const double Rb[9]);

/* ---- image_undistort (SURVEY.md 8(f) rank 1) --------------------------------------------------------
 * image_undistort::image_undistort + undistort<true>(Image<RGB24Pixel>&, Image<RGB24Pixel>&)
 * (src/VideoLib/image_undistort.cpp:29-94, include/VideoLib/image_undistort.h:63-123, call site
 * rebvo_first_t.cpp:231).  kc = {Kc2, Kc4, Kc6, P1, P2} of cam_model::rad_tan_distortion. */
typedef struct rb_undistort rb_undistort;
int rb_undistort_create(rb_ctx *c, const double kc[5], rb_undistort **out);
void rb_undistort_destroy(rb_undistort *u);
int rb_undistort_rgb(rb_undistort *u, const uint8_t *in, uint8_t *out); /* host RGB24 -> host RGB24 */
int rb_undistort_rgb_dev(rb_undistort *u, const uint8_t *in_dev, uint8_t *out_dev, int nimg);

/* ---- whole per-frame flow ------------------------------------------------------------------------
 * REBVO::FirstThr detector stage + REBVO::SecondThread tracker/mapper stage (ImuMode=0) with all
 * state (edge-map ring, threshold feedback, V/W/P_V, pose) resident on the device. */
int rb_pipeline_create(rb_pipeline **out, int device, const rb_params *p, int max_batch);
void rb_pipeline_destroy(rb_pipeline *pl);
const char *rb_pipeline_last_error(const rb_pipeline *pl);
/* Push n frames (host RGB24, n*w*h*3 bytes; timestamps ts[n]).  Detection of the n frames runs
 * batched, tracking runs frame by frame in order; nav_out[n] receives one record per frame (the first
 * frame ever pushed only initialises the ring: estimation_ok = 0).  Synchronous. */
int rb_pipeline_push(rb_pipeline *pl, const uint8_t *rgb, const double *ts, int n, rb_nav *nav_out);
/* same with frames already resident in device memory (device pointer), read in place.  rgb_dev may be at any byte address,
 * with and without undistortion and at every frame size: the kernels test the buffer's alignment on the device, so one
 * captured batch serves buffers of every alignment, and the records are those of the same frames pushed from host memory. */
int rb_pipeline_push_dev(rb_pipeline *pl, const uint8_t *rgb_dev, const double *ts, int n,
                         rb_nav *nav_out);
/* Mono input (8-bit grayscale cameras such as EuRoC cam0): n frames of w*h bytes, row-major, no stride.  A mono frame m is
 * defined to be the RGB24 frame (m, m, m), which is what the reference's ROS nodelet (MONO8) and DataSetCam build from a gray
 * image; the records, maps and mirror are bit-identical to rb_pipeline_push of the replicated frames, with and without
 * undistortion, and in IMU mode.  The host copy and the device staging are a third of the RGB24 ones.  A pipeline may
 * alternate formats from push to push.  Arguments are checked like rb_pipeline_push's; the device variant also returns
 * RB_ERR_ARG for a pointer that is not 4-byte aligned (the kernels read 32-bit words), before anything is enqueued.  When
 * w*h is not a multiple of 4 the frames after the first start at unaligned bytes of that buffer; they are read correctly.
 * (The mono rule stays where the RGB24 call takes any address: device allocators return aligned buffers, and mono frames at
 * any address can be pushed in place with rb_pipeline_push_frames_dev, whose kernels read sources at any byte.) */
int rb_pipeline_push_mono(rb_pipeline *pl, const uint8_t *mono, const double *ts, int n, rb_nav *nav_out);
int rb_pipeline_push_mono_dev(rb_pipeline *pl, const uint8_t *mono_dev, const double *ts, int n, rb_nav *nav_out);
/* Strided frames, one buffer per frame, as the reference's ROS nodelet reads a sensor_msgs/Image (data[step*y + x*3 + c] for
 * rgb8, data[step*y + x] for mono8): pixel (x, y) of frame i is at frames[i].data + y * frames[i].step + x * bpp, bytes r, g, b
 * for RB_FRAME_RGB24 (bpp 3), one byte for RB_FRAME_MONO8 (bpp 1).  Frames need not be adjacent, ordered or aligned, and each
 * may have its own step.  The frames array itself is host memory in both calls; the _dev call's data pointers are device
 * pointers on the pipeline's device.  A push reads only the bytes of each frame's span [data, data + (h-1)*step + w*bpp), and
 * the bytes between rows never change a result: the records, maps, mirror, depth grids and images and the threshold feedback
 * are those of rb_pipeline_push / push_mono / push_dev / push_mono_dev of the same pixels packed, with and without
 * undistortion, at every frame size, and in IMU mode (dataset and live).
 *   rb_pipeline_push_frames: each frame is copied into the pipeline's packed staging with one 2D copy, then the batch runs
 *     exactly as a packed push of that format (same kernels, same captured batches).
 *   rb_pipeline_push_frames_dev: the frames are read in place.  A device table of max_batch {data, step} entries is written
 *     before the batch runs; the gray pass (with or without undistortion) reads each frame through it.  Such pushes have
 *     captured batches of their own, so a pipeline may alternate packed and strided pushes, and they launch as many kernels
 *     as a packed device push of the same size and format.
 * RB_ERR_ARG, before anything is enqueued and with the state unchanged, for a format other than the two below, n outside
 * 1..max_batch, a NULL frames, ts or data, a step < w * bpp, and, for the _dev call with undistortion on, frames wider or
 * higher than 65535 pixels.  Live IMU mode checks the samples' coverage as for a packed
 * push.  Synchronous, like rb_pipeline_push. */
typedef struct rb_frame {
    const uint8_t *data; /* first byte of row 0 */
    int64_t step;        /* bytes from the start of one row to the next (sensor_msgs/Image step); >= w * bytes per pixel */
} rb_frame;
enum { RB_FRAME_RGB24 = 0, RB_FRAME_MONO8 = 1 };
int rb_pipeline_push_frames(rb_pipeline *pl, int format, const rb_frame *frames, const double *ts, int n, rb_nav *nav_out);
int rb_pipeline_push_frames_dev(rb_pipeline *pl, int format, const rb_frame *frames, const double *ts, int n,
                                rb_nav *nav_out);
/* Detection masks: keep keylines off pixels that must not be tracked (the robot's own body, the camera housing, burned-in
 * overlays, objects that move on their own).  A mask is w x h bytes with a row step (>= w).  A zero byte at (x, y) means
 * no keyline is detected at the detector's pixel (x, y), the one that becomes the keyline's p_inx = y * w + x (c_p is that
 * pixel plus the sub-pixel offset); any other value allows detection there.  With undistortion on, (x, y) is a pixel of
 * the undistorted image: the caller draws the mask in that frame (masks are not undistorted).  A masked pixel is simply
 * not a candidate; everything after the candidate test is unchanged: the raster-order compaction, the kl_max cut (which
 * counts unmasked candidates only), join_edges, the threshold feedback (l_kl_num = the masked count) and the rest of the
 * flow.  A pixel is kept only when no mask that is set zeroes it.
 *
 * rb_pipeline_set_detect_mask(pl, mask, step, on_device): copies the mask (host or device memory) into device memory the
 *   pipeline owns.  It applies to every later push and enqueue, in every input layout, with and without undistortion, and
 *   in IMU dataset and live mode.  mask = NULL clears it.  Setting or clearing it re-captures no batch: pipelines with no
 *   mask set launch the kernels, with the arguments, of a pipeline that never had one.  The fixed mask is configuration,
 *   not session state: rb_pipeline_reset and rb_pipeline_load_state keep it, and session blobs do not carry it.
 *   RB_ERR_ARG for a step < w; RB_ERR_STATE while asynchronous tickets are outstanding (as every set_* call).
 * rb_pipeline_push_masked(pl, format, on_device, frames, masks, ts, n, nav_out) and
 * rb_pipeline_masked_enqueue(pl, format, on_device, frames, masks, ts, n, &ticket): frames exactly as
 *   rb_pipeline_push_frames(_dev) and rb_pipeline_enqueue_frames take them, plus one rb_frame {data, step} per frame for
 *   its mask, in device memory on the pipeline's device (masks[] itself is host memory).  The masks are read in place
 *   through a per-frame device table written before the batch, so one captured batch serves every mask buffer; masked
 *   pushes have captured batches of their own.  The masks must be complete when the call is made and stay unchanged until
 *   the push returns or the ticket is waited, as device frames.  A fixed mask applies as well.  Argument checks are those
 *   of the strided calls, plus RB_ERR_ARG for a NULL masks, a NULL mask data or a mask step < w, before anything is
 *   enqueued and with the state unchanged.  rb_pipeline_masked_enqueue is refused in IMU mode, as rb_pipeline_enqueue;
 *   rb_pipeline_push_masked works there. */
int rb_pipeline_set_detect_mask(rb_pipeline *pl, const uint8_t *mask, int64_t step, int on_device);
int rb_pipeline_push_masked(rb_pipeline *pl, int format, int on_device, const rb_frame *frames, const rb_frame *masks,
                            const double *ts, int n, rb_nav *nav_out);
int rb_pipeline_masked_enqueue(rb_pipeline *pl, int format, int on_device, const rb_frame *frames,
                               const rb_frame *masks, const double *ts, int n, int64_t *ticket);
/* Asynchronous pushes: a live caller (a camera driver thread, a ROS image callback) hands over frames without waiting for
 * them to be tracked, and keeps up to `depth` pushes in flight, as the reference's FirstThr detects frame i+1 while its
 * SecondThread tracks frame i.  Each enqueued push (a ticket) has the records and outputs the synchronous push of the same
 * frames would have given, byte for byte; only when they are ready differs.  See DESIGN.md §5 for how a ticket runs.
 *
 * rb_pipeline_set_async(pl, depth): how many tickets may be outstanding, 1..8, or 0 (off, the default).  It allocates, at
 *   this call and never in an enqueue, an output ring of `depth` slots (nav, odometry, mirror, depth grid and depth image of
 *   max_batch frames each, in host or device memory as rb_pipeline_set_output_memory says; the set_* calls that switch an
 *   output on or enlarge it grow the slots too) and a second scale-space workspace of max_batch frames.  depth = 0 frees the
 *   ring; the synchronous pushes never use it and launch what they launched before.  RB_ERR_ARG in IMU mode and for a depth
 *   outside 0..8; RB_ERR_STATE while tickets are outstanding.
 * rb_pipeline_enqueue(pl, format, on_device, data, ts, n, &ticket): n packed frames of RB_FRAME_RGB24 or RB_FRAME_MONO8, in
 *   host (on_device = 0) or device memory, with the checks of rb_pipeline_push / push_mono / push_dev / push_mono_dev.
 *   rb_pipeline_enqueue_frames: n strided frames, with the checks of rb_pipeline_push_frames(_dev).  Both return once the
 *   work is enqueued; *ticket receives its number (0, 1, 2, ... for the pipeline's lifetime).  The frames (and the data the
 *   rb_frame entries point to) must stay valid and unchanged until that ticket is waited.  Device frames must be complete
 *   when the call is made: the copy and the scale space run on a stream of their own, ordered after nothing the caller
 *   enqueued.  Host frames in pageable memory may make the call wait for the copy; pinned memory does not.  RB_ERR_STATE,
 *   changing nothing, when `depth` tickets are outstanding; RB_ERR_ARG when asynchronous pushes are off or in IMU mode.
 * rb_pipeline_wait(pl, ticket, nav_out): blocks until the ticket is complete and retires it with every earlier ticket, in
 *   order, doing for each what a synchronous push does on the host after its work (odometry QK, the first frame's record, the
 *   minimiser abort check).  nav_out (may be NULL) receives the ticket's n records.  From then until the next wait or push,
 *   rb_pipeline_odometry, rb_pipeline_mirror(_dev), rb_pipeline_depth(_dev) and rb_pipeline_depth_image(_dev) return the
 *   ticket's outputs; they stay valid until the enqueue that reuses the ticket's slot (ticket + depth), or the next push or
 *   set_* call.  RB_ERR_CUDA when a minimiser of a ticket it retired aborted (as a push reports it); RB_ERR_ARG for a
 *   ticket never issued or already retired.
 * rb_pipeline_poll(pl, &newest): without blocking, the newest ticket whose work is complete, retired or not (-1 if none).
 *
 * While tickets are outstanding the synchronous pushes, rb_pipeline_reset, rb_pipeline_save_state / load_state, every set_*
 * call (rb_pipeline_set_async, set_consumer_stream and set_imu among them), rb_pipeline_batch_plane, rb_pipeline_stage_ms
 * and rb_pipeline_bench_pass return RB_ERR_STATE and change nothing; with none outstanding they behave as before.
 * rb_pipeline_batch_plane has no planes to show after an enqueue, and rb_pipeline_stage_ms describes the last synchronous
 * push.  In device output mode, each enqueue first makes the tracker stream wait for the work enqueued so far on the
 * consumer stream (rb_pipeline_set_consumer_stream), which covers whatever still reads the slot it is about to overwrite.
 * The calls of one pipeline are made from one thread at a time, as its pushes are. */
int rb_pipeline_set_async(rb_pipeline *pl, int depth);
int rb_pipeline_enqueue(rb_pipeline *pl, int format, int on_device, const uint8_t *data, const double *ts, int n,
                        int64_t *ticket);
int rb_pipeline_enqueue_frames(rb_pipeline *pl, int format, int on_device, const rb_frame *frames, const double *ts, int n,
                               int64_t *ticket);
int rb_pipeline_wait(rb_pipeline *pl, int64_t ticket, rb_nav *nav_out);
int rb_pipeline_poll(rb_pipeline *pl, int64_t *newest_complete);
/* REBVO::Reset (rebvo_second_t.cpp:609-620) */
int rb_pipeline_reset(rb_pipeline *pl);
/* newest / previous edge map of the ring (valid until the next push) */
rb_map *rb_pipeline_map(rb_pipeline *pl, int age);
/* Per-frame host mirror of the edge map: the reference hands every frame's KeyLine array (edge_finder::operator[],
 * include/mtracklib/keyline.h) to its consumers (third thread: net_keypoint.cpp, keyframes).  With the mirror on, each frame's
 * keylines are packed right after its map update and written into pinned host memory while the following frames are tracked
 * (part of the batch: no extra calls).  mode 1: the 168-byte KeyLine records (rb_keyline); mode 2: the 15-byte net_keyline
 * wire records the third thread builds from them (copy_net_keyline + copy_net_keyline_nextid with pbuf.K,
 * rebvo_third_t.cpp:192-197); mode 0: off.  rb_pipeline_mirror(i) = the records of frame i of the last push, valid from the
 * return of that push until the next one.  Not available in IMU mode. */
int rb_pipeline_set_mirror(rb_pipeline *pl, int mode);
/* UseUndistort=1 (rebvo_first_t.cpp:211-231: image_undistort::undistort<true> on every captured frame before the scale
 * space): with a non-zero kc = {KcR2, KcR4, KcR6, KcP1, KcP2} every pushed frame is undistorted with the reference's
 * fixed-point bilinear map, fused into the RGB -> BW pass.  kc == NULL or all zero: off. */
int rb_pipeline_set_undistort(rb_pipeline *pl, const double kc[5]);
int rb_pipeline_mirror(rb_pipeline *pl, int i, const void **records, int *n);
/* Per-frame odometry measurements (rb_odometry, the reference's pose graph REBVO::poses).  on = 1: every push also produces one
 * record per frame; the products run in a spare thread of a kernel that already follows the match-count gate (k_reg_ekf, or the
 * gate kernel of the reference schedule) and the records reach the host with the nav records, so a push launches no more
 * kernels than without them (the constant is 0).  In IMU mode the records are built by the host flow.  May be called between
 * pushes; on = 0 restores the batches of a pipeline that never had it.  rb_pipeline_odometry: the n records of the last push,
 * record i for frame i (like nav_out[i]), valid until the next push; RB_ERR_STATE when the last push ran without them. */
int rb_pipeline_set_odometry(rb_pipeline *pl, int on);
int rb_pipeline_odometry(rb_pipeline *pl, const rb_odometry **recs, int *n);
int64_t rb_pipeline_launch_count(const rb_pipeline *pl);
/* CUDA-event time (ms) of the last push split by stage: [0] h2d+gray, [1] DoG, [2] detect,
 * [3] tracker (field + minimiser), [4] mapper, [5] total */
int rb_pipeline_stage_ms(const rb_pipeline *pl, float out[6]);
/* In-situ stage profile, enabled by REBVO_B200_STAGE_PROF=1 at creation (forces eager launches): accumulated CUDA-event
 * milliseconds per stage over all pushes so far: [0] copies, [1] gray, [2] scale space, [3] detect, [4] reEstimateThresh,
 * [5] quantile + build_field, [6] Minimizer_RV, [7] FordwardMatch + rotate, [8] directed_matching, [9] regularize + EKF,
 * [10] rescale, [11] pose/nav, [12] nav copy */
int rb_pipeline_stage_profile(rb_pipeline *pl, double out_ms[16], long long *frames);
/* opaque stream handle (cudaStream_t) the pipeline launches on, for CUDA-event timing by the caller */
void *rb_pipeline_stream(rb_pipeline *pl);
/* CUDA-event stopwatch on the pipeline's own stream (bench.py): record slot 0..7, elapsed(a,b) in ms
 * (synchronises on event b) */
int rb_pipeline_event_record(rb_pipeline *pl, int slot);
int rb_pipeline_event_elapsed_between(rb_pipeline *pa, int a, rb_pipeline *pb, int b, float *ms);
int rb_pipeline_event_elapsed(rb_pipeline *pl, int a, int b, float *ms);
/* Measurement hook: re-run ONE scale-space pass over the pipeline's batched workspace `iters` times and
 * return the mean CUDA-event duration per launch.  pass_id: 0 row pass (plain), 1 row pass with box
 * average (2*nimg images), 2 column pass (2*nimg images), 3 last box + DoG, 4 rgb->gray, 5 undistortion + rgb->gray
 * (needs rb_pipeline_set_undistort), 6 mono->gray, 7 undistortion + mono->gray (needs rb_pipeline_set_undistort).
 * bytes_per_launch receives the algorithmic bytes of one launch (DESIGN.md section 4). */
int rb_pipeline_bench_pass(rb_pipeline *pl, int pass_id, int nimg, int iters, float *ms_per_launch,
                           double *bytes_per_launch);
/* Test and debug accessor, like rb_map_get_plane: plane `which` (0 Img(0), 2 ImgDOG, 5 gray) of slot `slot` of the last
 * scale-space batch the pipeline built, w*h floats.  The last push's frames in order, except after a host push cut into a
 * head and the rest (REBVO_B200_SUB): the slots then hold the rest, frames sub..n-1.  RB_ERR_ARG for a slot not below the
 * size of that batch (none after creation, a failed push or rb_pipeline_bench_pass) or another `which`.  Synchronous. */
int rb_pipeline_batch_plane(rb_pipeline *pl, int slot, int which, float *out);

/* Wire egress of an edge map (monocular): the 15-byte packed net_keyline records of copy_net_keyline +
 * copy_net_keyline_nextid (src/CommLib/net_keypoint.cpp:29-107, struct net_keyline include/CommLib/net_keypoint.h:37-62,
 * NET_RHO_SCALING = 1e4), built on the device from the SoA: dst receives min(kn, capacity) records of 15 bytes, *n_out their
 * number.  k_prof is the depth scale the third thread passes (pbuf.K, rebvo_third_t.cpp:192). */
int rb_map_pack_net_keylines(rb_map *m, double k_prof, void *dst, int capacity, int *n_out);

/* Dense inverse-depth grid of a frame: the viewer's depth_filler on each net_keyline packet (src/visualizer/visualizer.cpp:436-440,
 * depth_filler(cam, {block_w, block_h}, BOUND_NONE) at :303; src/visualizer/depth_filler.cpp):
 *   ResetData; FillEdgeData(net_kl, n, {0,0}, thresh_rel_rho, thresh_match_num) (discart = true); InitCoarseFine;
 *   Integrate(iter_num) (init_cf = true); computeDistance(Zeros)
 * The grid is gw = w / block_w by gh = h / block_h cells (integer division); each cell holds the fused or filled inverse depth
 * rho, its deviation s_rho, the distance |P| of its centre's 3D point from the camera (get3DPos, depth_filler.h:115-122) and
 * whether a record fell into it.  min_dist is depth_filler::GetMinDist.  Bit-identical to the reference, with one deviation: a
 * record whose cell index is >= gw * gh (qy / block_h >= gh) writes out of bounds in the reference (undefined behaviour) and is
 * dropped here.  Every shipped viewer configuration uses block 10 x 10, thresh_rel_rho 1, thresh_match_num 5, iter_num 10.
 * RB_ERR_ARG for a block < 1 or larger than the frame, and for iter_num < 0. */
typedef struct rb_depth_params {
    int32_t block_w, block_h;   /* depth_filler's blockSize */
    double thresh_rel_rho;      /* DF_ThreshRelRho: records with s_rho / rho above it are skipped */
    int32_t thresh_match_num;   /* DF_ThreshMatchNum: records with m_num below it are skipped */
    int32_t iter_num;           /* DF_IterNum: Integrate1Step sweeps */
} rb_depth_params;
typedef struct rb_depth_cell {   /* df_point's rho, s_rho, dist, fixed; the grid is row-major gh x gw */
    double rho, s_rho, dist;
    int32_t fixed, _pad;
} rb_depth_cell;
/* the fill of n 15-byte net_keyline records in host memory on the context's camera; out receives gw * gh cells */
int rb_depth_fill_net(rb_ctx *c, const void *records, int n, const rb_depth_params *p, rb_depth_cell *out, int *gw, int *gh,
                      double *min_dist);
/* Per-frame depth grid in the pipeline: with p set, every pushed frame's edge map is packed as net_keyline records with the
 * frame's K (rebvo_third_t.cpp:191, pbuf.K; with mirror mode 2 the mirror's records are used) and filled by one CTA on a side
 * stream while the following frames are tracked; the cells go straight into pinned host memory.  p == NULL: off, and the
 * pushes run the batches of a pipeline that never had it.  Changing it drops the captured batches, like set_mirror.
 * RB_ERR_ARG for invalid p (as rb_depth_fill_net) and in IMU mode.  rb_pipeline_depth(i): the grid of frame i of the last push,
 * valid from the return of that push until the next one; RB_ERR_ARG when depth is off or i is out of range. */
int rb_pipeline_set_depth(rb_pipeline *pl, const rb_depth_params *p);
int rb_pipeline_depth(rb_pipeline *pl, int i, const rb_depth_cell **cells, int *gw, int *gh, double *min_dist);

/* Dense inverse-depth image of a depth grid: pixel (x, y) of the w x h frame (x = 0..w-1, y = 0..h-1) holds
 * depth_filler::getImgRho((float)x, (float)y, &s_rho) (include/visualizer/depth_filler.h:246-280) on the grid the same cells
 * and rb_depth_params give, i.e. the reference's expressions in its order, without contraction:
 *   x_histo = x / (float)block_w - 0.5    the quotient in float, the subtraction in double, stored as float (y likewise)
 *   xf, xc = floor, ceil of x_histo, clamped to [0, gw - 1]   (yf, yc to [0, gh - 1])
 *   dx = x_histo - xf                     in float (dy likewise)
 *   r00, r10, r01, r11 = the rho of cells (xf, yf), (xc, yf), (xf, yc), (xc, yc), cast to float
 *   rho = r00*(1-dx)*(1-dy) + r10*dx*(1-dy) + r01*(1-dx)*dy + r11*dx*dy   left to right in float
 * and s_rho the same expression on the cells' s_rho.  The reference returns that float widened to double, so the float32
 * planes hold it exactly.  The clamps are part of the definition: pixels left of or above the first cell centre
 * (x < block_w / 2) take a negative dx (dy), and pixels past gw * block_w (gh * block_h), when the frame is not a multiple of
 * the block, are clamped onto the last cell column (row), where dx (dy) may exceed 1.
 *
 * rb_depth_image: the planes of host cells (as rb_depth_fill_net / rb_pipeline_depth return them) on the context's camera;
 * rho and s_rho receive w * h floats, row-major; s_rho may be NULL.  RB_ERR_ARG when gw / gh are not the grid size of p on
 * this camera, and for the p rb_depth_fill_net rejects. */
int rb_depth_image(rb_ctx *c, const rb_depth_cell *cells, int gw, int gh, const rb_depth_params *p, float *rho, float *s_rho);
/* Per-frame images in the pipeline: mode 1 the rho plane, 2 the rho and s_rho planes, 0 off.  While the depth grid is on
 * (rb_pipeline_set_depth), every pushed frame also gets its image: the pass runs on the frame's depth side stream right
 * after its fill and writes straight into mapped pinned host memory; the batch's depth joins cover it.  May be called
 * before or after rb_pipeline_set_depth.  Changing the mode drops the captured batches, like set_mirror / set_depth; mode 0
 * gives the batches of a pipeline that never had it.  RB_ERR_ARG in IMU mode and for a mode outside 0..2.
 * rb_pipeline_depth_image(i): the planes of frame i of the last push (row-major w x h floats, no padding; *s_rho is NULL in
 * mode 1), valid until the next push; RB_ERR_ARG when the last push made no image or i is out of range. */
int rb_pipeline_set_depth_image(rb_pipeline *pl, int mode);
int rb_pipeline_depth_image(rb_pipeline *pl, int i, const float **rho, const float **s_rho);

/* Where the per-frame outputs go: where = 0 (the default) mapped pinned host memory, read with rb_pipeline_mirror,
 * rb_pipeline_depth and rb_pipeline_depth_image; where = 1 device memory, read with the _dev accessors below, for consumers
 * that work on the GPU.  It applies to the keyline mirror, the depth grid and the depth image, whichever are on; the nav and
 * odometry records stay on the host.  The same kernels write the same bytes in both modes: device mode only leaves out the
 * mirror's copy into host memory (one launch per frame fewer with the mirror on).  May be called between pushes; changing it
 * drops the captured batches, like set_mirror, and the outputs of the last push (the new mode's accessors return RB_ERR_ARG
 * until the next push).  RB_ERR_ARG for a value outside 0..1 and in IMU mode, where these outputs are not available.
 * In device mode the host accessors return RB_ERR_STATE; in host mode the _dev accessors do.
 *
 * Buffers: each mode's buffers are allocated by the set_* call that needs them, never by a push, and kept across switches.
 * A device pointer the _dev accessors return stays the same from push to push until one of these calls has to grow its
 * buffer: rb_pipeline_set_output_memory(pl, 1), when the grid or image was switched on or enlarged while in host mode;
 * rb_pipeline_set_depth, for a grid with more cells than any before in device mode; rb_pipeline_set_depth_image, for mode 2
 * after mode 1 in device mode.  The mirror's device slots are allocated once, by the first rb_pipeline_set_mirror, and
 * never move. */
int rb_pipeline_set_output_memory(rb_pipeline *pl, int where);
/* Device mode: every push first makes its tracker stream wait for the work enqueued on `stream` (a cudaStream_t of the
 * pipeline's device; NULL is the legacy default stream) at the time of the push, outside any captured batch, so that it
 * writes no output before a consumer of the last push's outputs on that stream is done with them.  The push synchronises
 * its own streams before it returns, so its outputs are complete on return and any stream may read them.  The stream must
 * stay valid while it is set; rb_pipeline_stream(pl) (the default) waits for nothing.  Kept across pushes and switches;
 * no effect in host mode. */
int rb_pipeline_set_consumer_stream(rb_pipeline *pl, void *stream);
/* Device pointers to the outputs of frame i of the last push, valid from the return of that push until the next push, in
 * the layouts of the host accessors: the mirror's *n records (rb_keyline or 15-byte net_keyline), the grid's gw * gh
 * row-major rb_depth_cell cells with *min_dist pointing at the double right after them, and the image's row-major w x h
 * float planes, s_rho (mode 2; else NULL) starting a padded plane stride after rho: w * h rounded up to a multiple of 64
 * floats.  Frame i + 1's planes start mode such strides after frame i's.  RB_ERR_ARG as the host accessors (output off or
 * not made by the last push, i out of range, NULL out-pointer for the records / cells / rho); RB_ERR_STATE in host mode. */
int rb_pipeline_mirror_dev(rb_pipeline *pl, int i, const void **records, int *n);
int rb_pipeline_depth_dev(rb_pipeline *pl, int i, const rb_depth_cell **cells, int *gw, int *gh, const double **min_dist);
int rb_pipeline_depth_image_dev(rb_pipeline *pl, int i, const float **rho, const float **s_rho);

/* IMU fusion (BASELINE configs[2], REBVOParameters ImuMode = 2: samples from a dataset file).  After this call every push runs
 * the IMU branch of REBVO::SecondThread (rebvo_second_t.cpp:182-336: gyro pre-rotation, Minimizer_V, ExtRotVel, BiasCorrect,
 * scale / gravity / bias filter of scaleestimator.cpp, filtered pose of :521-551) instead of Minimizer_RV.  samples: n rows
 * {t [s], gyro xyz [rad/s], accel xyz [m/s^2]} as ImuGrabber::LoadDataSet reads them (imugrabber.cpp:80-132, time already scaled).
 * Field names follow REBVOParameters (include/rebvo/rebvo.h:64-235). */
typedef struct rb_imu_params {
    double TimeDesinc;
    int32_t InitBias, InitBiasFrameNum;
    double BiasInitGuess[3];
    double GiroMeasStdDev, GiroBiasStdDev, AcelMeasStdDev;
    double g_module, g_module_uncer, g_uncert, VBiasStdDev, ScaleStdDevInit;
    int32_t use_se3, pad;          /* CamImuSE3File given: Rc2i / Tc2i below (ImuGrabber::LoadCamImuSE3), else identity / zero */
    double Rc2i[9], Tc2i[3];
} rb_imu_params;
int rb_pipeline_set_imu(rb_pipeline *pl, const rb_imu_params *ip, const double *samples, int n);
/* Live IMU input (REBVOParameters ImuMode = 1: ImuGrabber(CircBufferSize, SampleTime), imugrabber.cpp:34-40, fed by
 * REBVO::pushIMU).  Switches the pipeline to IMU mode, like rb_pipeline_set_imu, with an empty ring of buffer_size samples
 * (CircBufferSize; buffer_size + 1 slots) whose integration step is sample_time (SampleTime) instead of the mean sample spacing.
 * Each call replaces the IMU setup of an earlier rb_pipeline_set_imu or rb_pipeline_set_imu_live.  RB_ERR_ARG for
 * sample_time <= 0 and buffer_size < 1.
 *
 * rb_pipeline_push_imu appends n rows {t [s], gyro xyz [rad/s], accel xyz [m/s^2]} in time order (PushData,
 * imugrabber.cpp:258-269), all of them or none:
 *   RB_ERR_STATE  the ring cannot hold all n (a grabbed frame releases the samples before its last one); none is stored.
 *                 Deviation: the reference stores the samples that fit and throws overflow_error at the first that does not.
 *   RB_ERR_ARG    not in live IMU mode (off, or dataset mode), or a timestamp older than the one before it (this push's or the
 *                 last one stored).
 *
 * A push of frames in live mode first checks, for every frame, that the ring covers (t_prev + TimeDesinc, t + TimeDesinc]:
 * at least one sample after the window's start and one at or past its end.  If any frame is not covered, the push returns
 * RB_ERR_STATE before it enqueues anything and leaves the ring, the filter, the maps and the frame count as they were; push
 * the missing samples and repeat the push.  (The reference's FirstThr sleeps SampleTime and grabs again,
 * rebvo_first_t.cpp:293-302; its failed GrabAndIntegrate also releases the samples before the window, this check releases
 * none.)  The records are those of dataset mode with the same samples and the same integration step: rb_pipeline_set_imu on
 * the same samples gives the same bytes when sample_time is their mean spacing.  rb_pipeline_reset resets the filter and
 * keeps the ring: the samples it has not released and its read position.  Mono8 and device input and the odometry records
 * work as in dataset mode; the mirror and the depth grid are not available in IMU mode. */
int rb_pipeline_set_imu_live(rb_pipeline *pl, const rb_imu_params *ip, double sample_time, int buffer_size);
int rb_pipeline_push_imu(rb_pipeline *pl, const double *samples, int n);

/* ---- session checkpoints ------------------------------------------------------------------------
 * A tracking session as a versioned blob in host memory, written by one pipeline and loaded into any pipeline of the same
 * geometry, on any device and in any process: after the load the pushes continue the session exactly, with the bytes an
 * uninterrupted run would have produced (nav and odometry records, mirrors, depth grids and images).  Use it to survive a
 * process restart, to move a live stream to another GPU or worker, or to start a test or a debugging session at frame N of
 * a long stream without replaying the frames before it.
 *
 * The blob holds the session: the newest edge map (its live keylines and scalars; the keyline mask is rebuilt from them on
 * load), pose, velocity and their covariances, K / Kp / P_Kp, the detector's threshold feedback, the frame count, the last
 * timestamp, and in IMU mode the filter, the scale estimator's history and the sample ring's read position (live mode: also
 * the samples it has not released).  It does not hold the configuration, which stays with the pipeline object: mirror, depth
 * grid and image, odometry records, undistortion, the fixed detection mask, output memory, consumer stream, and the
 * rb_params fields other than the geometry.  About 120 bytes per keyline (2 MB at 15 k keylines).  Layout: DESIGN.md §5.
 *
 * rb_pipeline_save_state writes the blob into buf and its size into *written.  When cap is too small it writes nothing,
 * still reports the size needed and returns RB_ERR_ARG (buf = NULL, cap = 0 asks for the size).  Between pushes;
 * synchronous.  It changes nothing in the pipeline: the pushes after it give what they would have given.
 *
 * rb_pipeline_load_state replaces the session of pl with the blob's.  RB_ERR_ARG, with pl unchanged (its next push gives what
 * it would have given), when the blob is truncated or corrupt (checksum), of another version, of another camera (w, h, pp, zf),
 * Sigma0, KSigma or kl_capacity, or of another mode (vision only, IMU dataset, IMU live: rb_pipeline_set_imu /
 * rb_pipeline_set_imu_live must come before the load); in dataset mode when pl's samples are not the source's (count and
 * checksum); in live mode when pl's ring cannot hold the samples the source had not released.  The other rb_params fields may
 * differ: the session then continues with pl's parameters from its next frame on (a fork with other tracker settings, which
 * no uninterrupted run reproduces).  After a load the outputs of the last push are gone, as after the set_* calls: their
 * accessors return RB_ERR_ARG until the next push; rb_pipeline_map(pl, 0) is the restored map and rb_pipeline_map(pl, 1) is
 * NULL until the next push.  Neither call changes a push's captured batches: pushes launch what they launched before.
 * rb_pipeline_reset keeps its meaning (a new session).
 *
 * rb_state_info: host only, no device needed.  Checks the header and the checksum (RB_ERR_ARG otherwise) and describes the
 * blob. */
enum { RB_STATE_VISION = 0, RB_STATE_IMU_DATASET = 1, RB_STATE_IMU_LIVE = 2 };
struct rb_state_info {   /* (a struct tag, not a typedef: the function below has its name) */
    uint32_t version;
    int32_t mode;          /* RB_STATE_* */
    uint64_t bytes;        /* size of the blob */
    rb_camera cam;
    double Sigma0, KSigma;
    int32_t kl_capacity;
    int32_t kn;            /* keylines of the newest edge map */
    int64_t n_pushed;      /* frames pushed in the session */
};
int rb_pipeline_save_state(rb_pipeline *pl, void *buf, size_t cap, size_t *written);
int rb_pipeline_load_state(rb_pipeline *pl, const void *buf, size_t n);
int rb_state_info(const void *buf, size_t n, struct rb_state_info *out);

#ifdef __cplusplus
}
#endif
#endif /* REBVO_B200_H */

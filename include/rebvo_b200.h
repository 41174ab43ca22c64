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
 * name says dev.  Images are row-major without stride (Image<T>, include/VideoLib/image.h:42-217).
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

/* cam_model (include/UtilLib/cam_model.h:32-50): pinhole part used by the hot path */
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

/* ---- context ---------------------------------------------------------------------------------- */
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
/* which scale-space kernels a map's own workspace dispatches to, valid after its first rb_map_dog_build: bit 0 = row passes on
 * TMA tiles, bit 1 = last box + DoG on TMA tiles (0 = the pre-TMA kernels: width not a multiple of 4, environment switch, or
 * tensor-map creation failed) */
int rb_map_scale_space_path(const rb_map *m);

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
 * NULL when !reweight / not wanted). */
int rb_try_vel_rot(rb_map *fmap, rb_map *old, const double X[6], int reweight, int procjf,
                   double match_thresh, double s_rho_min, uint32_t match_num_thresh, double k_huber,
                   const double *res_in, double *res_out, double JtJ[36], double JtF[6], double *score);
/* global_tracker::Minimizer_RV<double,false> (global_tracker.cpp:578-819), device-resident LM loop */
int rb_minimizer_rv(rb_map *fmap, rb_map *old, double V[3], double W[3], double RVel[9], double RW0[9],
                    double match_thresh, int iter_max, int init_type, double reweight_distance,
                    double *rel_error, double *rel_error_score, double max_s_rho,
                    uint32_t match_num_thresh, int init_iter, double W_X[36], double *score);
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
/* same with frames already resident in device memory (device pointer) */
int rb_pipeline_push_dev(rb_pipeline *pl, const uint8_t *rgb_dev, const double *ts, int n,
                         rb_nav *nav_out);
/* Mono input (8-bit grayscale cameras such as EuRoC cam0): n frames of w*h bytes, row-major, no stride.  A mono frame m is
 * defined to be the RGB24 frame (m, m, m), which is what the reference's ROS nodelet (MONO8) and DataSetCam build from a gray
 * image; the records, maps and mirror are bit-identical to rb_pipeline_push of the replicated frames, with and without
 * undistortion, and in IMU mode.  The host copy and the device staging are a third of the RGB24 ones.  A pipeline may
 * alternate formats from push to push.  Arguments are checked like rb_pipeline_push's; the device variant also returns
 * RB_ERR_ARG for a pointer that is not 4-byte aligned (the kernels read 32-bit words), before anything is enqueued. */
int rb_pipeline_push_mono(rb_pipeline *pl, const uint8_t *mono, const double *ts, int n, rb_nav *nav_out);
int rb_pipeline_push_mono_dev(rb_pipeline *pl, const uint8_t *mono_dev, const double *ts, int n, rb_nav *nav_out);
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

/* Wire egress of an edge map (monocular): the 15-byte packed net_keyline records of copy_net_keyline +
 * copy_net_keyline_nextid (src/CommLib/net_keypoint.cpp:29-107, struct net_keyline include/CommLib/net_keypoint.h:37-62,
 * NET_RHO_SCALING = 1e4), built on the device from the SoA: dst receives min(kn, capacity) records of 15 bytes, *n_out their
 * number.  k_prof is the depth scale the third thread passes (pbuf.K, rebvo_third_t.cpp:192). */
int rb_map_pack_net_keylines(rb_map *m, double k_prof, void *dst, int capacity, int *n_out);

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

#ifdef __cplusplus
}
#endif
#endif /* REBVO_B200_H */

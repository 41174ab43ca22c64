// common.cuh -- shared declarations of librebvo_b200 (device layouts, context, launch helpers).
// Product code: CUDA for sm_90a only, no CPU fallback anywhere (functions fail with RB_ERR_CUDA /
// RB_ERR_NO_DEVICE when the device path is unavailable).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>

#include "../../include/rebvo_b200.h"

#define RB_RHO_MAX 20.0   // include/mtracklib/edge_finder.h:38
#define RB_RHO_MIN 1e-3   // :39
#define RB_RHO_INIT 1.0   // :40
#define RB_MAX_IMG_VALUE 765  // edge_tracker(cam, 255*3), rebvo.cpp:300

// DetectorPlaneFitSize (build_mask's win_s): the detector has one kernel instance per radius 1..RB_PLANE_FIT_MAX
#define RB_PLANE_FIT_MAX 4
// offset of radius r's 3 x (2r+1)^2 plane-fit pseudo inverse in the packed table of all radii (r = 1 first)
__host__ __device__ constexpr int rb_pinv_offset(int r) {
    int o = 0;
    for (int q = 1; q < r; q++) o += 3 * (2 * q + 1) * (2 * q + 1);
    return o;
}
#define RB_PINV_DOUBLES rb_pinv_offset(RB_PLANE_FIT_MAX + 1)   // 3 * (9 + 25 + 49 + 81) = 492

// ---- keyline storage: SoA on the device (the 168-byte AoS of the reference is produced on demand) ---
struct KLSoA {
    int *p_inx;
    float2 *m_m, *u_m, *c_p, *p_m, *p_m_0, *m_m0;
    float *n_m;
    double *rho, *s_rho, *rho0, *s_rho0, *n_m0;
    int *m_id, *m_id_f, *m_num, *p_id, *n_id;
    // one 32-byte record per keyline gathered by the minimiser through the field image:
    // {m_m.x, m_m.y, c_p.x, c_p.y, u_m.x, u_m.y, n_m, 0}
    float4 *pack;  // 2 x float4 per keyline
};

// per-map device scalars (everything a later kernel needs without a host round trip)
struct MapState {
    int kn;              // keylines in the map (edge_finder::kn)
    int total_cand;      // candidates before the kl_max cut
    float max_dog, min_dog;
    float retuned;       // edge_finder::reTunedThresh
    float thresh_used;   // detector threshold (float cast of tresh) used for this map
    int nmatch;          // edge_tracker::nmatch
    int fwd_match;
    int reg_num;
    unsigned int frame_count;  // global_tracker::FrameCount of this slot
    int do_map;          // the per-frame pipeline's mapping gate of the frame that built this map (k_regularize_a_gate)
    double s_rho_q;
    double Kp, RKp;
};

// detector feedback state of FirstThr (rebvo_first_t.cpp:92-94) kept on the device
struct DetChain {
    double tresh;
    int l_kl_num;
    int pad;
};

struct BoxPlan {
    int d[2][3];         // box widths per filter (iigauss.cpp:43-81)
    double sigma_r[2];
};

struct DogWS {           // batched scale-space workspace, B images of N floats per plane
    int B;
    uint8_t *rgb;        // B * 3N    host-input staging: B RGB24 frames, or B mono frames in its first B * N bytes
    float *gray;         // B * N
    float *S;            // 2B * N   row-scanned plane (per filter)
    float *I0;           // B * N    integral of the input (shared by both filters)
    float *I;            // 2B * N   integral image (per filter)
    float *img0;         // B * N    blur 0
    float *dog;          // B * N    blur1 - blur0
    float *aux;          // 3 * N    on-demand planes (Img(1), dx, dy) for the test/debug accessor
    void *tmaps;         // CUtensorMap[] (host, dog.cu TM_*): TMA-staged row passes, last box + DoG
    bool tma_ok;
    int tma_row_mask;
    bool tma_row_ok;     // the row passes run on TMA tiles (k_rowscan_tma_*)
};

struct rb_ctx {
    std::recursive_mutex *mtx;   // the stage-level C ABI may be called from several host threads (RB_ENTER)
    int device;
    cudaStream_t stream;
    rb_camera cam;
    int w, h, N;
    float ppx, ppy;
    double zfm;
    double sigma0, ksigma;
    int kcap;
    BoxPlan plan;
    int64_t launches;
    int sm_count;
    char err[256];
    // scratch shared by all maps of the context
    int *seg_cnt;        // detect: per (row, 32-px chunk) candidate counts / offsets
    int nseg;
    float4 *cand;        // detect: per-pixel candidate payload {m.x, m.y, xs, ys}
    double *red_part;    // reduction partials
    int red_cap;
    unsigned int *ticket;  // last-block-done counters
    void *pinned;        // small pinned host buffer for scalar read-back
    void *dev_small;     // small device buffer for scalar parameters / results (64 KiB, zero-initialised)
    float *boxtab;       // 6 x 64 reciprocal clipped-area tables (iimage::build_average), see dog.cu
    bool counters_preset; // set by rb_pipeline: match / regularise counters are zeroed by k_frame_pre
    int dog_sub;         // frames per scale-space sub-batch, env REBVO_B200_DOG_SUB (0 = whole batch, the default)
    bool pdl;            // programmatic dependent launch of the per-frame chain (env REBVO_B200_PDL=0 disables)
    bool min_persist;    // whole Minimizer_RV in one launch (env REBVO_B200_MIN_PERSIST=0: one launch per evaluation)
    bool min_cluster;    // Minimizer_RV in one 16-CTA cluster (min_cluster.cuh); env REBVO_B200_MIN_CLUSTER=0 disables
    int min_cluster_kpc; // keylines per CTA its shared memory is sized for (0: not available on this device / capacity)
    size_t min_cluster_dyn;
    int min_cluster_g;   // clusters per minimisation (env REBVO_B200_MIN_G, default 4; 1 = one cluster, co-residency guaranteed)
    int min_cluster_kpc_multi;
    size_t min_cluster_dyn_multi;
    int min_debug_abort;
    bool mu_xchg;        // env REBVO_B200_MU_XCHG (default 1): st.async all-reduce in k_map_update's rescaling iterations
    bool min_early;      // set by rb_pipeline around its Minimizer_RV launch: operands may be staged before the PDL wait  // test hook (env REBVO_B200_MIN_FORCE_ABORT=1): the kernel raises its abort flag at once
    int min_cluster_xchg; // 1: st.async + mbarrier exchange, 0: DSMEM stores + barrier.cluster (env REBVO_B200_MIN_XCHG)
    int row_ns;          // env REBVO_B200_ROW_NS: depth of the TMA tile ring of the row passes (0 = default 4)
    int colscan_mode;    // env REBVO_B200_COLSCAN: 1 = unpipelined column pass
    int rowscan_mode;    // env REBVO_B200_ROWSCAN: 1 = register-prefetch kernel, 2 = cp.async shared-memory ring
};
// layout of rb_ctx::dev_small / pinned (byte offsets)
#define RB_DS_REEST 0        // int[2 + nbins + 1]  reEstimateThresh min/max bits + histogram
#define RB_DS_CHAIN 32768    // DetChain for the single-map detect API
#define RB_DS_ARGS 36864     // argument / result staging of the stage-level API (4 KiB)
#define RB_DS_TMA_FAIL 45056 // int: a TMA-staged kernel timed out waiting for its tile (checked by the tests)
#define RB_DS_QHISTO 49152   // int[nbins] EstimateQuantile histogram (kept zero between calls)

// Levenberg-Marquardt variables of Minimizer_RV (global_tracker.cpp:596-625), resident in device memory so
// that the ~12 dependent TryVelRot evaluations of a frame run back to back without host round trips.
struct LMState {
    // request for the next evaluation
    double Xeval[6];
    int res_in, res_out;  // indices into rb_map::res[3] (Res0, Res1, Rest); res_in < 0: none
    // configuration of this minimisation
    double max_r;         // global_tracker::max_r (search radius of the field)
    double match_thresh, s_rho_min, k_huber;
    unsigned int match_num_thresh, frame_count;
    int iter_max, init_type, init_iter;
    double Vel_in[3], W0_in[3];
    // LM variables
    double X[6], Xnew[6], Xt[6], h[6];
    double JtJ[36], JtF[6], JtJn[36], JtFn[6];
    double F, Fnew, F0, Ft, F0t, u, v, ut, vt, gain;
    int eff_steps, eff_steps_t;
    int iR, iRN, iRt;     // Residual, ResidualNew, Rest
    int n_eval;
    // results
    double Vel[3], W0[3], RVel[9], RW0[9], W_X[36];
    double rel_error, rel_error_score, score;
    double last_score;    // score of the most recent evaluation
    int no_keylines, pad_;   // Minimizer_RV returned at once ("if(klist.KNum()<=0) return 0", :601): outputs are not valid
};

struct TrackState {
    LMState lm;
    int *blk_has;
    double *blk_last_fi;  // per block: residual of its last matched keyline
    double *partials;     // per block x 28 reduction partials
    double *carry;        // [3][256]: per residual buffer and block, the stale-fi value its leading misses inherit
    int nblk;
    struct MinCtl *ctl;   // request slots / sequence base of the persistent minimiser kernel
    unsigned long long *ll;   // its inter-cluster slots
    // scratch for FordwardMatch / Regularize_1_iter
    struct FmBest *fm_best;   // per new keyline: the old keyline that wins it (see d_fm_offer)
    double *reg_r, *reg_s;
    unsigned char *reg_set;
};


struct rb_map {
    rb_ctx *c;
    DogWS ws;            // own workspace (B = 1), allocated lazily
    bool owns_ws;
    float *img0, *dog;   // planes the detector reads (own ws or a slot of a batched ws)
    int *mask;           // Image<int> img_mask_kl
    unsigned long long *field;  // packed {dist<<32 | ~ikl}, ~0 = empty
    KLSoA kl;
    MapState *st;        // device
    double *res[3];      // minimiser residual buffers Res0, Res1, Rest
    unsigned char *carry_flag[3];
    TrackState *ts;      // device-resident LM state of this slot's global_tracker
    TrackState ts_host;  // host copy of the pointers inside *ts
    int field_radius;
    int det_r;           // plane-fit radius of this map's last detect (0: none yet, the mask is all -1)
};

// Every stage-level entry point starts with RB_ENTER(ctx): the calls of one context share its stream and its pinned /
// device staging areas, and the reference's detector thread and tracker thread call into the library concurrently
// (include/UtilLib/pipeline.h:42-89 only serialises per ring slot).  The lock makes each call atomic with respect to the
// context; it also selects the context's device for the calling thread.
#define RB_ENTER(ctxp)                                                \
    std::lock_guard<std::recursive_mutex> rb_lock__(*(ctxp)->mtx);    \
    cudaSetDevice((ctxp)->device)

#define RB_CUDA(call)                                                                          \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            snprintf(c->err, sizeof(c->err), "%s:%d %s: %s", __FILE__, __LINE__, #call,        \
                     cudaGetErrorString(e__));                                                 \
            return RB_ERR_CUDA;                                                                \
        }                                                                                      \
    } while (0)

#define RB_LAUNCH_CHECK()                                                                      \
    do {                                                                                       \
        c->launches++;                                                                         \
        cudaError_t e__ = cudaGetLastError();                                                  \
        if (e__ != cudaSuccess) {                                                              \
            snprintf(c->err, sizeof(c->err), "%s:%d launch: %s", __FILE__, __LINE__,           \
                     cudaGetErrorString(e__));                                                 \
            return RB_ERR_CUDA;                                                                \
        }                                                                                      \
    } while (0)

static inline int rb_div_up(int a, int b) { return (a + b - 1) / b; }

// ---- programmatic dependent launch (PDL) -----------------------------------------------------------
// The per-frame chain is ~10 short dependent kernels; with plain stream order each pays the full launch latency after
// its predecessor drains.  Kernels of the chain start with pdl_wait() + pdl_launch(): launched through RB_KLAUNCH
// (programmatic stream serialization), the next grid is set up and resident while this one runs and only waits at
// griddepcontrol.wait for this grid to complete (memory flushed).  Without the launch attribute both instructions
// are no-ops, so the stage-level API can launch the same kernels the ordinary way.
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
template <typename... KArgs, typename... Args>
static inline cudaError_t rb_klaunch(bool pdl, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                     cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#define RB_KLAUNCH(kernel, grid, block, smem, ...)                                                  \
    do {                                                                                            \
        c->launches++;                                                                              \
        cudaError_t e__ = rb_klaunch(c->pdl, kernel, dim3(grid), dim3(block), smem, c->stream, __VA_ARGS__); \
        if (e__ != cudaSuccess) {                                                                   \
            snprintf(c->err, sizeof(c->err), "%s:%d launch: %s", __FILE__, __LINE__,                \
                     cudaGetErrorString(e__));                                                      \
            return RB_ERR_CUDA;                                                                     \
        }                                                                                           \
    } while (0)
#endif

// ---- stage entry points (host side, enqueue on c->stream) ------------------------------------------
// dog.cu
int rb_dogws_alloc(rb_ctx *c, DogWS *ws, int B);
void rb_dogws_free(DogWS *ws);
int rb_dog_gray(rb_ctx *c, DogWS *ws, int nimg, const void *const *src_pp = nullptr);   // rgb -> gray
int rb_dog_gray_mono(rb_ctx *c, DogWS *ws, int nimg, const void *const *src_pp = nullptr);   // mono -> gray
int rb_dog_build_batch(rb_ctx *c, DogWS *ws, int nimg);          // gray -> img0, dog
int rb_dog_build_range(rb_ctx *c, DogWS *ws, int f0, int m);     // the same for the images [f0, f0 + m)
int rb_dog_aux_planes(rb_ctx *c, DogWS *ws, int img);            // Img(1), dx, dy into ws->aux
int rb_dog_make_tables(rb_ctx *c);
int rb_dog_make_tmaps(rb_ctx *c, DogWS *ws);
int rb_dog_device_setup(rb_ctx *c);
// detect.cu
int rb_detect_enqueue(rb_ctx *c, rb_map *m, const float *img0, const float *dog,
                      const rb_detect_params *p, DetChain *chain_dev);
int rb_reestimate_enqueue(rb_ctx *c, rb_map *m, int knum, int nbins);

// pipeline.cu -- the per-frame flow of REBVO with every piece of state resident on the device:
//   detector stage  = REBVO::FirstThr   (src/rebvo/rebvo_first_t.cpp:259-272)
//   tracker/mapper  = REBVO::SecondThread, ImuMode=0 branch (src/rebvo/rebvo_second_t.cpp:128-629)
// The host only enqueues kernels: threshold feedback, LM driver, NaN / match-count decisions, pose
// integration and the NavData record are all computed by 1-thread kernels from device state, so a batch of
// frames costs one H2D copy, one stream of launches and one D2H copy of the nav records.
#include <math.h>
#include <stdlib.h>
#include <new>

#include "common.cuh"
#include "lm.cuh"
#include "tracker.cuh"
#include "frame.cuh"

int rb_map_alloc(rb_ctx *c, rb_map **out, bool with_ws);

// SecondThread locals (rebvo_second_t.cpp:57-66, 167-169)
#define RB_NMAPS 3

// Device-side timeline for profiling builds (-DRB_TVR_PROF): marker kernels stamp %globaltimer, so that the overlap of
// the two streams can be read back from a graph replay (no nsys in this image).  Compiled out of the product.
#ifdef RB_TVR_PROF
__device__ unsigned long long g_trace[8192];
__device__ unsigned int g_trace_n;
__global__ void k_trace_mark(int tag) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    const unsigned int k = atomicAdd(&g_trace_n, 1u);
    if (k < 8192) g_trace[k] = ((unsigned long long)tag << 56) | (t & 0x00FFFFFFFFFFFFFFull);
}
extern "C" int rb_debug_fetch_trace(unsigned long long *out, unsigned int *n) {
    cudaMemcpyFromSymbol(n, g_trace_n, sizeof(unsigned int));
    cudaMemcpyFromSymbol(out, g_trace, sizeof(unsigned long long) * 8192);
    unsigned int z = 0;
    return (int)cudaMemcpyToSymbol(g_trace_n, &z, sizeof(z));
}
#define RB_TRACE(stream, tag) k_trace_mark<<<1, 1, 0, stream>>>(tag)
#else
#define RB_TRACE(stream, tag) do { } while (0)
#endif

struct ImuFlow;
struct rb_pipeline {
    rb_ctx *c;
    ImuFlow *imu;         // IMU mode (rb_pipeline_set_imu), nullptr otherwise
    rb_params p;
    int max_batch;
    DogWS ws;
    rb_map *maps[RB_NMAPS];   // ring: frame f lives in maps[f % RB_NMAPS]
    // detector stream: detect(f+1) (+ reEstimateThresh) runs beside the tracker/mapper of frame f; the third map is
    // what lets it write while frame f still reads map f-1
    cudaStream_t det_stream;
    cudaEvent_t ev_dog, *ev_det, *ev_trk;
    bool overlap;
    bool q_fold;          // EstimateQuantile + loop-body start of the next frame folded into this frame's map-update kernel
    int ss_sub;           // frames per scale-space sub-batch built on the detector stream (env REBVO_B200_SS_SUB, 0 = whole batch)
    bool map_fused;       // gate + Regularize_1_iter + EKF inside the map-update cluster kernel (env REBVO_B200_MAP_FUSED)
    // FordwardMatch's apply + directed_matching in k_match, then gate + Regularize_1_iter + EKF + rotate_keylines in
    // k_reg_ekf (env REBVO_B200_MAP_CHAIN=0: the four-kernel chain).  Not with map_fused, whose kernel reads the new map's
    // rho after matching, which k_match leaves in the regularisation scratch.
    bool map_chain;
    // rescaling stream: with DoReScaling=0 a frame's EstimateReScalingOpt changes no keyline and only fills in its nav record,
    // so it runs here (lowest priority) instead of at the end of the frame's tracker chain; the tracker stream joins it
    // before the next frame's first kernel after the minimiser (k_match, or k_fm_apply_rotate in the four-kernel chain,
    // which writes the map's rho / s_rho)
    cudaStream_t resc_stream;     // nullptr: the rescaling stays in the frame's map-update kernel on the tracker stream
    cudaEvent_t ev_rfork, ev_rjoin;
    bool resc_open;               // a rescaling was forked and not joined yet
    // host-input pushes are cut into a short head and the rest: the H2D copy of the rest (copy stream) runs beside the
    // kernels of the head.  The gray kernel reads its source through rgb_src_dev, so one graph serves every region.
    cudaStream_t copy_stream;
    cudaEvent_t *ev_copy;
    const void **rgb_src_dev;     // device: pointer to the RGB24 (or mono) frames of the sub-batch being processed
    const void **rgb_src_pin;     // pinned: one pointer per sub-batch of the current push
    int sub;                      // head sub-batch of a host-input push (env REBVO_B200_SUB, default 8 frames)
    DetChain *chain;      // device
    FrameState *fs;       // device
    rb_nav *nav_dev;
    rb_nav *nav_pin;
    int *abort_pin;       // pinned: abort flags of the three maps' minimisers, read back with every push
    uint8_t *rgb_pin;     // optional pinned staging (unused when the caller's buffer is pinned)
    long long n_pushed;   // frames pushed so far
    double t_prev;
    cudaEvent_t ev[4];
    cudaEvent_t user_ev[8];
    float stage_ms[6];
    struct FrameArgs *fa_dev, *fa_pin;
    // one instantiated CUDA graph per (input format, ring phase of the first frame, batch size): the kernel sequence of a
    // batch is static once the per-frame scalars live in fa_dev
    cudaGraphExec_t *gexec;       // [RB_NFMT * RB_NMAPS * (max_batch + 1)], see graph_slot
    int *glaunches;               // kernel launches inside each graph
    bool use_graph;
    // optional in-situ stage profile (REBVO_B200_STAGE_PROF=1, forces eager launches): CUDA events between stages
    bool prof_on;
    cudaEvent_t *pev;
    int *ptag;
    int pcap, pn;
    double pacc[16];
    long long pframes;
    // optional per-frame host mirror of the edge map (rb_pipeline_set_mirror): every frame's keylines are packed into a device
    // staging slot right after its map update (tracker stream), then a small kernel on mirror_stream writes exactly kn records
    // into mapped pinned host memory while the next frames are tracked; both are part of the captured batch
    int mirror_on;                                // 0 off, 1 = 168-byte KeyLine records, 2 = 15-byte net_keyline records
    size_t mirror_rec, mirror_stride;             // bytes per record / per frame slot (multiple of 256)
    unsigned char *mirror_dev, *mirror_host;      // [max_batch * mirror_stride]: device staging, mapped pinned host memory
    unsigned char **mirror_base_dev;              // device: {staging, host} address of frame 0 of the sub-batch being processed
    unsigned char **mirror_base_pin;              // pinned: one pair per sub-batch of the current push
    cudaStream_t mirror_stream;
    cudaEvent_t *ev_mpack, ev_mjoin;
    int mirror_n;                                 // frames of the last push
    rb_undistort *und;                            // UseUndistort=1 (rb_pipeline_set_undistort): fused into the gray pass
};

int rb_undistort_gray_enqueue(rb_undistort *u, const void *const *src_pp, float *gray, int nimg);
int rb_undistort_gray_mono_enqueue(rb_undistort *u, const void *const *src_pp, float *gray, int nimg);

// input formats of a push: RGB24 (3 bytes per pixel) or mono8, which stands for the RGB24 frame (m, m, m)
enum { RB_IN_RGB = 0, RB_IN_MONO = 1, RB_NFMT = 2 };
static inline size_t frame_bytes(const rb_ctx *c, int fmt) { return (fmt == RB_IN_MONO ? (size_t)1 : (size_t)3) * c->N; }
static inline int graph_slots(const rb_pipeline *pl) { return RB_NFMT * RB_NMAPS * (pl->max_batch + 1); }
static inline int graph_slot(const rb_pipeline *pl, int fmt, int phase, int n) {
    return (fmt * RB_NMAPS + phase) * (pl->max_batch + 1) + n;
}
// captured batches contain the gray kernel, the undistortion and the mirror's pack kernels: drop them all
static void drop_graphs(rb_pipeline *pl) {
    for (int i = 0; i < graph_slots(pl); i++)
        if (pl->gexec[i]) {
            cudaGraphExecDestroy(pl->gexec[i]);
            pl->gexec[i] = nullptr;
        }
}
// the batch's gray plane from the frames at *rgb_src_dev (rebvo_first_t.cpp:231 undistortion + RGB -> BW)
static int gray_pass(rb_pipeline *pl, int fmt, int n) {
    if (pl->und)
        return fmt == RB_IN_MONO ? rb_undistort_gray_mono_enqueue(pl->und, pl->rgb_src_dev, pl->ws.gray, n)
                                 : rb_undistort_gray_enqueue(pl->und, pl->rgb_src_dev, pl->ws.gray, n);
    return fmt == RB_IN_MONO ? rb_dog_gray_mono(pl->c, &pl->ws, n, pl->rgb_src_dev)
                             : rb_dog_gray(pl->c, &pl->ws, n, pl->rgb_src_dev);
}
#include "imu_flow.cuh"

enum { ST_H2D = 0, ST_GRAY, ST_DOG, ST_DETECT, ST_REEST, ST_FIELD, ST_MINIM, ST_FWD_ROT, ST_DMATCH, ST_REG_EKF, ST_RESCALE,
       ST_FINISH, ST_NAV };
static inline void prof_mark(rb_pipeline *pl, int tag) {
    if (!pl->prof_on || pl->pn >= pl->pcap) return;
    cudaEventRecord(pl->pev[pl->pn], pl->c->stream);
    pl->ptag[pl->pn++] = tag;
}

int rb_dog_single_pass(rb_ctx *c, DogWS *ws, int pass_id, int nimg, double *bytes);
int rb_map_pack_aos_enqueue(rb_ctx *c, rb_map *m, unsigned char *const *base, size_t offset_bytes);
int rb_map_pack_net_enqueue(rb_ctx *c, rb_map *m, unsigned char *const *base, size_t offset_bytes, const double *k_prof);

// staging slot -> mapped pinned host memory: exactly kn records, 16-byte stores (posted writes over PCIe)
__global__ void __launch_bounds__(256) k_mirror_to_host(unsigned char *const *bases, size_t offset, const int *kn_p, int rec) {
    const size_t nbytes = (size_t)(*kn_p > 0 ? *kn_p : 0) * rec;
    const uint4 *src = reinterpret_cast<const uint4 *>(bases[0] + offset);
    uint4 *dst = reinterpret_cast<uint4 *>(bases[1] + offset);
    const size_t n16 = nbytes >> 4;
    for (size_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n16; k += (size_t)gridDim.x * blockDim.x) dst[k] = src[k];
    if (blockIdx.x == 0 && threadIdx.x < (nbytes & 15))
        bases[1][offset + (n16 << 4) + threadIdx.x] = bases[0][offset + (n16 << 4) + threadIdx.x];
}
int rb_read_map_state(rb_map *m, MapState *host);

static void set_eye(double *M, double v) {
    for (int i = 0; i < 9; i++) M[i] = 0;
    M[0] = M[4] = M[8] = v;
}

__global__ void k_frame_pre(FrameState *fs, const FrameArgs *fa, MapState *nst) { d_frame_pre(fs, fa->frame_count, nst); }
__global__ void k_frame_post_min(FrameState *fs, const TrackState *ts) { d_frame_post_min(fs, ts->lm); }
__global__ void k_frame_post_match(FrameState *fs, const MapState *nst, int match_threshold) {
    d_frame_post_match(fs, nst, match_threshold);
}
__global__ void k_frame_finish(FrameState *fs, const MapState *nst, const MapState *ost, const TrackState *ts,
                               rb_nav *nav, const FrameArgs *fa) {
    d_frame_finish(fs, nst, ost, ts->lm.score, nav, fa, true);
}

// record for the very first frame (it only initialises the ring, :109-121)
__global__ void k_frame_first(const FrameState *fs, const MapState *nst, rb_nav *nav, const FrameArgs *fa) {
    rb_nav o;
    memset(&o, 0, sizeof(o));
    o.t = fa->t;
    for (int i = 0; i < 9; i++) {
        o.Rot[i] = (i % 4 == 0) ? 1 : 0;
        o.Pose[i] = fs->Pose[i];
    }
    o.K = fs->K;
    o.Kp = fs->Kp;
    o.RKp = fs->P_Kp;
    o.kn = nst->kn;
    o.estimation_ok = 0;
    o.thresh = nst->thresh_used;
    o.retuned_thresh = nst->retuned;
    *nav = o;
}

static int pl_reset_state(rb_pipeline *pl) {
    rb_ctx *c = pl->c;
    FrameState h;
    memset(&h, 0, sizeof(h));
    set_eye(h.R, 1);
    set_eye(h.Pose, 1);
    set_eye(h.P_V, 1e50);
    set_eye(h.P_W, 1e-10);
    h.Kp = 1;
    h.K = 1;
    h.P_Kp = 5e-6;
    RB_CUDA(cudaMemcpy(pl->fs, &h, sizeof(h), cudaMemcpyHostToDevice));
    DetChain ch;
    ch.tresh = pl->p.DetectorThresh;
    ch.l_kl_num = 0;
    ch.pad = 0;
    RB_CUDA(cudaMemcpy(pl->chain, &ch, sizeof(ch), cudaMemcpyHostToDevice));
    for (int k = 0; k < RB_NMAPS; k++)
        if (pl->maps[k]) RB_CUDA(cudaMemset(&pl->maps[k]->ts_host.ctl->abort, 0, sizeof(int)));
    if (pl->imu) imu_flow_reset(*pl->imu);
    pl->n_pushed = 0;
    pl->t_prev = 0;
    return RB_OK;
}

extern "C" int rb_pipeline_create(rb_pipeline **out, int device, const rb_params *p, int max_batch) {
    if (!out || !p || max_batch < 1) return RB_ERR_ARG;
    *out = nullptr;
    // the detector's check, at creation: a bad DetectorPlaneFitSize must not surface at the first push
    if (p->det.plane_fit_size < 1 || p->det.plane_fit_size > RB_PLANE_FIT_MAX) return RB_ERR_ARG;
    rb_ctx *c = nullptr;
    int kcap = p->kl_capacity > 0 ? p->kl_capacity : 50000;
    int r = rb_ctx_create(&c, device, &p->cam, p->Sigma0, p->KSigma, kcap);
    if (r) {
        if (c) rb_ctx_destroy(c);
        return r;
    }
    rb_pipeline *pl = new (std::nothrow) rb_pipeline;
    if (!pl) {
        rb_ctx_destroy(c);
        return RB_ERR_ARG;
    }
    memset(pl, 0, sizeof(*pl));
    pl->c = c;
    c->counters_preset = true;
    pl->p = *p;
    pl->max_batch = max_batch;
    *out = pl;
    if ((r = rb_dogws_alloc(c, &pl->ws, max_batch))) return r;
    for (int i = 0; i < RB_NMAPS; i++)
        if ((r = rb_map_alloc(c, &pl->maps[i], false))) return r;
    RB_CUDA(cudaMalloc(&pl->chain, sizeof(DetChain)));
    RB_CUDA(cudaMalloc(&pl->fs, sizeof(FrameState)));
    RB_CUDA(cudaMalloc(&pl->nav_dev, sizeof(rb_nav) * max_batch));
    RB_CUDA(cudaMallocHost(&pl->nav_pin, sizeof(rb_nav) * max_batch));
    RB_CUDA(cudaMallocHost(&pl->abort_pin, sizeof(int) * RB_NMAPS));
    memset(pl->abort_pin, 0, sizeof(int) * RB_NMAPS);
    RB_CUDA(cudaMalloc(&pl->fa_dev, sizeof(FrameArgs) * max_batch));
    RB_CUDA(cudaMallocHost(&pl->fa_pin, sizeof(FrameArgs) * max_batch));
    pl->gexec = new (std::nothrow) cudaGraphExec_t[graph_slots(pl)];
    pl->glaunches = new (std::nothrow) int[graph_slots(pl)];
    if (!pl->gexec || !pl->glaunches) return RB_ERR_ARG;
    for (int i = 0; i < graph_slots(pl); i++) {
        pl->gexec[i] = nullptr;
        pl->glaunches[i] = 0;
    }
    const char *ng = getenv("REBVO_B200_NO_GRAPH");
    pl->use_graph = !(ng && ng[0] == '1');
    const char *sp = getenv("REBVO_B200_STAGE_PROF");
    pl->prof_on = sp && sp[0] == '1';
    if (pl->prof_on) {
        pl->use_graph = false;
        pl->pcap = max_batch * 12 + 8;
        pl->pev = new (std::nothrow) cudaEvent_t[pl->pcap];
        pl->ptag = new (std::nothrow) int[pl->pcap];
        if (!pl->pev || !pl->ptag) return RB_ERR_ARG;
        for (int i = 0; i < pl->pcap; i++) RB_CUDA(cudaEventCreate(&pl->pev[i]));
    }
    {
        const char *mf = getenv("REBVO_B200_MAP_FUSED");
        pl->map_fused = mf ? atoi(mf) != 0 : false;   // off by default: the wide kernels under PDL serve
        const char *mc = getenv("REBVO_B200_MAP_CHAIN");
        pl->map_chain = !(mc && atoi(mc) == 0) && !pl->map_fused;
        const char *ov = getenv("REBVO_B200_OVERLAP");
        pl->overlap = !(ov && ov[0] == '0') && !pl->prof_on;
        // (off by default: the launch it saves is already hidden by programmatic dependent launch, and it costs the
        // minimiser its early operand staging)
        pl->q_fold = getenv("REBVO_B200_Q_FOLD") && atoi(getenv("REBVO_B200_Q_FOLD")) != 0 && p->QCutOffNumBins >= 1 &&
                     p->QCutOffNumBins <= 128;
        pl->ss_sub = getenv("REBVO_B200_SS_SUB") ? atoi(getenv("REBVO_B200_SS_SUB")) : 0;
        if (pl->ss_sub < 4) pl->ss_sub = 0;   // (a sub-batch must cover the frames the detector runs ahead)
        pl->ev_det = new (std::nothrow) cudaEvent_t[max_batch];
        pl->ev_trk = new (std::nothrow) cudaEvent_t[max_batch];
        if (!pl->ev_det || !pl->ev_trk) return RB_ERR_ARG;
        memset(pl->ev_det, 0, sizeof(cudaEvent_t) * max_batch);
        memset(pl->ev_trk, 0, sizeof(cudaEvent_t) * max_batch);
        RB_CUDA(cudaStreamCreateWithFlags(&pl->det_stream, cudaStreamNonBlocking));
        RB_CUDA(cudaStreamCreateWithFlags(&pl->copy_stream, cudaStreamNonBlocking));
        const char *sb = getenv("REBVO_B200_SUB");
        pl->sub = sb ? atoi(sb) : 8;
        if (pl->sub < 1) pl->sub = max_batch;
        pl->ev_copy = new (std::nothrow) cudaEvent_t[max_batch];
        if (!pl->ev_copy) return RB_ERR_ARG;
        memset(pl->ev_copy, 0, sizeof(cudaEvent_t) * max_batch);
        for (int i = 0; i < max_batch; i++) RB_CUDA(cudaEventCreateWithFlags(&pl->ev_copy[i], cudaEventDisableTiming));
        RB_CUDA(cudaMalloc(&pl->rgb_src_dev, sizeof(void *)));
        RB_CUDA(cudaMallocHost(&pl->rgb_src_pin, sizeof(void *) * max_batch));
        RB_CUDA(cudaEventCreateWithFlags(&pl->ev_dog, cudaEventDisableTiming));
        for (int i = 0; i < max_batch; i++) {
            RB_CUDA(cudaEventCreateWithFlags(&pl->ev_det[i], cudaEventDisableTiming));
            RB_CUDA(cudaEventCreateWithFlags(&pl->ev_trk[i], cudaEventDisableTiming));
        }
        // (the inline schedule where the rescaled keylines feed the next frame, the next quantile is folded into the
        // map-update kernel, the map update is fused, or everything runs on one stream)
        if (pl->overlap && !pl->q_fold && !pl->map_fused && p->DoReScaling <= 0) {
            int lo = 0, hi = 0;
            RB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
            RB_CUDA(cudaStreamCreateWithPriority(&pl->resc_stream, cudaStreamNonBlocking, lo));   // minimiser blocks first
            RB_CUDA(cudaEventCreateWithFlags(&pl->ev_rfork, cudaEventDisableTiming));
            RB_CUDA(cudaEventCreateWithFlags(&pl->ev_rjoin, cudaEventDisableTiming));
        }
    }
    for (int i = 0; i < 4; i++) RB_CUDA(cudaEventCreate(&pl->ev[i]));
    for (int i = 0; i < 8; i++) RB_CUDA(cudaEventCreate(&pl->user_ev[i]));
    if ((r = pl_reset_state(pl))) return r;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

extern "C" int rb_pipeline_set_imu(rb_pipeline *pl, const rb_imu_params *ip, const double *samples, int n) {
    if (!pl || !ip || !samples || n < 2) return RB_ERR_ARG;
    if (!pl->imu) pl->imu = new (std::nothrow) ImuFlow();
    if (!pl->imu) return RB_ERR_ARG;
    ImuFlow &f = *pl->imu;
    f.ip = *ip;
    f.samples.resize(n);
    for (int i = 0; i < n; i++) {
        f.samples[i].t = samples[i * 7];
        for (int k = 0; k < 3; k++) {
            f.samples[i].giro[k] = samples[i * 7 + 1 + k];
            f.samples[i].acel[k] = samples[i * 7 + 4 + k];
        }
    }
    f.enabled = true;
    imu_flow_reset(f);
    return RB_OK;
}

extern "C" void rb_pipeline_destroy(rb_pipeline *pl) {
    if (!pl) return;
    rb_ctx *c = pl->c;
    delete pl->imu;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (pl->det_stream) cudaStreamSynchronize(pl->det_stream);
    if (pl->resc_stream) cudaStreamSynchronize(pl->resc_stream);
    for (int i = 0; i < RB_NMAPS; i++)
        if (pl->maps[i]) rb_map_destroy(pl->maps[i]);
    if (pl->ev_dog) cudaEventDestroy(pl->ev_dog);
    for (int i = 0; i < pl->max_batch; i++) {
        if (pl->ev_det && pl->ev_det[i]) cudaEventDestroy(pl->ev_det[i]);
        if (pl->ev_trk && pl->ev_trk[i]) cudaEventDestroy(pl->ev_trk[i]);
    }
    delete[] pl->ev_det;
    delete[] pl->ev_trk;
    if (pl->det_stream) cudaStreamDestroy(pl->det_stream);
    if (pl->resc_stream) cudaStreamDestroy(pl->resc_stream);
    if (pl->ev_rfork) cudaEventDestroy(pl->ev_rfork);
    if (pl->ev_rjoin) cudaEventDestroy(pl->ev_rjoin);
    if (pl->copy_stream) {
        cudaStreamSynchronize(pl->copy_stream);
        cudaStreamDestroy(pl->copy_stream);
    }
    for (int i = 0; i < pl->max_batch; i++)
        if (pl->ev_copy && pl->ev_copy[i]) cudaEventDestroy(pl->ev_copy[i]);
    delete[] pl->ev_copy;
    cudaFree(pl->rgb_src_dev);
    if (pl->rgb_src_pin) cudaFreeHost(pl->rgb_src_pin);
    if (pl->mirror_stream) {
        cudaStreamSynchronize(pl->mirror_stream);
        cudaStreamDestroy(pl->mirror_stream);
    }
    if (pl->und) rb_undistort_destroy(pl->und);
    cudaFree(pl->mirror_dev);
    if (pl->mirror_host) cudaFreeHost(pl->mirror_host);
    for (int i = 0; i < pl->max_batch; i++)
        if (pl->ev_mpack && pl->ev_mpack[i]) cudaEventDestroy(pl->ev_mpack[i]);
    delete[] pl->ev_mpack;
    if (pl->ev_mjoin) cudaEventDestroy(pl->ev_mjoin);
    cudaFree(pl->mirror_base_dev);
    if (pl->mirror_base_pin) cudaFreeHost(pl->mirror_base_pin);
    rb_dogws_free(&pl->ws);
    cudaFree(pl->chain);
    cudaFree(pl->fs);
    cudaFree(pl->nav_dev);
    if (pl->nav_pin) cudaFreeHost(pl->nav_pin);
    if (pl->abort_pin) cudaFreeHost(pl->abort_pin);
    cudaFree(pl->fa_dev);
    if (pl->fa_pin) cudaFreeHost(pl->fa_pin);
    if (pl->gexec) {
        for (int i = 0; i < graph_slots(pl); i++)
            if (pl->gexec[i]) cudaGraphExecDestroy(pl->gexec[i]);
        delete[] pl->gexec;
    }
    delete[] pl->glaunches;
    for (int i = 0; i < 4; i++)
        if (pl->ev[i]) cudaEventDestroy(pl->ev[i]);
    for (int i = 0; i < 8; i++)
        if (pl->user_ev[i]) cudaEventDestroy(pl->user_ev[i]);
    rb_ctx_destroy(c);
    delete pl;
}

extern "C" const char *rb_pipeline_last_error(const rb_pipeline *pl) { return pl ? pl->c->err : "null pipeline"; }
extern "C" int64_t rb_pipeline_launch_count(const rb_pipeline *pl) { return pl->c->launches; }
extern "C" void *rb_pipeline_stream(rb_pipeline *pl) { return (void *)pl->c->stream; }
extern "C" rb_map *rb_pipeline_map(rb_pipeline *pl, int age) {
    if (age < 0 || age > 1 || pl->n_pushed <= age) return nullptr;
    return pl->maps[(pl->n_pushed - 1 - age) % RB_NMAPS];
}
extern "C" int rb_pipeline_stage_ms(const rb_pipeline *pl, float out[6]) {
    memcpy(out, pl->stage_ms, sizeof(float) * 6);
    return RB_OK;
}

extern "C" int rb_pipeline_reset(rb_pipeline *pl) {
    rb_ctx *c = pl->c;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return pl_reset_state(pl);
}

// the tracker stream waits for the rescaling forked by the previous frame (or of the batch's last frame)
static int resc_join(rb_pipeline *pl) {
    rb_ctx *c = pl->c;
    if (!pl->resc_open) return RB_OK;
    RB_CUDA(cudaStreamWaitEvent(c->stream, pl->ev_rjoin, 0));
    pl->resc_open = false;
    return RB_OK;
}

// one frame of the tracker/mapper stage: new = maps[f % RB_NMAPS] (already detected), old = the map of frame f-1
static int track_frame(rb_pipeline *pl, rb_map *neu, rb_map *old, rb_map *next, const FrameArgs *fa, rb_nav *nav_slot) {
    rb_ctx *c = pl->c;
    const rb_params &p = pl->p;
    int r;
    RB_TRACE(c->stream, 1);
    // :167-169 loop-body start (folded into the quantile kernel) ; :172  s_rho_q = old_buf.ef->EstimateQuantile(...)
    // (q_fold: both were done by the previous frame's map-update kernel, or after k_frame_first for frame 1)
    if (!pl->q_fold)
        if ((r = rb_quantile_enqueue(c, old, RB_RHO_MIN, RB_RHO_MAX, p.QCutOffQuantile, p.QCutOffNumBins, pl->fs,
                                     &fa->frame_count, neu->st)))
            return r;
    // :177  new_buf.gt->build_field(...) only needs the new edge map: enqueue_batch runs it on the detector stream, and
    // clears the new map's FordwardMatch arg-max scratch there, which the minimiser's last evaluation already fills
    // (the clear first: the minimiser stages its operands while the kernel before it runs, and build_field is the longer one)
    if (!pl->overlap) {
        if ((r = rb_forward_match_init_enqueue(c, neu))) return r;
        if ((r = rb_build_field_enqueue(c, neu, p.SearchRange, 0.f, true))) return r;
    }
    prof_mark(pl, ST_FIELD);
    // :346  Minimizer_RV<double>(V,W,P_V,P_W,*old_buf.ef,...) ; :346-398 outputs / NaN guard folded into its last block
    rb_minimizer_args a;
    a.match_thresh = p.TrackerMatchThresh;
    a.iter_max = p.TrackerIterNum;
    a.init_type = p.TrackerInitType;
    a.init_iter = p.TrackerInitIterNum;
    a.reweight_distance = p.ReweigthDistance;
    a.match_num_thresh = p.MatchNumThresh;
    // FrameCount comes from fa (written into neu->st by the folded loop-body start)
    RB_TRACE(c->stream, 2);
    bool folded = false;
    // (since the old map's update only EstimateQuantile -- and build_field of the NEW map without the second stream -- ran
    // on this stream: the minimiser may stage the old map's operands while that kernel is still running)
    // (with q_fold the previous kernel is the old map's update itself: no early staging)
    c->min_early = !pl->q_fold && (getenv("REBVO_B200_MIN_EARLY") ? atoi(getenv("REBVO_B200_MIN_EARLY")) != 0 : true);
    // (folded: the one-thread stage after the minimiser and FordwardMatch's arg-max ran in its epilogue / last evaluation)
    r = rb_minimizer_enqueue(c, neu, old, pl->fs->VW, &a, 0.0, true, 0, true, pl->fs, &folded);
    c->min_early = false;
    if (r) return r;
    RB_TRACE(c->stream, 3);
    prof_mark(pl, ST_MINIM);
    if (!folded) {
        k_frame_post_min<<<1, 1, 0, c->stream>>>(pl->fs, neu->ts);
        RB_LAUNCH_CHECK();
        if ((r = rb_forward_match_argmax_enqueue(c, old, neu))) return r;
    }
    // :480-487 EstimateReScalingOpt and :545-585 pose integration + NavData: in one cluster kernel (k_map_update) after the
    // EKF, or with the rescaling stream, pose integration + NavData ride in the EKF kernel and the rescaling leaves the chain.
    // (Not with the 168-byte keyline mirror: there the inline schedule measured 2-3 % faster on H100, while the 15-byte
    // records gain from the side stream like the plain push; set_mirror drops the captured batches.)
    const bool side = pl->resc_stream != nullptr && pl->mirror_on != 1;
    if (pl->map_chain) {
        // (the old map's rescaling is joined here although k_match only reads that map: joining it before k_reg_ekf
        // instead measured no faster on H100)
        if ((r = resc_join(pl))) return r;
        // (the eager stage profile reports k_match under "directed_match", nothing under "fwdmatch+rotate", and
        // k_reg_ekf under "regularize+ekf")
        prof_mark(pl, ST_FWD_ROT);
        // :354  FordwardMatch + :410 directed_matching(V,P_V,R,old_buf.ef,...) against the old map before :369
        // rotate_keylines(R0), which k_reg_ekf runs; this kernel rotates the old keylines it probes itself
        if ((r = rb_match_enqueue(c, neu, old, &pl->fs->dm, pl->fs->R0, p.MatchThreshModule, p.MatchThreshAngle,
                                  (double)p.SearchRange, p.LocationUncertaintyMatch, &pl->fs->do_match)))
            return r;
        RB_TRACE(c->stream, 4);
        prof_mark(pl, ST_DMATCH);
        // :410-423 match-count gate + :452-470 Regularize_1_iter / UpdateInverseDepthKalman + :369 rotate_keylines
        if ((r = rb_reg_ekf_enqueue(c, neu, old, p.RegularizeThresh, pl->fs, p.MatchThreshold, p.ReshapeQAbsolute,
                                    p.LocationUncertainty, pl->fs->R0, side ? nav_slot : nullptr, fa)))
            return r;
    } else {
        // :354  FordwardMatch ; :369 rotate_keylines(R0) in one kernel.  Until then, this frame only reads the old map's
        // rho / s_rho (the minimiser writes its m_id_f, which the rescaling does not read): the old map's rescaling may
        // run until then.
        if ((r = resc_join(pl))) return r;
        if ((r = rb_forward_match_apply_enqueue(c, old, neu, pl->fs->R0))) return r;
        RB_TRACE(c->stream, 11);
        prof_mark(pl, ST_FWD_ROT);
        // :410  directed_matching(V,P_V,R,old_buf.ef,...)
        if ((r = rb_directed_matching_enqueue(c, neu, old, &pl->fs->dm, p.MatchThreshModule, p.MatchThreshAngle,
                                              (double)p.SearchRange, p.LocationUncertaintyMatch, &pl->fs->do_match)))
            return r;
        RB_TRACE(c->stream, 4);
        prof_mark(pl, ST_DMATCH);
        // :410-423 match-count gate + :452-470 Regularize_1_iter / UpdateInverseDepthKalman on wide grids (or in the
        // map-update kernel with map_fused)
        if (!pl->map_fused)
            if ((r = rb_regularize_ekf_enqueue(c, neu, p.RegularizeThresh, pl->fs, p.MatchThreshold, pl->fs->V,
                                               p.ReshapeQAbsolute, p.LocationUncertainty, &pl->fs->do_map,
                                               side ? old->st : nullptr, side ? nav_slot : nullptr, fa)))
                return r;
    }
    RB_TRACE(c->stream, 9);
    prof_mark(pl, ST_REG_EKF);
    if (side) {   // gated by the map's own copy of do_map; writes the map's Kp / RKp and the record's, no FrameState
        cudaStream_t main_stream = c->stream;
        RB_CUDA(cudaEventRecord(pl->ev_rfork, main_stream));
        RB_CUDA(cudaStreamWaitEvent(pl->resc_stream, pl->ev_rfork, 0));
        c->stream = pl->resc_stream;
        r = rb_rescale_enqueue(c, neu, RB_RHO_MAX, 1, 0, &neu->st->do_map, nav_slot);
        c->stream = main_stream;
        if (r) return r;
        RB_CUDA(cudaEventRecord(pl->ev_rjoin, pl->resc_stream));
        pl->resc_open = true;
        RB_TRACE(c->stream, 5);
        return RB_OK;
    }
    rb_quantile_fold qf = {pl->q_fold ? p.QCutOffNumBins : 0, RB_RHO_MIN, RB_RHO_MAX, p.QCutOffQuantile, next->st};
    if ((r = rb_map_update_enqueue(c, neu, p.RegularizeThresh, pl->fs->V, p.ReshapeQAbsolute, p.LocationUncertainty,
                                   RB_RHO_MAX, 1, p.DoReScaling > 0 ? 1 : 0, pl->fs, p.MatchThreshold, old->st,
                                   nav_slot, fa, pl->map_fused, &qf)))
        return r;
    prof_mark(pl, ST_RESCALE);   // rescaling + pose integration / nav record (folded)
    RB_TRACE(c->stream, 5);
    prof_mark(pl, ST_FINISH);
    return RB_OK;
}

// everything of a batch after the H2D copy: gray, batched scale space, then per frame detect + track + map
static int enqueue_batch(rb_pipeline *pl, int fmt, int n, long long first_frame, bool with_events) {
    rb_ctx *c = pl->c;
    const rb_params &p = pl->p;
    int r;
    pl->resc_open = false;   // (a batch joins its last rescaling at its end; a failed enqueue must not leave a join behind)
    prof_mark(pl, ST_H2D);
    if ((r = gray_pass(pl, fmt, n))) return r;
    prof_mark(pl, ST_GRAY);
    if (with_events) RB_CUDA(cudaEventRecord(pl->ev[1], c->stream));
    // The scale space of a batch is a serial prefix of its first frame.  With two
    // streams only the first ss_sub frames are built here; the detector stream builds the next sub-batch while the
    // tracker works on this one (it runs up to two frames ahead, more than a sub-batch costs).
    const int SB = (pl->overlap && pl->ss_sub > 0 && pl->ss_sub < n) ? pl->ss_sub : n;
    if (SB == n) r = rb_dog_build_batch(c, &pl->ws, n);
    else r = rb_dog_build_range(c, &pl->ws, 0, SB);
    if (r) return r;
    prof_mark(pl, ST_DOG);
    if (with_events) RB_CUDA(cudaEventRecord(pl->ev[2], c->stream));
    // Two streams, like the reference's first and second thread: the detector of frame f+1 only needs the scale space
    // and the previous detector state (threshold chain), so it runs on det_stream while the main stream tracks
    // frame f.  detect(f) overwrites the map of frame f-3, which track(f-2) was the last to read.
    cudaStream_t main_stream = c->stream;
    const bool ov = pl->overlap;
    if (ov) {
        RB_CUDA(cudaEventRecord(pl->ev_dog, main_stream));
        RB_CUDA(cudaStreamWaitEvent(pl->det_stream, pl->ev_dog, 0));
    }
    for (int i = 0; i < n; i++) {
        const long long fr = first_frame + i;
        rb_map *neu = pl->maps[fr % RB_NMAPS], *old = pl->maps[(fr + RB_NMAPS - 1) % RB_NMAPS];
        const float *img0 = pl->ws.img0 + (size_t)i * c->N, *dog = pl->ws.dog + (size_t)i * c->N;
        // FirstThr: detect + reEstimateThresh (rebvo_first_t.cpp:266-272)
        if (ov) {
            if (i >= 2) RB_CUDA(cudaStreamWaitEvent(pl->det_stream, pl->ev_trk[i - 2], 0));
            c->stream = pl->det_stream;
        }
        RB_TRACE(c->stream, 6);
        if (SB < n && i % SB == 2 && i - 2 + SB < n) {   // (after the detector has its two frames of lead)
            const int f0 = i - 2 + SB;
            if ((r = rb_dog_build_range(c, &pl->ws, f0, n - f0 < SB ? n - f0 : SB))) {
                c->stream = main_stream;
                return r;
            }
        }
        r = rb_detect_enqueue(c, neu, img0, dog, &p.det, pl->chain);
        prof_mark(pl, ST_DETECT);
        if (!r) r = rb_reestimate_enqueue(c, neu, p.TrackPoints, p.QCutOffNumBins);
        prof_mark(pl, ST_REEST);
        if (ov && fr > 0) {   // tracker inputs that only depend on the new edge map: distance field, arg-max scratch
            if (!r) r = rb_build_field_enqueue(c, neu, p.SearchRange, 0.f, true);
            if (!r) r = rb_forward_match_init_enqueue(c, neu);
        }
        RB_TRACE(c->stream, 7);
        c->stream = main_stream;
        if (r) return r;
        if (ov) {
            RB_CUDA(cudaEventRecord(pl->ev_det[i], pl->det_stream));
            RB_CUDA(cudaStreamWaitEvent(main_stream, pl->ev_det[i], 0));
        }
        if (fr == 0) {
            k_frame_first<<<1, 1, 0, c->stream>>>(pl->fs, neu->st, pl->nav_dev + i, pl->fa_dev + i);
            RB_LAUNCH_CHECK();
            if (pl->q_fold)   // what frame 1 starts with: EstimateQuantile of this map + its loop-body start
                if ((r = rb_quantile_enqueue(c, neu, RB_RHO_MIN, RB_RHO_MAX, p.QCutOffQuantile, p.QCutOffNumBins, pl->fs,
                                             &(pl->fa_dev + i)->next_frame_count, pl->maps[(fr + 1) % RB_NMAPS]->st)))
                    return r;
        } else {
            if ((r = track_frame(pl, neu, old, pl->maps[(fr + 1) % RB_NMAPS], pl->fa_dev + i, pl->nav_dev + i))) return r;
        }
        if (pl->mirror_on) {   // the frame's edge map as the reference's records, before the next frame touches it
            const size_t ofs = (size_t)i * pl->mirror_stride;
            if (pl->mirror_on == 1)
                r = rb_map_pack_aos_enqueue(c, neu, pl->mirror_base_dev, ofs);
            else   // copy_net_keyline(..., pbuf.K) of the third thread (rebvo_third_t.cpp:192-197): K of this frame's nav record
                r = rb_map_pack_net_enqueue(c, neu, pl->mirror_base_dev, ofs, &(pl->nav_dev + i)->K);
            if (r) return r;
            RB_CUDA(cudaEventRecord(pl->ev_mpack[i], main_stream));
            RB_CUDA(cudaStreamWaitEvent(pl->mirror_stream, pl->ev_mpack[i], 0));
            k_mirror_to_host<<<8, 256, 0, pl->mirror_stream>>>(pl->mirror_base_dev, ofs, &(pl->nav_dev + i)->kn, (int)pl->mirror_rec);
            RB_LAUNCH_CHECK();
        }
        if (ov && i + 2 < n) RB_CUDA(cudaEventRecord(pl->ev_trk[i], main_stream));
    }
    if ((r = resc_join(pl))) return r;   // the last frame's Kp / RKp are in its record before the nav copy
    if (pl->mirror_on) {   // the batch is complete when its last map has reached the host
        RB_CUDA(cudaEventRecord(pl->ev_mjoin, pl->mirror_stream));
        RB_CUDA(cudaStreamWaitEvent(main_stream, pl->ev_mjoin, 0));
    }
    return RB_OK;
}

// rgb: n frames of frame_bytes(fmt) each, host or device memory
static int push_impl(rb_pipeline *pl, const uint8_t *rgb, int fmt, bool on_device, const double *ts, int n,
                     rb_nav *nav_out) {
    rb_ctx *c = pl->c;
    const rb_params &p = pl->p;
    if (n < 1 || n > pl->max_batch || !rgb || !ts) return RB_ERR_ARG;
    // (the mono kernels read the frames as 32-bit words; the RGB kernels have a byte-wise path for unaligned buffers)
    if (fmt == RB_IN_MONO && on_device && (reinterpret_cast<uintptr_t>(rgb) & 3)) return RB_ERR_ARG;
    RB_CUDA(cudaSetDevice(c->device));
    int r;
    if (pl->imu) {   // IMU mode: host-driven frame loop (imu_flow.cuh)
        if ((r = imu_push(pl, *pl->imu, rgb, fmt, on_device, ts, n, pl->nav_pin))) return r;
        RB_CUDA(cudaStreamSynchronize(c->stream));
        if (nav_out) memcpy(nav_out, pl->nav_pin, sizeof(rb_nav) * n);
        return RB_OK;
    }
    const long long first = pl->n_pushed;
    // per-frame scalars -> device (SecondThread :146-149 for dt; FrameCount of the reference's 8-slot ring:
    // frame fr is served by slot (fr+1)%8, whose global_tracker has run (fr-1)/8 minimisations before)
    for (int i = 0; i < n; i++) {
        const long long fr = first + i;
        double dt = ts[i] - (i == 0 ? pl->t_prev : ts[i - 1]);
        if (dt < 0.001) dt = 1 / p.config_fps;
        pl->fa_pin[i].t = ts[i];
        pl->fa_pin[i].dt = dt;
        pl->fa_pin[i].frame_count = fr > 0 ? (unsigned int)((fr - 1) / 8) : 0;
        pl->fa_pin[i].next_frame_count = (unsigned int)(fr / 8);   // frame fr+1: ((fr+1)-1)/8
    }
    pl->pn = 0;
    prof_mark(pl, ST_NAV);   // origin of this push
    RB_CUDA(cudaEventRecord(pl->ev[0], c->stream));
    // sub-batches: device input = one (the caller's buffer is read in place).  Host input = a short head (pl->sub
    // frames) and the rest: only the head's H2D copy is exposed, the rest of the frames are copied on the copy stream into
    // their own staging region while the head computes (a frame costs ~8x more to track than to copy), and the scale
    // space of the rest still runs as one large batch.
    // (REBVO_B200_SUB3=1: three stages -- sub/2, 3*sub/2, the rest -- expose half the copy, but add a launch and
    // smaller scale-space batches)
    static const bool three = getenv("REBVO_B200_SUB3") && atoi(getenv("REBVO_B200_SUB3")) != 0;
    int soff[4] = {0, n, n, n}, nsub = 1;
    if (!(on_device || pl->prof_on || n < 3 * pl->sub)) {
        if (three && pl->sub >= 4) {
            const int s0 = pl->sub / 2;
            soff[1] = s0;
            soff[2] = 4 * s0;
            soff[3] = n;
            nsub = 3;
        } else {
            soff[1] = pl->sub;
            soff[2] = n;
            nsub = 2;
        }
    }
    const size_t fbytes = frame_bytes(c, fmt);   // (ws.rgb holds max_batch frames of either format)
    for (int j = 0; j < nsub; j++) {
        const int off = soff[j], nj = soff[j + 1] - soff[j];
        if (on_device) {
            pl->rgb_src_pin[j] = rgb;
        } else {
            pl->rgb_src_pin[j] = pl->ws.rgb + (size_t)off * fbytes;
            cudaStream_t cs = nsub > 1 ? pl->copy_stream : c->stream;
            RB_CUDA(cudaMemcpyAsync(pl->ws.rgb + (size_t)off * fbytes, rgb + (size_t)off * fbytes, (size_t)nj * fbytes,
                                    cudaMemcpyHostToDevice, cs));
            if (nsub > 1) RB_CUDA(cudaEventRecord(pl->ev_copy[j], cs));
        }
    }
    for (int j = 0; j < nsub; j++) {
        const int off = soff[j], nj = soff[j + 1] - soff[j];
        const long long first_j = first + (long long)off;
        if (!on_device && nsub > 1) RB_CUDA(cudaStreamWaitEvent(c->stream, pl->ev_copy[j], 0));
        RB_CUDA(cudaMemcpyAsync(pl->fa_dev, pl->fa_pin + off, sizeof(FrameArgs) * nj, cudaMemcpyHostToDevice, c->stream));
        RB_CUDA(cudaMemcpyAsync(pl->rgb_src_dev, pl->rgb_src_pin + j, sizeof(void *), cudaMemcpyHostToDevice, c->stream));
        if (pl->mirror_on) {
            pl->mirror_base_pin[2 * j] = pl->mirror_dev + (size_t)off * pl->mirror_stride;
            pl->mirror_base_pin[2 * j + 1] = pl->mirror_host + (size_t)off * pl->mirror_stride;
            RB_CUDA(cudaMemcpyAsync(pl->mirror_base_dev, pl->mirror_base_pin + 2 * j, 2 * sizeof(void *), cudaMemcpyHostToDevice,
                                    c->stream));
        }
        const bool graph_ok = pl->use_graph && first_j > 0;
        if (!graph_ok) {
            if ((r = enqueue_batch(pl, fmt, nj, first_j, j == 0))) return r;
        } else {
            const int key = graph_slot(pl, fmt, (int)(first_j % RB_NMAPS), nj);
            // capture the batch once per ring phase; replays only differ through fa_dev / rgb_src_dev contents.  All
            // phases of this format and batch size are instantiated together, so that no later push pays for a capture.
            // The other format's graphs are left as they are: a stream may alternate formats.
            const bool build = !pl->gexec[key];
            for (int ph = 0; ph < RB_NMAPS && build; ph++) {
                const int k = graph_slot(pl, fmt, ph, nj);
                if (pl->gexec[k]) continue;
                cudaGraph_t g = nullptr;
                const int64_t l0 = c->launches;
                RB_CUDA(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
                r = enqueue_batch(pl, fmt, nj, ph == 0 ? RB_NMAPS : ph, false);   // any first frame > 0 of that phase
                cudaError_t e = cudaStreamEndCapture(c->stream, &g);
                if (r) {
                    if (g) cudaGraphDestroy(g);
                    return r;
                }
                if (e != cudaSuccess) {
                    snprintf(c->err, sizeof(c->err), "graph capture: %s", cudaGetErrorString(e));
                    return RB_ERR_CUDA;
                }
                pl->glaunches[k] = (int)(c->launches - l0);
                c->launches = l0;
                e = cudaGraphInstantiate(&pl->gexec[k], g, 0);
                cudaGraphDestroy(g);
                if (e != cudaSuccess) {
                    pl->gexec[k] = nullptr;
                    snprintf(c->err, sizeof(c->err), "graph instantiate: %s", cudaGetErrorString(e));
                    return RB_ERR_CUDA;
                }
            }
            if (j == 0) RB_CUDA(cudaEventRecord(pl->ev[1], c->stream));
            RB_CUDA(cudaGraphLaunch(pl->gexec[key], c->stream));
            if (j == 0) RB_CUDA(cudaEventRecord(pl->ev[2], c->stream));
            c->launches += pl->glaunches[key];
        }
        RB_CUDA(cudaMemcpyAsync(pl->nav_pin + off, pl->nav_dev, sizeof(rb_nav) * nj, cudaMemcpyDeviceToHost, c->stream));
    }
    for (int k = 0; k < RB_NMAPS; k++)
        RB_CUDA(cudaMemcpyAsync(&pl->abort_pin[k], &pl->maps[k]->ts_host.ctl->abort, sizeof(int), cudaMemcpyDeviceToHost,
                                c->stream));
    pl->t_prev = ts[n - 1];
    pl->n_pushed += n;
    prof_mark(pl, ST_NAV);
    RB_CUDA(cudaEventRecord(pl->ev[3], c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    if (pl->prof_on) {
        for (int i = 1; i < pl->pn; i++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, pl->pev[i - 1], pl->pev[i]);
            pl->pacc[pl->ptag[i]] += ms;
        }
        pl->pframes += n;
    }
    if (nav_out) memcpy(nav_out, pl->nav_pin, sizeof(rb_nav) * n);
    pl->mirror_n = pl->mirror_on ? n : 0;
    {   // did a minimiser of this push abort (an exchange between its CTAs timed out)?  Checked on every push.
        bool aborted = false;
        for (int k = 0; k < RB_NMAPS; k++) aborted = aborted || pl->abort_pin[k] != 0;
        if (aborted) {
            for (int k = 0; k < RB_NMAPS; k++) cudaMemset(&pl->maps[k]->ts_host.ctl->abort, 0, sizeof(int));
            snprintf(c->err, sizeof(c->err), "Minimizer_RV: an exchange between the kernel's CTAs timed out (poses are NaN)");
            return RB_ERR_CUDA;
        }
    }
    float ms;
    cudaEventElapsedTime(&ms, pl->ev[0], pl->ev[1]);
    pl->stage_ms[0] = ms;   // copies (+ gray when not replayed as a graph)
    cudaEventElapsedTime(&ms, pl->ev[1], pl->ev[2]);
    pl->stage_ms[1] = ms;   // scale space (eager) or the whole batch graph
    cudaEventElapsedTime(&ms, pl->ev[2], pl->ev[3]);
    pl->stage_ms[2] = ms;   // detect + tracker + mapper of all frames (eager) / nav copy (graph)
    pl->stage_ms[3] = pl->stage_ms[4] = 0;
    cudaEventElapsedTime(&ms, pl->ev[0], pl->ev[3]);
    pl->stage_ms[5] = ms;
    return RB_OK;
}

extern "C" int rb_pipeline_set_undistort(rb_pipeline *pl, const double kc[5]) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    if (pl->und) {
        rb_undistort_destroy(pl->und);
        pl->und = nullptr;
    }
    bool any = false;
    for (int i = 0; kc && i < 5; i++) any = any || kc[i] != 0.0;
    if (any) {
        int r = rb_undistort_create(c, kc, &pl->und);
        if (r) {
            if (pl->und) rb_undistort_destroy(pl->und);
            pl->und = nullptr;
            return r;
        }
    }
    drop_graphs(pl);   // the captured batches contain the other gray kernel (both input formats)
    return RB_OK;
}
extern "C" int rb_pipeline_set_mirror(rb_pipeline *pl, int on) {
    if (!pl || on < 0 || on > 2) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    RB_CUDA(cudaSetDevice(c->device));
    if (pl->imu) {
        snprintf(c->err, sizeof(c->err), "set_mirror: not available in IMU mode");
        return RB_ERR_ARG;
    }
    RB_CUDA(cudaStreamSynchronize(c->stream));
    const size_t stride = ((size_t)c->kcap * sizeof(rb_keyline) + 255) & ~(size_t)255;   // (sized for the larger record)
    if (on && !pl->mirror_dev) {
        const size_t bytes = (size_t)pl->max_batch * stride;
        RB_CUDA(cudaMalloc(&pl->mirror_dev, bytes));
        RB_CUDA(cudaHostAlloc(&pl->mirror_host, bytes, cudaHostAllocMapped));
        RB_CUDA(cudaMalloc(&pl->mirror_base_dev, 2 * sizeof(void *)));
        RB_CUDA(cudaMallocHost(&pl->mirror_base_pin, 8 * sizeof(void *)));
        RB_CUDA(cudaStreamCreateWithFlags(&pl->mirror_stream, cudaStreamNonBlocking));
        pl->ev_mpack = new (std::nothrow) cudaEvent_t[pl->max_batch];
        if (!pl->ev_mpack) return RB_ERR_ARG;
        memset(pl->ev_mpack, 0, sizeof(cudaEvent_t) * pl->max_batch);
        for (int i = 0; i < pl->max_batch; i++) RB_CUDA(cudaEventCreateWithFlags(&pl->ev_mpack[i], cudaEventDisableTiming));
        RB_CUDA(cudaEventCreateWithFlags(&pl->ev_mjoin, cudaEventDisableTiming));
    }
    if (on != pl->mirror_on) drop_graphs(pl);   // the captured batches contain (or not) the pack kernels
    pl->mirror_on = on;
    pl->mirror_rec = on == 2 ? 15 : sizeof(rb_keyline);
    pl->mirror_stride = stride;
    pl->mirror_n = 0;
    return RB_OK;
}
extern "C" int rb_pipeline_mirror(rb_pipeline *pl, int i, const void **records, int *n) {
    if (!pl || !pl->mirror_on || !records || !n) return RB_ERR_ARG;
    if (i < 0 || i >= pl->mirror_n) return RB_ERR_ARG;
    *records = pl->mirror_host + (size_t)i * pl->mirror_stride;
    *n = pl->nav_pin[i].kn;
    return RB_OK;
}

extern "C" int rb_pipeline_push(rb_pipeline *pl, const uint8_t *rgb, const double *ts, int n, rb_nav *nav_out) {
    return push_impl(pl, rgb, RB_IN_RGB, false, ts, n, nav_out);
}
extern "C" int rb_pipeline_push_dev(rb_pipeline *pl, const uint8_t *rgb_dev, const double *ts, int n,
                                    rb_nav *nav_out) {
    return push_impl(pl, rgb_dev, RB_IN_RGB, true, ts, n, nav_out);
}
extern "C" int rb_pipeline_push_mono(rb_pipeline *pl, const uint8_t *mono, const double *ts, int n, rb_nav *nav_out) {
    return push_impl(pl, mono, RB_IN_MONO, false, ts, n, nav_out);
}
extern "C" int rb_pipeline_push_mono_dev(rb_pipeline *pl, const uint8_t *mono_dev, const double *ts, int n,
                                         rb_nav *nav_out) {
    return push_impl(pl, mono_dev, RB_IN_MONO, true, ts, n, nav_out);
}

extern "C" int rb_pipeline_event_record(rb_pipeline *pl, int slot) {
    rb_ctx *c = pl->c;
    if (slot < 0 || slot > 7) return RB_ERR_ARG;
    RB_CUDA(cudaEventRecord(pl->user_ev[slot], c->stream));
    return RB_OK;
}
extern "C" int rb_pipeline_event_elapsed(rb_pipeline *pl, int a, int b, float *ms) {
    rb_ctx *c = pl->c;
    if (a < 0 || a > 7 || b < 0 || b > 7) return RB_ERR_ARG;
    RB_CUDA(cudaEventSynchronize(pl->user_ev[b]));
    RB_CUDA(cudaEventElapsedTime(ms, pl->user_ev[a], pl->user_ev[b]));
    return RB_OK;
}
// elapsed time between an event of one pipeline and an event of another (several pipelines share a GPU: bench.py --config 4)
extern "C" int rb_pipeline_event_elapsed_between(rb_pipeline *pa, int a, rb_pipeline *pb, int b, float *ms) {
    if (!pa || !pb || a < 0 || a > 7 || b < 0 || b > 7 || !ms) return RB_ERR_ARG;
    rb_ctx *c = pb->c;
    RB_CUDA(cudaEventSynchronize(pb->user_ev[b]));
    RB_CUDA(cudaEventElapsedTime(ms, pa->user_ev[a], pb->user_ev[b]));
    return RB_OK;
}
extern "C" int rb_pipeline_bench_pass(rb_pipeline *pl, int pass_id, int nimg, int iters, float *ms_per_launch,
                                      double *bytes_per_launch) {
    rb_ctx *c = pl->c;
    if (nimg < 1 || nimg > pl->max_batch || iters < 1) return RB_ERR_ARG;
    int r;
    double bytes = 0;
    // pass 5: the gray pass with the undistortion fused in (needs rb_pipeline_set_undistort; source = the workspace's RGB);
    // algorithmic bytes: 3N in + 4N out per frame + the 32N-byte map once per launch.  Pass 7: the same from mono frames
    // (N in + 4N out per frame + the map)
    const bool und_pass = pass_id == 5 || pass_id == 7;
    auto one = [&]() -> int {
        if (!und_pass) return rb_dog_single_pass(c, &pl->ws, pass_id, nimg, &bytes);
        if (!pl->und) return RB_ERR_STATE;
        if (pass_id == 7) {
            bytes = 5.0 * c->N * nimg + 32.0 * c->N;
            return rb_undistort_gray_mono_enqueue(pl->und, pl->rgb_src_dev, pl->ws.gray, nimg);
        }
        bytes = 7.0 * c->N * nimg + 32.0 * c->N;
        return rb_undistort_gray_enqueue(pl->und, pl->rgb_src_dev, pl->ws.gray, nimg);
    };
    if (und_pass) {
        const void *src = pl->ws.rgb;
        RB_CUDA(cudaMemcpyAsync(pl->rgb_src_dev, &src, sizeof(void *), cudaMemcpyHostToDevice, c->stream));
    }
    for (int i = 0; i < 3; i++)
        if ((r = one())) return r;
    RB_CUDA(cudaEventRecord(pl->user_ev[6], c->stream));
    for (int i = 0; i < iters; i++)
        if ((r = one())) return r;
    RB_CUDA(cudaEventRecord(pl->user_ev[7], c->stream));
    RB_CUDA(cudaEventSynchronize(pl->user_ev[7]));
    float ms = 0;
    RB_CUDA(cudaEventElapsedTime(&ms, pl->user_ev[6], pl->user_ev[7]));
    *ms_per_launch = ms / iters;
    *bytes_per_launch = bytes;
    return RB_OK;
}

extern "C" int rb_pipeline_stage_profile(rb_pipeline *pl, double out_ms[16], long long *frames) {
    if (!pl->prof_on) return RB_ERR_STATE;
    for (int i = 0; i < 16; i++) out_ms[i] = pl->pacc[i];
    if (frames) *frames = pl->pframes;
    return RB_OK;
}

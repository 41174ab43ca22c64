// pipeline.cu -- the per-frame flow of REBVO with every piece of state resident on the device:
//   detector stage  = REBVO::FirstThr   (src/rebvo/rebvo_first_t.cpp:259-272)
//   tracker/mapper  = REBVO::SecondThread, ImuMode=0 branch (src/rebvo/rebvo_second_t.cpp:128-629)
// The host only enqueues kernels: threshold feedback, LM driver, NaN / match-count decisions, pose
// integration and the NavData record are all computed by 1-thread kernels from device state, so a batch of
// frames costs one H2D copy, one stream of launches and one D2H copy of the nav records.
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <new>

#include "common.cuh"
#include "lm.cuh"
#include "tracker.cuh"
#include "frame.cuh"
#include "depth.cuh"
#include "state.cuh"

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

// The device addresses a sub-batch's kernels read, so that one captured batch serves every region of a push: one table on
// the device, rewritten by one H2D copy per sub-batch from its pinned entry
struct SubBatchPtrs {
    const void *src;            // the RGB24 (or mono) frames of the sub-batch
    unsigned char *mirror[2];   // keyline mirror: {device staging, mapped host} slot of the sub-batch's first frame
    unsigned char *depth[3];    // depth grid: {record staging, output cells, output image} of that frame (output: mapped
                                // pinned host memory, or device memory with rb_pipeline_set_output_memory(pl, 1))
};

// The per-push sources and outputs of one push: rb_pipeline::out for the synchronous pushes, AsyncRing::slot[k % depth] for
// ticket k of the asynchronous ones (rb_pipeline_set_async / rb_pipeline_enqueue / rb_pipeline_wait).  The output accessors
// read the slot rb_pipeline::view points at.
struct OutSlot {
    long long first;                  // frame number of the push's first frame
    int n;                            // its frames
    rb_nav *nav;                      // pinned [max_batch]: the nav records, copied from nav_dev after each batch
    rb_odometry *odom;                // pinned [max_batch] (odometry on)
    int *abort;                       // pinned [RB_NMAPS]: the ring maps' minimiser abort flags after the push
    struct FrameArgs *fa;             // pinned [max_batch]: per-frame scalars, the source of the fa_dev copies
    SubBatchPtrs *tbl;                // pinned [2]: per sub-batch the table copied into sb_dev (a ticket: the front's table
                                      // in [0], the back's in [1])
    rb_frame *frames;                 // pinned [max_batch]: strided device input, the source of the frame table
    DetMask *masks;                   // pinned [max_batch]: the detection masks of a masked push, the source of the
                                      // det_mask_dev copies
    // the mirror, depth grid and depth image: host buffers in host output mode, device ones in device mode.  The
    // synchronous slot's mirror_dev is the mirror's staging in either mode; the ring slots pack into it in host mode too
    unsigned char *mirror_host, *mirror_dev, *depth_host, *depth_dev, *dimg_host, *dimg_dev;
    size_t mirror_host_bytes, mirror_dev_bytes, depth_host_bytes, depth_dev_bytes, dimg_host_bytes, dimg_dev_bytes;
    cudaEvent_t done;                 // a ticket's: recorded on the tracker stream after its last copy
};
// captured graphs by key: exec[k] (nullptr: not captured yet) launches launches[k] kernels
struct GraphCache {
    cudaGraphExec_t *exec;
    int *launches;
    int size;
};
// Asynchronous pushes.  Ticket k runs its front (staging, gray, scale space) on the front stream into workspace k % 2 and its
// back (detect ... depth image) on the tracker stream, writing its outputs into slot k % depth; see DESIGN.md §5.
struct AsyncRing {
    int depth;                        // 1..8 tickets in flight, one output slot each
    OutSlot slot[8];
    DogWS ws1;                        // workspace of odd tickets (even tickets use rb_pipeline::ws)
    SubBatchPtrs *front_dev[2];       // device, per workspace: the table the front's gray pass reads
    rb_frame *frames_dev[2];          // device, per workspace: strided device input's {data, step} table
    cudaStream_t front;
    cudaEvent_t ev_front[2];          // per workspace: its front is complete (the back waits for it)
    cudaEvent_t ev_free[2];           // per workspace: the back that read it last is complete (the next front waits for it)
    // captured halves: the front per (input format, workspace, batch size), the back per (masked, workspace, ring phase, batch
    // size)
    GraphCache front_graphs, back_graphs;
};

struct ImuFlow;
struct rb_pipeline {
    rb_ctx *c;
    ImuFlow *imu;         // IMU mode (rb_pipeline_set_imu, rb_pipeline_set_imu_live), nullptr otherwise
    rb_params p;
    int max_batch;
    DogWS ws;
    rb_map *maps[RB_NMAPS];   // ring: frame f lives in maps[f % RB_NMAPS]
    // one event for every hand-over between two streams whose wait follows its record at once (stream_wait)
    cudaEvent_t ev_hop;
    // detector stream: detect(f+1) (+ reEstimateThresh) runs beside the tracker/mapper of frame f; the third map is
    // what lets it write while frame f still reads map f-1.  detect(f) waits for track(f-2): ev_trk[f % 2]
    cudaStream_t det_stream;
    cudaEvent_t ev_trk[2];
    bool overlap;
    // FordwardMatch's apply + directed_matching in k_match, then gate + Regularize_1_iter + EKF + rotate_keylines in
    // k_reg_ekf (env REBVO_B200_MAP_CHAIN=0: the stage kernels in the reference's order, the bitwise reference of the two)
    bool map_chain;
    // rescaling stream: with DoReScaling=0 a frame's EstimateReScalingOpt changes no keyline and only fills in its nav record,
    // so it runs here (lowest priority) instead of at the end of the frame's tracker chain; the tracker stream joins it
    // before the next frame's first kernel after the minimiser (k_match, or k_fm_apply before k_rotate, which writes the
    // map's rho / s_rho, in the reference schedule)
    cudaStream_t resc_stream;     // nullptr: the rescaling stays in the frame's map-update kernel on the tracker stream
    cudaEvent_t ev_rjoin;
    bool resc_open;               // a rescaling was forked and not joined yet
    // host-input pushes are cut into a short head and the rest: the H2D copy of the rest (copy stream) runs beside the
    // kernels of the head
    cudaStream_t copy_stream;
    cudaEvent_t ev_copy[2];       // per sub-batch: its frames are on the device
    SubBatchPtrs *sb_dev;         // device: the table of the sub-batch being processed, from its slot's tbl entry
    // strided device input (rb_pipeline_push_frames_dev): frame i of the push is frames_dev[i], written from the slot's
    // frames before the batch runs, so that one captured batch serves every push of that layout.  Apart from SubBatchPtrs:
    // the packed pushes' per-sub-batch copy does not grow.
    rb_frame *frames_dev;         // device [max_batch]
    // detection masks (rb_pipeline_set_detect_mask, rb_pipeline_push_masked): a masked push writes frame i's DetMask into
    // det_mask_dev[i] before its batch, as frames_dev, so that one captured batch serves every mask buffer.  Unmasked pushes
    // neither write nor read the table.  det_fixed: the fixed mask, packed w x h (kept when cleared, for the next set).
    DetMask *det_mask_dev;        // device [max_batch]
    unsigned char *det_fixed;     // device [w * h]
    bool det_fixed_on;
    int sub;                      // head sub-batch of a host-input push (env REBVO_B200_SUB, default 8 frames)
    int last_sub;                 // frames of the last scale-space batch (the rest of a head / rest push): ws slots in use
    DetChain *chain;      // device
    FrameState *fs;       // device
    rb_nav *nav_dev;
    long long n_pushed;   // frames pushed so far
    bool restored;        // rb_pipeline_load_state since the last push: the ring holds the newest map alone
    unsigned char *state_host;    // mapped pinned staging of a state blob's device section (rb_pipeline_save_state)
    size_t state_host_bytes;
    double t_prev;
    cudaEvent_t ev[4];
    cudaEvent_t user_ev[8];
    float stage_ms[6];
    struct FrameArgs *fa_dev;
    // one instantiated CUDA graph per (masked, input format, ring phase of the first frame, batch size): the kernel sequence
    // of a batch is static once the per-frame scalars live in fa_dev
    GraphCache graphs;            // [2 * RB_NFMT * RB_NMAPS * (max_batch + 1)], see graph_slot
    bool use_graph;
    // optional in-situ stage profile (REBVO_B200_STAGE_PROF=1, forces eager launches): CUDA events between stages
    bool prof_on;
    cudaEvent_t *pev;
    int *ptag;
    int pcap, pn;
    double pacc[16];
    long long pframes;
    rb_undistort *und;    // UseUndistort=1 (rb_pipeline_set_undistort): fused into the gray pass
    // where the mirror, the depth grid and the depth image go (rb_pipeline_set_output_memory): 0 mapped pinned host memory,
    // 1 device memory.  In device mode the mirror's staging slots are its output (no k_mirror_to_host), and the fill and
    // the image pass write into a slot's depth_dev / dimg_dev instead of depth_host / dimg_host; no kernel changes.  Each
    // mode's buffers are made by the set_* call that needs them and kept (grown, never shrunk) across switches.
    int out_dev;
    // device mode: each push first waits for the work enqueued on this stream so far (rb_pipeline_set_consumer_stream), so
    // that it overwrites no output a consumer of the last push still reads; the pipeline's own stream = nothing to wait for
    cudaStream_t consumer;
    // The optional per-frame outputs, whose buffers are in the OutSlots.  Each keeps its own frame count of the shown push,
    // which its set_* call clears (and set_depth the image's too: the images are of the grid).
    // Keyline mirror (rb_pipeline_set_mirror): every frame's keylines are packed into a device staging slot right after its
    // map update (tracker stream), then (host mode) a small kernel on the mirror's stream writes exactly kn records into
    // mapped pinned host memory while the next frames are tracked; both are part of the captured batch
    struct {
        int on;                        // 0 off, 1 = 168-byte KeyLine records, 2 = 15-byte net_keyline records
        size_t rec, stride;            // bytes per record / per frame slot (multiple of 256)
        cudaStream_t stream;
        int n;                         // frames of the shown push
    } mirror;
    // odometry records (rb_pipeline_set_odometry): written beside the nav records, copied with them
    struct {
        int on;
        rb_odometry *dev;              // [max_batch]
        int n;                         // records of the shown push
        double rkp_last;               // RKp of the last frame pushed: QK of the next push's first record
    } odom;
    // depth grid (rb_pipeline_set_depth): right after its map update each frame's net_keyline records are packed into a
    // staging slot (tracker stream; with mirror mode 2 the mirror's slot is read instead), then one fill CTA on a side stream
    // writes the frame's cells and min_dist into mapped pinned host memory; both are part of the captured batch.  Frame i's
    // fill runs on stream[i % RB_DEPTH_STREAMS] with that stream's workspace: one fill takes longer than a tracked frame, so
    // the fills of consecutive frames run side by side on their own SMs
    struct {
        int on;
        DepthPlan plan;
        size_t rec_stride;             // bytes per frame staging slot (kcap records, multiple of 256)
        unsigned char *stage;          // [max_batch * rec_stride]: device staging
        void *ws;                      // per stream: bucketing scratch (and the grid when it does not fit in smem)
        size_t ws_bytes;               // (per stream)
        cudaStream_t stream[RB_DEPTH_STREAMS];
        int n;                         // frames of the shown push
    } depth;
    // dense image of the grid (rb_pipeline_set_depth_image): right after each frame's fill, on the same side stream,
    // k_depth_image reads the fill's final cells from that stream's workspace and writes 1 (rho) or 2 (rho, s_rho) w x h
    // float planes into mapped pinned host memory; part of the captured batch, covered by its depth joins.  A kernel of its
    // own: the fill is one latency-bound CTA, the image pass writes megabytes from many CTAs.
    struct {
        int mode;                      // 0 off, 1 rho, 2 rho and s_rho
        DepthImgPlan plan;             // (of depth.plan's grid, when both are on)
        size_t plane, stride;          // floats per plane (a multiple of 64); bytes per frame slot
        int n;                         // frames of the shown push
    } dimg;
    OutSlot out;                  // the synchronous pushes'
    // asynchronous pushes (nullptr: off).  Tickets count up from 0 for the pipeline's lifetime; [tk_retired, tk_next) are
    // outstanding
    AsyncRing *ar;
    long long tk_next, tk_retired;
    // the slot the output accessors read: &out, or after a wait the retired ticket's until the next wait or push (show)
    const OutSlot *view;
};

// input layouts of a push: packed RGB24 (3 bytes per pixel) or mono8, which stands for the RGB24 frame (m, m, m), at
// sb_dev->src; or the same two formats as strided device frames, one {data, step} entry per frame in frames_dev.  Each
// layout has graph slots of its own.
enum { RB_IN_RGB = 0, RB_IN_MONO = 1, RB_IN_RGB_STRIDED = 2, RB_IN_MONO_STRIDED = 3, RB_NFMT = 4 };
static inline bool in_mono(int fmt) { return fmt == RB_IN_MONO || fmt == RB_IN_MONO_STRIDED; }
static inline bool in_strided(int fmt) { return fmt == RB_IN_RGB_STRIDED || fmt == RB_IN_MONO_STRIDED; }
static inline size_t frame_bytes(const rb_ctx *c, int fmt) { return (in_mono(fmt) ? (size_t)1 : (size_t)3) * c->N; }
// (masked: the batch detects through k_detect_a_masked, with the frames' detection masks in det_mask_dev)
static inline int graph_slots(const rb_pipeline *pl) { return 2 * RB_NFMT * RB_NMAPS * (pl->max_batch + 1); }
static inline int graph_slot(const rb_pipeline *pl, bool masked, int fmt, int phase, int n) {
    return (((masked ? RB_NFMT : 0) + fmt) * RB_NMAPS + phase) * (pl->max_batch + 1) + n;
}
// the asynchronous pushes' halves (AsyncRing::front_graphs / back_graphs)
static inline int afront_slots(const rb_pipeline *pl) { return RB_NFMT * 2 * (pl->max_batch + 1); }
static inline int afront_slot(const rb_pipeline *pl, int fmt, int par, int n) {
    return (fmt * 2 + par) * (pl->max_batch + 1) + n;
}
static inline int aback_slots(const rb_pipeline *pl) { return 2 * 2 * RB_NMAPS * (pl->max_batch + 1); }
static inline int aback_slot(const rb_pipeline *pl, bool masked, int par, int phase, int n) {
    return (((masked ? 2 : 0) + par) * RB_NMAPS + phase) * (pl->max_batch + 1) + n;
}
static int graphs_alloc(GraphCache &g, int size) {
    g.exec = new (std::nothrow) cudaGraphExec_t[size]();
    g.launches = new (std::nothrow) int[size]();
    g.size = size;
    return g.exec && g.launches ? RB_OK : RB_ERR_ARG;
}
static void graphs_drop(GraphCache &g) {
    for (int i = 0; g.exec && i < g.size; i++)
        if (g.exec[i]) {
            cudaGraphExecDestroy(g.exec[i]);
            g.exec[i] = nullptr;
        }
}
static void graphs_free(GraphCache &g) {
    graphs_drop(g);
    delete[] g.exec;
    delete[] g.launches;
    g = GraphCache();
}
// captured batches contain the gray kernel, the undistortion and the mirror's pack kernels: drop them all
static void drop_graphs(rb_pipeline *pl) {
    graphs_drop(pl->graphs);
    if (pl->ar) {
        graphs_drop(pl->ar->front_graphs);
        graphs_drop(pl->ar->back_graphs);
    }
}
// `to` waits for the work enqueued on `from` so far.  One event serves every such hand-over: a wait (eager or captured)
// takes the event's most recent record at the time of the call.
static int stream_wait(rb_pipeline *pl, cudaStream_t from, cudaStream_t to) {
    rb_ctx *c = pl->c;
    RB_CUDA(cudaEventRecord(pl->ev_hop, from));
    RB_CUDA(cudaStreamWaitEvent(to, pl->ev_hop, 0));
    return RB_OK;
}
// *buf: mapped pinned host memory of at least `bytes`, kept when it is large enough (its contents are not kept otherwise)
static int grow_mapped(rb_ctx *c, unsigned char **buf, size_t *have, size_t bytes) {
    if (bytes <= *have) return RB_OK;
    if (*buf) cudaFreeHost(*buf);
    *buf = nullptr;
    *have = 0;
    RB_CUDA(cudaHostAlloc(buf, bytes, cudaHostAllocMapped));
    *have = bytes;
    return RB_OK;
}
// *buf: device memory of at least `bytes`, kept when it is large enough (its contents are not kept otherwise)
static int grow_dev(rb_ctx *c, unsigned char **buf, size_t *have, size_t bytes) {
    if (bytes <= *have) return RB_OK;
    cudaFree(*buf);
    *buf = nullptr;
    *have = 0;
    RB_CUDA(cudaMalloc(buf, bytes));
    *have = bytes;
    return RB_OK;
}
// an output buffer of `bytes` where the pipeline's outputs go now (rb_pipeline_set_output_memory)
static int grow_out(rb_pipeline *pl, unsigned char **host, size_t *host_have, unsigned char **dev, size_t *dev_have,
                    size_t bytes) {
    return pl->out_dev ? grow_dev(pl->c, dev, dev_have, bytes) : grow_mapped(pl->c, host, host_have, bytes);
}

// ---- output slots ----------------------------------------------------------------------------------------------------------
// a slot's pinned sources and records; its outputs are slot_grow's
static int slot_alloc(rb_pipeline *pl, OutSlot &s) {
    rb_ctx *c = pl->c;
    const size_t mb = (size_t)pl->max_batch;
    RB_CUDA(cudaMallocHost(&s.nav, sizeof(rb_nav) * mb));
    RB_CUDA(cudaMallocHost(&s.abort, sizeof(int) * RB_NMAPS));
    memset(s.abort, 0, sizeof(int) * RB_NMAPS);
    RB_CUDA(cudaMallocHost(&s.fa, sizeof(FrameArgs) * mb));
    RB_CUDA(cudaMallocHost(&s.tbl, 2 * sizeof(SubBatchPtrs)));
    RB_CUDA(cudaMallocHost(&s.frames, sizeof(rb_frame) * mb));
    RB_CUDA(cudaMallocHost(&s.masks, sizeof(DetMask) * mb));
    return RB_OK;
}
// slot s's outputs as large as the outputs that are on now need, where rb_pipeline_set_output_memory puts them.  The
// synchronous slot's mirror_dev is the mirror's staging, so it is there in both modes; a ring slot's is its device output.
static int slot_grow(rb_pipeline *pl, OutSlot &s) {
    rb_ctx *c = pl->c;
    const size_t mb = (size_t)pl->max_batch;
    int r = RB_OK;
    if (pl->odom.on && !s.odom) RB_CUDA(cudaMallocHost(&s.odom, sizeof(rb_odometry) * mb));
    if (pl->mirror.on && (pl->out_dev || &s == &pl->out))
        r = grow_dev(c, &s.mirror_dev, &s.mirror_dev_bytes, mb * pl->mirror.stride);
    if (!r && pl->mirror.on && !pl->out_dev)
        r = grow_mapped(c, &s.mirror_host, &s.mirror_host_bytes, mb * pl->mirror.stride);
    if (!r && pl->depth.on)
        r = grow_out(pl, &s.depth_host, &s.depth_host_bytes, &s.depth_dev, &s.depth_dev_bytes, mb * pl->depth.plan.cells_bytes);
    if (!r && pl->dimg.mode)
        r = grow_out(pl, &s.dimg_host, &s.dimg_host_bytes, &s.dimg_dev, &s.dimg_dev_bytes, mb * pl->dimg.stride);
    return r;
}
// slot_grow for every slot: by the set_* calls that switch an output on, enlarge it or move it, and by rb_pipeline_set_async,
// never by a push
static int grow_outputs(rb_pipeline *pl) {
    int r = slot_grow(pl, pl->out);
    for (int k = 0; pl->ar && k < pl->ar->depth && !r; k++) r = slot_grow(pl, pl->ar->slot[k]);
    return r;
}
static void slot_free(OutSlot &s) {
    if (s.done) cudaEventDestroy(s.done);
    void *host[] = {s.nav, s.odom, s.abort, s.fa, s.tbl, s.frames, s.masks, s.mirror_host, s.depth_host, s.dimg_host};
    for (void *p : host)
        if (p) cudaFreeHost(p);
    void *dev[] = {s.mirror_dev, s.depth_dev, s.dimg_dev};
    for (void *p : dev) cudaFree(p);
}
// the output accessors show n frames of slot s (n = 0: none)
static void show(rb_pipeline *pl, const OutSlot &s, int n) {
    pl->view = &s;
    pl->odom.n = pl->odom.on ? n : 0;
    pl->mirror.n = pl->mirror.on ? n : 0;
    pl->depth.n = pl->depth.on ? n : 0;
    pl->dimg.n = pl->depth.on && pl->dimg.mode ? n : 0;
}
// the host side of a push or ticket whose records in s are complete, in push order: odometry QK, the P_Kp a frame found =
// RKp of the previous frame's record, which holds the value after that frame's rescaling also when the rescaling ran on the
// side stream (:382, :480-487); the zero record of a sequence's first frame, which only initialises the ring (:109-121);
// and the minimisers' abort flags (an exchange between a minimiser's CTAs timed out)
static int retire(rb_pipeline *pl, OutSlot &s) {
    for (int i = 0; i < s.n && pl->odom.on; i++) {
        if (s.first + i == 0) {
            memset(&s.odom[i], 0, sizeof(rb_odometry));
            continue;
        }
        s.odom[i].QK = i == 0 ? pl->odom.rkp_last : s.nav[i - 1].RKp;
    }
    pl->odom.rkp_last = s.nav[s.n - 1].RKp;
    for (int m = 0; m < RB_NMAPS; m++)
        if (s.abort[m]) {
            snprintf(pl->c->err, sizeof(pl->c->err), "Minimizer_RV: an exchange between the kernel's CTAs timed out in frames "
                     "%lld to %lld (poses are NaN)", s.first, s.first + s.n - 1);
            return RB_ERR_CUDA;
        }
    return RB_OK;
}

// true, with the reason in the pipeline's error, while asynchronous tickets are outstanding: `what` would change or read
// what they use
static bool refuse_busy(rb_pipeline *pl, const char *what) {
    if (pl->tk_next == pl->tk_retired) return false;
    snprintf(pl->c->err, sizeof(pl->c->err), "%s: %lld asynchronous tickets are outstanding (rb_pipeline_wait them first)",
             what, pl->tk_next - pl->tk_retired);
    return true;
}

// ---- a push's input --------------------------------------------------------------------------------------------------------
// as the C entry point received it; push_in checks it and sets fmt
struct PushIn {
    const uint8_t *data;          // n packed frames (host or device memory), or nullptr for
    const rb_frame *frames;       // n strided frames
    int format;                   // RB_FRAME_RGB24 or RB_FRAME_MONO8
    bool on_device;
    bool with_masks;              // the call takes per-frame detection masks:
    const rb_frame *masks;        // n device {data, step} entries
    const double *ts;
    int n;
    int fmt;                      // the input layout (RB_IN_*): host strided frames run the packed format's batches
};
// every argument check of a push, before anything is enqueued
static int push_in(rb_pipeline *pl, const char *what, PushIn &in) {
    rb_ctx *c = pl->c;
    if (in.format != RB_FRAME_RGB24 && in.format != RB_FRAME_MONO8) {
        snprintf(c->err, sizeof(c->err), "%s: format %d is neither RB_FRAME_RGB24 nor RB_FRAME_MONO8", what, in.format);
        return RB_ERR_ARG;
    }
    if (in.n < 1 || in.n > pl->max_batch || !(in.data || in.frames) || !in.ts) return RB_ERR_ARG;
    const bool mono = in.format == RB_FRAME_MONO8;
    const int64_t row = (int64_t)(mono ? 1 : 3) * c->w;
    for (int i = 0; in.frames && i < in.n; i++)
        if (!in.frames[i].data || in.frames[i].step < row) {
            snprintf(c->err, sizeof(c->err), "%s: frame %d has %s (rows need %lld bytes)", what, i,
                     in.frames[i].data ? "a step shorter than a row" : "no data", (long long)row);
            return RB_ERR_ARG;
        }
    const bool strided = in.frames && in.on_device;
    if (strided && pl->und && (c->w > 65535 || c->h > 65535)) {   // (the strided undistortion's 16-bit tap coordinates)
        snprintf(c->err, sizeof(c->err), "%s_dev: undistorted frames wider or higher than 65535 pixels", what);
        return RB_ERR_ARG;
    }
    if (in.with_masks && !in.masks) {
        snprintf(c->err, sizeof(c->err), "%s: no masks", what);
        return RB_ERR_ARG;
    }
    for (int i = 0; in.with_masks && i < in.n; i++)   // (each step at least a row of w bytes)
        if (!in.masks[i].data || in.masks[i].step < c->w) {
            snprintf(c->err, sizeof(c->err), "%s: mask %d has %s (rows need %d bytes)", what, i,
                     in.masks[i].data ? "a step shorter than a row" : "no data", c->w);
            return RB_ERR_ARG;
        }
    in.fmt = (mono ? RB_IN_MONO : RB_IN_RGB) + (strided ? RB_IN_RGB_STRIDED : 0);
    // (the packed mono kernels read a device buffer as aligned 32-bit words; the RGB kernels test the alignment of the source
    // on the device -- k_gray<false, GRAY_ALIGNED> and ug_pixel take a path for unaligned sources -- and the any-width kernels
    // read every source through aligned words around it)
    if (in.fmt == RB_IN_MONO && in.on_device && (reinterpret_cast<uintptr_t>(in.data) & 3)) return RB_ERR_ARG;
    return RB_OK;
}
// host frames [i0, i0 + count) of a push into the packed staging (ws's, by default the pipeline's), one 2D copy each when
// strided, on stream s
static int stage_host_frames(rb_pipeline *pl, const PushIn &in, int i0, int count, cudaStream_t s, DogWS *ws = nullptr) {
    rb_ctx *c = pl->c;
    const size_t fbytes = frame_bytes(c, in.fmt), row = fbytes / c->h;
    uint8_t *dst = (ws ? ws : &pl->ws)->rgb + (size_t)i0 * fbytes;
    if (!in.frames) {
        RB_CUDA(cudaMemcpyAsync(dst, in.data + (size_t)i0 * fbytes, (size_t)count * fbytes, cudaMemcpyHostToDevice, s));
        return RB_OK;
    }
    for (int i = 0; i < count; i++)
        RB_CUDA(cudaMemcpy2DAsync(dst + (size_t)i * fbytes, row, in.frames[i0 + i].data, (size_t)in.frames[i0 + i].step, row,
                                  c->h, cudaMemcpyHostToDevice, s));
    return RB_OK;
}
// a synchronous push's frames onto the device, before its batches: host frames into the pipeline's staging, sub-batch j
// (frames [soff[j], soff[j + 1])) on the copy stream, recording ev_copy[j], when there are two, else on the tracker stream;
// strided device frames as their {data, step} table in frames_dev, on the tracker stream
static int stage_push(rb_pipeline *pl, const PushIn &in, const int *soff, int nsub) {
    rb_ctx *c = pl->c;
    int r;
    for (int j = 0; j < nsub && !in.on_device; j++) {
        cudaStream_t cs = nsub > 1 ? pl->copy_stream : c->stream;
        if ((r = stage_host_frames(pl, in, soff[j], soff[j + 1] - soff[j], cs))) return r;
        if (nsub > 1) RB_CUDA(cudaEventRecord(pl->ev_copy[j], cs));
    }
    if (in_strided(in.fmt)) {
        memcpy(pl->out.frames, in.frames, sizeof(rb_frame) * in.n);
        RB_CUDA(cudaMemcpyAsync(pl->frames_dev, pl->out.frames, sizeof(rb_frame) * in.n, cudaMemcpyHostToDevice, c->stream));
    }
    return RB_OK;
}
// the per-frame scalars of a push of n frames, the next frames of the stream, into s (SecondThread :146-149 for dt;
// FrameCount of the reference's 8-slot ring: frame fr is served by slot (fr+1)%8, whose global_tracker has run (fr-1)/8
// minimisations before)
static void write_args(rb_pipeline *pl, OutSlot &s, const double *ts, int n) {
    s.first = pl->n_pushed;
    s.n = n;
    for (int i = 0; i < n; i++) {
        const long long fr = s.first + i;
        double dt = ts[i] - (i == 0 ? pl->t_prev : ts[i - 1]);
        if (dt < 0.001) dt = 1 / pl->p.config_fps;
        s.fa[i].t = ts[i];
        s.fa[i].dt = dt;
        s.fa[i].frame_count = fr > 0 ? (unsigned int)((fr - 1) / 8) : 0;
    }
}
// the detection masks of the n frames of a push into s: the fixed mask and masks[i] (device rb_frame entries, or nullptr).
// False, writing nothing, when no mask applies: the push runs the unmasked batches.
static bool fill_masks(const rb_pipeline *pl, const rb_frame *masks, int n, OutSlot &s) {
    if (!masks && !pl->det_fixed_on) return false;
    for (int i = 0; i < n; i++) {
        s.masks[i].fixed = pl->det_fixed_on ? pl->det_fixed : nullptr;
        s.masks[i].fixed_step = pl->c->w;
        s.masks[i].frame = masks ? masks[i].data : nullptr;
        s.masks[i].frame_step = masks ? masks[i].step : 0;
    }
    return true;
}
// on the tracker stream before a batch of frames [off, off + nj) of slot s: their detection masks into det_mask_dev
// (masked), and the batch's pointer table -- its frames at src, its outputs in s -- from s.tbl[j] into sb_dev
static int write_tables(rb_pipeline *pl, OutSlot &s, int j, const void *src, int off, int nj, bool masked) {
    rb_ctx *c = pl->c;
    if (masked)
        RB_CUDA(cudaMemcpyAsync(pl->det_mask_dev, s.masks + off, sizeof(DetMask) * nj, cudaMemcpyHostToDevice, c->stream));
    SubBatchPtrs &t = s.tbl[j];
    memset(&t, 0, sizeof(t));
    t.src = src;
    if (pl->mirror.on) {   // (host mode: packed into the synchronous slot's staging, then copied into s's mapped memory)
        t.mirror[0] = (pl->out_dev ? s.mirror_dev : pl->out.mirror_dev) + (size_t)off * pl->mirror.stride;
        t.mirror[1] = pl->out_dev ? nullptr : s.mirror_host + (size_t)off * pl->mirror.stride;
    }
    if (pl->depth.on) {
        t.depth[0] = pl->depth.stage + (size_t)off * pl->depth.rec_stride;
        t.depth[1] = (pl->out_dev ? s.depth_dev : s.depth_host) + (size_t)off * pl->depth.plan.cells_bytes;
        t.depth[2] = pl->dimg.mode ? (pl->out_dev ? s.dimg_dev : s.dimg_host) + (size_t)off * pl->dimg.stride : nullptr;
    }
    RB_CUDA(cudaMemcpyAsync(pl->sb_dev, &t, sizeof(t), cudaMemcpyHostToDevice, c->stream));
    return RB_OK;
}
static int enqueue_front(rb_pipeline *pl, DogWS *ws, SubBatchPtrs *tbl, const rb_frame *frames_dev, int fmt, int n,
                         bool with_events);
#include "imu_flow.cuh"
static void async_free(rb_pipeline *pl);

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

__global__ void k_frame_post_match(FrameState *fs, MapState *nst, int match_threshold, const TrackState *ts, rb_odometry *odom) {
    d_frame_post_match(fs, nst, match_threshold);
    nst->do_map = fs->do_map;   // for this map's rescaling on the side stream: the next frame rewrites FrameState
    if (odom) d_frame_odometry(fs, ts->lm, odom);
}
// the nav record before the map's rescaling, which runs on the side stream and fills in its Kp / RKp
__global__ void k_frame_finish(FrameState *fs, const MapState *nst, const MapState *ost, const TrackState *ts,
                               rb_nav *nav, const FrameArgs *fa) {
    d_frame_finish(fs, nst, ost, ts->lm.score, nav, fa, false);
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
    // FrameCount 0 in every ring map: the vision flow rewrites it each frame, but the IMU flow only reads it (the
    // reference raises FrameCount in Minimizer_RV alone, so its IMU mode never gates on m_num)
    for (int k = 0; k < RB_NMAPS; k++)
        if (pl->maps[k]) {
            RB_CUDA(cudaMemset(&pl->maps[k]->ts_host.ctl->abort, 0, sizeof(int)));
            RB_CUDA(cudaMemset(&pl->maps[k]->st->frame_count, 0, sizeof(unsigned int)));
        }
    if (pl->imu) imu_flow_reset(*pl->imu);
    pl->n_pushed = 0;
    pl->restored = false;
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
    RB_CUDA(cudaMalloc(&pl->fa_dev, sizeof(FrameArgs) * max_batch));
    if ((r = slot_alloc(pl, pl->out))) return r;
    pl->view = &pl->out;
    if ((r = graphs_alloc(pl->graphs, graph_slots(pl)))) return r;
    const char *ng = getenv("REBVO_B200_NO_GRAPH");
    pl->use_graph = !(ng && ng[0] == '1');
    const char *sp = getenv("REBVO_B200_STAGE_PROF");
    pl->prof_on = sp && sp[0] == '1';
    if (pl->prof_on) {
        pl->use_graph = false;
        pl->pcap = max_batch * 12 + 8;
        pl->pev = new (std::nothrow) cudaEvent_t[pl->pcap]();
        pl->ptag = new (std::nothrow) int[pl->pcap];
        if (!pl->pev || !pl->ptag) return RB_ERR_ARG;
        for (int i = 0; i < pl->pcap; i++) RB_CUDA(cudaEventCreate(&pl->pev[i]));
    }
    {
        const char *mc = getenv("REBVO_B200_MAP_CHAIN");
        pl->map_chain = !(mc && atoi(mc) == 0);
        const char *ov = getenv("REBVO_B200_OVERLAP");
        pl->overlap = !(ov && ov[0] == '0') && !pl->prof_on;
        RB_CUDA(cudaStreamCreateWithFlags(&pl->det_stream, cudaStreamNonBlocking));
        RB_CUDA(cudaStreamCreateWithFlags(&pl->copy_stream, cudaStreamNonBlocking));
        const char *sb = getenv("REBVO_B200_SUB");
        pl->sub = sb ? atoi(sb) : 8;
        if (pl->sub < 1) pl->sub = max_batch;
        RB_CUDA(cudaMalloc(&pl->sb_dev, sizeof(SubBatchPtrs)));
        RB_CUDA(cudaMalloc(&pl->frames_dev, sizeof(rb_frame) * max_batch));
        RB_CUDA(cudaMalloc(&pl->det_mask_dev, sizeof(DetMask) * max_batch));
        RB_CUDA(cudaEventCreateWithFlags(&pl->ev_hop, cudaEventDisableTiming));
        for (int i = 0; i < 2; i++) {
            RB_CUDA(cudaEventCreateWithFlags(&pl->ev_trk[i], cudaEventDisableTiming));
            RB_CUDA(cudaEventCreateWithFlags(&pl->ev_copy[i], cudaEventDisableTiming));
        }
        // (the inline schedule where the rescaled keylines feed the next frame, or everything runs on one stream)
        if (pl->overlap && p->DoReScaling <= 0) {
            int lo = 0, hi = 0;
            RB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
            RB_CUDA(cudaStreamCreateWithPriority(&pl->resc_stream, cudaStreamNonBlocking, lo));   // minimiser blocks first
            RB_CUDA(cudaEventCreateWithFlags(&pl->ev_rjoin, cudaEventDisableTiming));
        }
    }
    for (int i = 0; i < 4; i++) RB_CUDA(cudaEventCreate(&pl->ev[i]));
    for (int i = 0; i < 8; i++) RB_CUDA(cudaEventCreate(&pl->user_ev[i]));
    pl->consumer = c->stream;
    if ((r = pl_reset_state(pl))) return r;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

extern "C" int rb_pipeline_set_imu(rb_pipeline *pl, const rb_imu_params *ip, const double *samples, int n) {
    if (!pl || !ip || !samples || n < 2) return RB_ERR_ARG;
    if (refuse_busy(pl, "set_imu")) return RB_ERR_STATE;
    if (!pl->imu) pl->imu = new (std::nothrow) ImuFlow();
    if (!pl->imu) return RB_ERR_ARG;
    ImuFlow &f = *pl->imu;
    f.ip = *ip;
    f.samples.resize(n);
    imu_rows(samples, n, f.samples.data());
    f.enabled = true;
    f.live = false;
    imu_flow_reset(f);
    return RB_OK;
}

extern "C" int rb_pipeline_set_imu_live(rb_pipeline *pl, const rb_imu_params *ip, double sample_time, int buffer_size) {
    if (!pl || !ip || !(sample_time > 0) || buffer_size < 1 || buffer_size == INT_MAX) return RB_ERR_ARG;
    if (refuse_busy(pl, "set_imu_live")) return RB_ERR_STATE;
    std::vector<rbimu::ImuSample> slots;
    try {
        slots.resize((size_t)buffer_size + 1);
    } catch (const std::bad_alloc &) {
        snprintf(pl->c->err, sizeof(pl->c->err), "set_imu_live: no host memory for %d samples", buffer_size);
        return RB_ERR_ARG;
    }
    if (!pl->imu) pl->imu = new (std::nothrow) ImuFlow();
    if (!pl->imu) return RB_ERR_ARG;
    ImuFlow &f = *pl->imu;
    f.samples.swap(slots);
    f.ip = *ip;
    f.enabled = true;
    f.live = true;
    f.t_last = -INFINITY;
    f.buf.init_live(f.samples.data(), buffer_size, sample_time, ip->use_se3 ? ip->Rc2i : nullptr,
                    ip->use_se3 ? ip->Tc2i : nullptr);
    imu_flow_reset(f);
    return RB_OK;
}

extern "C" int rb_pipeline_push_imu(rb_pipeline *pl, const double *samples, int n) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    if (!pl->imu || !pl->imu->live) {
        snprintf(c->err, sizeof(c->err), "push_imu: the pipeline is not in live IMU mode (rb_pipeline_set_imu_live)");
        return RB_ERR_ARG;
    }
    if (n < 0 || (n > 0 && !samples)) return RB_ERR_ARG;
    ImuFlow &f = *pl->imu;
    double t = f.t_last;
    for (int i = 0; i < n; i++) {
        if (!(samples[i * 7] >= t)) {   // (and NaN)
            snprintf(c->err, sizeof(c->err), "push_imu: sample %d at t=%.9f is older than the one before it (t=%.9f)", i,
                     samples[i * 7], t);
            return RB_ERR_ARG;
        }
        t = samples[i * 7];
    }
    if (n > f.buf.free_slots()) {
        snprintf(c->err, sizeof(c->err), "push_imu: %d samples do not fit in the ring (%d free slots): push frames to release "
                 "samples, then push these again", n, f.buf.free_slots());
        return RB_ERR_STATE;
    }
    std::vector<rbimu::ImuSample> rows(n);
    imu_rows(samples, n, rows.data());
    f.buf.push(rows.data(), n);
    if (n > 0) f.t_last = t;
    return RB_OK;
}

extern "C" void rb_pipeline_destroy(rb_pipeline *pl) {
    if (!pl) return;
    rb_ctx *c = pl->c;
    delete pl->imu;
    cudaSetDevice(c->device);
    // every stream first, so that no work still uses what is freed below; whatever a create that failed halfway did not
    // make yet is null.  (c->stream is the context's: rb_ctx_destroy destroys it.)
    cudaStream_t own[4 + RB_DEPTH_STREAMS] = {pl->det_stream, pl->resc_stream, pl->copy_stream, pl->mirror.stream};
    memcpy(own + 4, pl->depth.stream, sizeof(pl->depth.stream));
    cudaStreamSynchronize(c->stream);
    for (cudaStream_t s : own)
        if (s) cudaStreamSynchronize(s);
    for (cudaStream_t s : own)
        if (s) cudaStreamDestroy(s);
    async_free(pl);
    cudaEvent_t events[] = {pl->ev_hop, pl->ev_trk[0], pl->ev_trk[1], pl->ev_rjoin, pl->ev_copy[0], pl->ev_copy[1],
                            pl->ev[0], pl->ev[1], pl->ev[2], pl->ev[3]};
    for (cudaEvent_t e : events)
        if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : pl->user_ev)
        if (e) cudaEventDestroy(e);
    for (int i = 0; pl->pev && i < pl->pcap; i++)
        if (pl->pev[i]) cudaEventDestroy(pl->pev[i]);
    delete[] pl->pev;
    delete[] pl->ptag;
    graphs_free(pl->graphs);
    for (int i = 0; i < RB_NMAPS; i++)
        if (pl->maps[i]) rb_map_destroy(pl->maps[i]);
    if (pl->und) rb_undistort_destroy(pl->und);
    rb_dogws_free(&pl->ws);
    slot_free(pl->out);
    void *dev[] = {pl->chain, pl->fs, pl->nav_dev, pl->fa_dev, pl->sb_dev, pl->frames_dev, pl->odom.dev, pl->depth.stage,
                   pl->depth.ws, pl->det_mask_dev, pl->det_fixed};
    for (void *p : dev) cudaFree(p);
    if (pl->state_host) cudaFreeHost(pl->state_host);
    rb_ctx_destroy(c);
    delete pl;
}

extern "C" const char *rb_pipeline_last_error(const rb_pipeline *pl) { return pl ? pl->c->err : "null pipeline"; }
extern "C" int64_t rb_pipeline_launch_count(const rb_pipeline *pl) { return pl->c->launches; }
extern "C" void *rb_pipeline_stream(rb_pipeline *pl) { return (void *)pl->c->stream; }
extern "C" rb_map *rb_pipeline_map(rb_pipeline *pl, int age) {
    if (age < 0 || age > 1 || pl->n_pushed <= age || (age == 1 && pl->restored)) return nullptr;
    return pl->maps[(pl->n_pushed - 1 - age) % RB_NMAPS];
}
extern "C" int rb_pipeline_stage_ms(const rb_pipeline *pl, float out[6]) {
    if (refuse_busy(const_cast<rb_pipeline *>(pl), "stage_ms")) return RB_ERR_STATE;
    memcpy(out, pl->stage_ms, sizeof(float) * 6);
    return RB_OK;
}

extern "C" int rb_pipeline_reset(rb_pipeline *pl) {
    rb_ctx *c = pl->c;
    if (refuse_busy(pl, "reset")) return RB_ERR_STATE;
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
static int track_frame(rb_pipeline *pl, rb_map *neu, rb_map *old, const FrameArgs *fa, rb_nav *nav_slot,
                       rb_odometry *odom_slot) {
    rb_ctx *c = pl->c;
    const rb_params &p = pl->p;
    int r;
    RB_TRACE(c->stream, 1);
    // :167-169 loop-body start (folded into the quantile kernel) ; :172  s_rho_q = old_buf.ef->EstimateQuantile(...)
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
    // (since the old map's update only EstimateQuantile -- and build_field of the NEW map without the second stream -- ran
    // on this stream: the minimiser may stage the old map's operands while that kernel is still running)
    c->min_early = getenv("REBVO_B200_MIN_EARLY") ? atoi(getenv("REBVO_B200_MIN_EARLY")) != 0 : true;
    // (the one-thread stage after the minimiser and FordwardMatch's arg-max run in its epilogue / last evaluation)
    r = rb_minimizer_enqueue(c, neu, old, pl->fs->VW, &a, 0.0, true, 0, true, pl->fs);
    c->min_early = false;
    if (r) return r;
    RB_TRACE(c->stream, 3);
    prof_mark(pl, ST_MINIM);
    // :480-487 EstimateReScalingOpt and :545-585 pose integration + NavData: in one cluster kernel (k_map_update) after the
    // EKF, or with the rescaling stream, pose integration + NavData ride in the EKF kernel and the rescaling leaves the chain.
    // (Not with the 168-byte keyline mirror: there the inline schedule measured 2-3 % faster on H100, while the 15-byte
    // records gain from the side stream like the plain push; set_mirror drops the captured batches.)
    const bool side = pl->resc_stream != nullptr && pl->mirror.on != 1;
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
                                    p.LocationUncertainty, pl->fs->R0, side ? nav_slot : nullptr, fa, odom_slot)))
            return r;
    } else {
        // The reference's order (rebvo_second_t.cpp:354-470) on the stage kernels that tests/test_gpu_parity.py and
        // tests/test_gpu_mapper_states.py pin to the reference: the bitwise reference of the two kernels above
        // (tests/test_gpu_map_chain.py), not a schedule to tune.  k_rotate writes the old map's rho / s_rho, which its
        // rescaling reads: joined before the first kernel.
        if ((r = resc_join(pl))) return r;
        // :354  FordwardMatch (its arg-max ran with the minimiser) ; :369 rotate_keylines(R0)
        if ((r = rb_forward_match_apply_enqueue(c, old, neu))) return r;
        if ((r = rb_rotate_enqueue(c, old, pl->fs->R0))) return r;
        RB_TRACE(c->stream, 11);
        prof_mark(pl, ST_FWD_ROT);
        // :410  directed_matching(V,P_V,R,old_buf.ef,...)
        if ((r = rb_directed_matching_enqueue(c, neu, old, &pl->fs->dm, p.MatchThreshModule, p.MatchThreshAngle,
                                              (double)p.SearchRange, p.LocationUncertaintyMatch, &pl->fs->do_match)))
            return r;
        RB_TRACE(c->stream, 4);
        prof_mark(pl, ST_DMATCH);
        // :410-423 match-count gate ; :452-470 Regularize_1_iter, UpdateInverseDepthKalman
        k_frame_post_match<<<1, 1, 0, c->stream>>>(pl->fs, neu->st, p.MatchThreshold, neu->ts, odom_slot);
        RB_LAUNCH_CHECK();
        if ((r = rb_regularize_enqueue(c, neu, p.RegularizeThresh, &pl->fs->do_map))) return r;
        if ((r = rb_ekf_enqueue(c, neu, pl->fs->V, p.ReshapeQAbsolute, p.LocationUncertainty, &pl->fs->do_map))) return r;
        if (side) {   // :545-585 pose integration + NavData (else in k_map_update's tail)
            k_frame_finish<<<1, 1, 0, c->stream>>>(pl->fs, neu->st, old->st, neu->ts, nav_slot, fa);
            RB_LAUNCH_CHECK();
        }
    }
    RB_TRACE(c->stream, 9);
    prof_mark(pl, ST_REG_EKF);
    if (side) {   // gated by the map's own copy of do_map; writes the map's Kp / RKp and the record's, no FrameState
        cudaStream_t main_stream = c->stream;
        if ((r = stream_wait(pl, main_stream, pl->resc_stream))) return r;
        c->stream = pl->resc_stream;
        r = rb_rescale_enqueue(c, neu, RB_RHO_MAX, 1, 0, &neu->st->do_map, nav_slot);
        c->stream = main_stream;
        if (r) return r;
        RB_CUDA(cudaEventRecord(pl->ev_rjoin, pl->resc_stream));
        pl->resc_open = true;
        RB_TRACE(c->stream, 5);
        return RB_OK;
    }
    if ((r = rb_map_update_enqueue(c, neu, RB_RHO_MAX, 1, p.DoReScaling > 0 ? 1 : 0, pl->fs, old->st, nav_slot, fa)))
        return r;
    prof_mark(pl, ST_RESCALE);   // rescaling + pose integration / nav record (folded)
    RB_TRACE(c->stream, 5);
    prof_mark(pl, ST_FINISH);
    return RB_OK;
}

// the front of a batch, after the H2D copy: its gray plane (rebvo_first_t.cpp:231 undistortion + RGB -> BW) from the
// frames at tbl->src, or through frames_dev for the strided layouts, then the batched scale space, into ws
static int enqueue_front(rb_pipeline *pl, DogWS *ws, SubBatchPtrs *tbl, const rb_frame *frames_dev, int fmt, int n,
                         bool with_events) {
    rb_ctx *c = pl->c;
    int r;
    prof_mark(pl, ST_H2D);
    if ((r = rb_gray_enqueue(c, ws, pl->und, in_mono(fmt), &tbl->src, in_strided(fmt) ? frames_dev : nullptr, n))) return r;
    prof_mark(pl, ST_GRAY);
    if (with_events) RB_CUDA(cudaEventRecord(pl->ev[1], c->stream));
    if ((r = rb_dog_build_batch(c, ws, n))) return r;
    prof_mark(pl, ST_DOG);
    if (with_events) RB_CUDA(cudaEventRecord(pl->ev[2], c->stream));
    return RB_OK;
}

// the back of a batch: per frame detect + track + map on the scale space in ws, and the per-frame outputs.  masked: frame i
// detects through the detection masks of det_mask_dev[i].
static int enqueue_back(rb_pipeline *pl, const DogWS *ws, int n, long long first_frame, bool masked) {
    rb_ctx *c = pl->c;
    const rb_params &p = pl->p;
    int r;
    pl->resc_open = false;   // (a batch joins its last rescaling at its end; a failed enqueue must not leave a join behind)
    // Two streams, like the reference's first and second thread: the detector of frame f+1 only needs the scale space
    // and the previous detector state (threshold chain), so it runs on det_stream while the main stream tracks
    // frame f.  detect(f) overwrites the map of frame f-3, which track(f-2) was the last to read.
    cudaStream_t main_stream = c->stream;
    const bool ov = pl->overlap;
    if (ov && (r = stream_wait(pl, main_stream, pl->det_stream))) return r;
    SubBatchPtrs *tbl = pl->sb_dev;
    for (int i = 0; i < n; i++) {
        const long long fr = first_frame + i;
        rb_map *neu = pl->maps[fr % RB_NMAPS], *old = pl->maps[(fr + RB_NMAPS - 1) % RB_NMAPS];
        const float *img0 = ws->img0 + (size_t)i * c->NP, *dog = ws->dog + (size_t)i * c->NP;
        // FirstThr: detect + reEstimateThresh (rebvo_first_t.cpp:266-272)
        if (ov) {
            if (i >= 2) RB_CUDA(cudaStreamWaitEvent(pl->det_stream, pl->ev_trk[i % 2], 0));   // track(i-2)
            c->stream = pl->det_stream;
        }
        RB_TRACE(c->stream, 6);
        r = rb_detect_enqueue(c, neu, img0, dog, &p.det, pl->chain, masked ? pl->det_mask_dev + i : nullptr);
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
        if (ov && (r = stream_wait(pl, pl->det_stream, main_stream))) return r;
        if (fr == 0) {
            k_frame_first<<<1, 1, 0, c->stream>>>(pl->fs, neu->st, pl->nav_dev + i, pl->fa_dev + i);
            RB_LAUNCH_CHECK();
        } else {
            if ((r = track_frame(pl, neu, old, pl->fa_dev + i, pl->nav_dev + i, pl->odom.on ? pl->odom.dev + i : nullptr)))
                return r;
        }
        if (pl->mirror.on) {   // the frame's edge map as the reference's records, before the next frame touches it
            const size_t ofs = (size_t)i * pl->mirror.stride;
            if (pl->mirror.on == 1)
                r = rb_map_pack_aos_enqueue(c, neu, tbl->mirror, ofs);
            else   // copy_net_keyline(..., pbuf.K) of the third thread (rebvo_third_t.cpp:192-197): K of this frame's nav record
                r = rb_map_pack_net_enqueue(c, neu, tbl->mirror, ofs, &(pl->nav_dev + i)->K);
            if (r) return r;
            if (!pl->out_dev) {   // (device mode: the staging slot is the output)
                if ((r = stream_wait(pl, main_stream, pl->mirror.stream))) return r;
                k_mirror_to_host<<<8, 256, 0, pl->mirror.stream>>>(tbl->mirror, ofs, &(pl->nav_dev + i)->kn,
                                                                   (int)pl->mirror.rec);
                RB_LAUNCH_CHECK();
            }
        }
        if (pl->depth.on) {   // the viewer's depth_filler on this frame's wire records (visualizer.cpp:436-440)
            unsigned char *const *rec_pp = tbl->mirror;
            size_t rec_ofs = (size_t)i * pl->mirror.stride;
            if (pl->mirror.on != 2) {   // copy_net_keyline(..., pbuf.K) of the third thread (rebvo_third_t.cpp:191)
                rec_pp = tbl->depth;
                rec_ofs = (size_t)i * pl->depth.rec_stride;
                if ((r = rb_map_pack_net_enqueue(c, neu, tbl->depth, rec_ofs, &(pl->nav_dev + i)->K))) return r;
            }
            const int k = i % RB_DEPTH_STREAMS;
            if ((r = stream_wait(pl, main_stream, pl->depth.stream[k]))) return r;
            c->stream = pl->depth.stream[k];
            void *ws = (unsigned char *)pl->depth.ws + (size_t)k * pl->depth.ws_bytes;
            r = rb_depth_fill_enqueue(c, pl->depth.plan, rec_pp, rec_ofs, nullptr, &(pl->nav_dev + i)->kn, 0, c->kcap, ws,
                                      tbl->depth, (size_t)i * pl->depth.plan.cells_bytes, nullptr, pl->dimg.mode != 0);
            if (!r && pl->dimg.mode)   // depth_filler::getImgRho at every pixel, from the cells the fill left in ws
                r = rb_depth_image_enqueue(c, pl->dimg.plan, (const double *)rb_depth_ws_final(pl->depth.plan, c->kcap, ws), 2,
                                           reinterpret_cast<float *const *>(tbl->depth + 2), (size_t)i * pl->dimg.stride,
                                           nullptr, pl->dimg.plane);
            c->stream = main_stream;
            if (r) return r;
        }
        if (ov && i + 2 < n) RB_CUDA(cudaEventRecord(pl->ev_trk[i % 2], main_stream));
    }
    if ((r = resc_join(pl))) return r;   // the last frame's Kp / RKp are in its record before the nav copy
    // the batch is complete when its last map has reached the host, and its last grids
    if (pl->mirror.on && !pl->out_dev && (r = stream_wait(pl, pl->mirror.stream, main_stream))) return r;
    for (int k = 0; pl->depth.on && k < RB_DEPTH_STREAMS && k < n; k++)
        if ((r = stream_wait(pl, pl->depth.stream[k], main_stream))) return r;
    return RB_OK;
}

// everything of a batch after the H2D copy, on the tracker stream in the pipeline's workspace: front, then back
static int enqueue_batch(rb_pipeline *pl, int fmt, int n, long long first_frame, bool with_events, bool masked) {
    int r = enqueue_front(pl, &pl->ws, pl->sb_dev, pl->frames_dev, fmt, n, with_events);
    return r ? r : enqueue_back(pl, &pl->ws, n, first_frame, masked);
}

// Capture the work body() enqueues on stream s (and the streams it forks) as one graph, instantiated into *exec; *launches
// receives the kernels it launches, which are counted at each replay and not at the capture.
template <class F>
static int capture_graph(rb_pipeline *pl, cudaStream_t s, F &&body, cudaGraphExec_t *exec, int *launches) {
    rb_ctx *c = pl->c;
    cudaGraph_t g = nullptr;
    const int64_t l0 = c->launches;
    RB_CUDA(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    int r = body();
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (r) {
        if (g) cudaGraphDestroy(g);
        return r;
    }
    if (e != cudaSuccess) {
        snprintf(c->err, sizeof(c->err), "graph capture: %s", cudaGetErrorString(e));
        return RB_ERR_CUDA;
    }
    *launches = (int)(c->launches - l0);
    c->launches = l0;
    e = cudaGraphInstantiate(exec, g, 0);
    cudaGraphDestroy(g);
    if (e != cudaSuccess) {
        *exec = nullptr;
        snprintf(c->err, sizeof(c->err), "graph instantiate: %s", cudaGetErrorString(e));
        return RB_ERR_CUDA;
    }
    return RB_OK;
}

// Launch graph `key` of g on stream s.  One that is not captured yet is captured first, together with those of its nsib
// siblings that are missing: sibling i is graph sib_key(i) with the body sib_body(i), and the key is one of them.
template <class K, class B>
static int graph_launch(rb_pipeline *pl, GraphCache &g, cudaStream_t s, int key, int nsib, K &&sib_key, B &&sib_body) {
    rb_ctx *c = pl->c;
    int r;
    if (!g.exec[key])
        for (int i = 0; i < nsib; i++) {
            const int k = sib_key(i);
            if (g.exec[k]) continue;
            auto body = [&]() { return sib_body(i); };
            if ((r = capture_graph(pl, s, body, &g.exec[k], &g.launches[k]))) return r;
        }
    RB_CUDA(cudaGraphLaunch(g.exec[key], s));
    c->launches += g.launches[key];
    return RB_OK;
}

// a synchronous push of input that push_in has checked, into the pipeline's slot
static int push_impl(rb_pipeline *pl, const PushIn &in, rb_nav *nav_out) {
    rb_ctx *c = pl->c;
    if (refuse_busy(pl, "push")) return RB_ERR_STATE;
    const int n = in.n;
    int r;
    if (pl->imu && pl->imu->live && (r = imu_live_check(pl, *pl->imu, in.ts, n))) return r;
    RB_CUDA(cudaSetDevice(c->device));
    OutSlot &s = pl->out;
    show(pl, s, 0);
    pl->last_sub = 0;
    write_args(pl, s, in.ts, n);
    const bool masked = fill_masks(pl, in.masks, n, s);
    if (pl->imu) {   // IMU mode: host-driven frame loop (imu_flow.cuh)
        if ((r = imu_push(pl, *pl->imu, in, masked))) return r;
        RB_CUDA(cudaStreamSynchronize(c->stream));
        pl->last_sub = n;   // (one scale-space batch)
        if (nav_out) memcpy(nav_out, s.nav, sizeof(rb_nav) * n);
        pl->odom.n = pl->odom.on ? n : 0;
        return RB_OK;
    }
    // device outputs: nothing of this push may overwrite them before the consumer's reads of the last push's are done.  The
    // side streams that write them fork from the tracker stream, so one wait at its head covers them (outside any graph).
    if (pl->out_dev && pl->consumer != c->stream && (r = stream_wait(pl, pl->consumer, c->stream))) return r;
    pl->pn = 0;
    prof_mark(pl, ST_NAV);   // origin of this push
    RB_CUDA(cudaEventRecord(pl->ev[0], c->stream));
    // sub-batches: device input = one (the caller's buffer is read in place).  Host input = a short head (pl->sub
    // frames) and the rest: only the head's H2D copy is exposed, the rest of the frames are copied on the copy stream into
    // their own staging region while the head computes (a frame costs ~8x more to track than to copy), and the scale
    // space of the rest still runs as one large batch.
    int soff[3] = {0, n, n}, nsub = 1;
    if (!(in.on_device || pl->prof_on || n < 3 * pl->sub)) {
        soff[1] = pl->sub;
        nsub = 2;
    }
    if ((r = stage_push(pl, in, soff, nsub))) return r;
    const size_t fbytes = frame_bytes(c, in.fmt);   // (ws.rgb holds max_batch frames of either format)
    for (int j = 0; j < nsub; j++) {
        const int off = soff[j], nj = soff[j + 1] - soff[j];
        const long long first_j = s.first + off;
        if (!in.on_device && nsub > 1) RB_CUDA(cudaStreamWaitEvent(c->stream, pl->ev_copy[j], 0));
        RB_CUDA(cudaMemcpyAsync(pl->fa_dev, s.fa + off, sizeof(FrameArgs) * nj, cudaMemcpyHostToDevice, c->stream));
        const void *src = in.on_device ? (const void *)in.data : (const void *)(pl->ws.rgb + (size_t)off * fbytes);
        if ((r = write_tables(pl, s, j, src, off, nj, masked))) return r;   // (strided: src unused)
        if (!pl->use_graph || first_j == 0) {
            if ((r = enqueue_batch(pl, in.fmt, nj, first_j, j == 0, masked))) return r;
        } else {
            // capture the batch once per ring phase (from any first frame > 0 of that phase); replays only differ through
            // fa_dev / sb_dev contents.  All phases of this format and batch size are instantiated together, so that no later
            // push pays for a capture.  The other format's graphs are left as they are: a stream may alternate formats.
            if (j == 0) RB_CUDA(cudaEventRecord(pl->ev[1], c->stream));
            auto sib_key = [&](int ph) { return graph_slot(pl, masked, in.fmt, ph, nj); };
            auto sib_body = [&](int ph) { return enqueue_batch(pl, in.fmt, nj, ph == 0 ? RB_NMAPS : ph, false, masked); };
            if ((r = graph_launch(pl, pl->graphs, c->stream, sib_key((int)(first_j % RB_NMAPS)), RB_NMAPS, sib_key, sib_body)))
                return r;
            if (j == 0) RB_CUDA(cudaEventRecord(pl->ev[2], c->stream));
        }
        RB_CUDA(cudaMemcpyAsync(s.nav + off, pl->nav_dev, sizeof(rb_nav) * nj, cudaMemcpyDeviceToHost, c->stream));
        if (pl->odom.on)
            RB_CUDA(cudaMemcpyAsync(s.odom + off, pl->odom.dev, sizeof(rb_odometry) * nj, cudaMemcpyDeviceToHost, c->stream));
    }
    for (int k = 0; k < RB_NMAPS; k++)
        RB_CUDA(cudaMemcpyAsync(&s.abort[k], &pl->maps[k]->ts_host.ctl->abort, sizeof(int), cudaMemcpyDeviceToHost,
                                c->stream));
    pl->t_prev = in.ts[n - 1];
    pl->n_pushed += n;
    pl->restored = false;
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
    if (nav_out) memcpy(nav_out, s.nav, sizeof(rb_nav) * n);
    pl->last_sub = soff[nsub] - soff[nsub - 1];
    show(pl, s, n);
    if ((r = retire(pl, s))) {   // (checked on every push; the flags are cleared for the next one)
        for (int k = 0; k < RB_NMAPS; k++) cudaMemset(&pl->maps[k]->ts_host.ctl->abort, 0, sizeof(int));
        return r;
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

// the opening of the set_* calls, under RB_ENTER: refused in IMU mode when `imu_refused` names the call, then the pushes
// enqueued so far finish, so that the call may replace what they use
static int set_begin(rb_pipeline *pl, const char *imu_refused) {
    rb_ctx *c = pl->c;
    RB_CUDA(cudaSetDevice(c->device));
    if (refuse_busy(pl, "set_* call")) return RB_ERR_STATE;
    if (imu_refused && pl->imu) {
        snprintf(c->err, sizeof(c->err), "%s: not available in IMU mode", imu_refused);
        return RB_ERR_ARG;
    }
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}
// the ring and everything it owns (no ticket outstanding, or the pipeline is being destroyed); the outputs of a ticket it
// held are gone with it
static void async_free(rb_pipeline *pl) {
    AsyncRing *ar = pl->ar;
    if (!ar) return;
    if (ar->front) {
        cudaStreamSynchronize(ar->front);
        cudaStreamDestroy(ar->front);
    }
    graphs_free(ar->front_graphs);
    graphs_free(ar->back_graphs);
    cudaEvent_t events[] = {ar->ev_front[0], ar->ev_front[1], ar->ev_free[0], ar->ev_free[1]};
    for (cudaEvent_t e : events)
        if (e) cudaEventDestroy(e);
    for (OutSlot &s : ar->slot) slot_free(s);
    for (int k = 0; k < 2; k++) {
        cudaFree(ar->front_dev[k]);
        cudaFree(ar->frames_dev[k]);
    }
    rb_dogws_free(&ar->ws1);
    if (pl->view != &pl->out) show(pl, pl->out, 0);
    delete ar;
    pl->ar = nullptr;
}
static int async_alloc(rb_pipeline *pl, int depth) {
    rb_ctx *c = pl->c;
    AsyncRing *ar = new (std::nothrow) AsyncRing();
    if (!ar) return RB_ERR_ARG;
    memset(ar, 0, sizeof(*ar));
    pl->ar = ar;
    ar->depth = depth;
    int r;
    if ((r = rb_dogws_alloc(c, &ar->ws1, pl->max_batch))) return r;
    // lowest priority: the back of the ticket before is the critical path, and a front has the whole of it to finish in
    int lo = 0, hi = 0;
    RB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    RB_CUDA(cudaStreamCreateWithPriority(&ar->front, cudaStreamNonBlocking, lo));
    for (int k = 0; k < 2; k++) {
        RB_CUDA(cudaEventCreateWithFlags(&ar->ev_front[k], cudaEventDisableTiming));
        RB_CUDA(cudaEventCreateWithFlags(&ar->ev_free[k], cudaEventDisableTiming));
        RB_CUDA(cudaMalloc(&ar->front_dev[k], sizeof(SubBatchPtrs)));
        RB_CUDA(cudaMalloc(&ar->frames_dev[k], sizeof(rb_frame) * pl->max_batch));
    }
    if ((r = graphs_alloc(ar->front_graphs, afront_slots(pl))) || (r = graphs_alloc(ar->back_graphs, aback_slots(pl))))
        return r;
    for (int k = 0; k < depth; k++) {
        if ((r = slot_alloc(pl, ar->slot[k]))) return r;
        RB_CUDA(cudaEventCreateWithFlags(&ar->slot[k].done, cudaEventDisableTiming));
    }
    return grow_outputs(pl);
}

extern "C" int rb_pipeline_set_undistort(rb_pipeline *pl, const double kc[5]) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    int r = set_begin(pl, nullptr);
    if (r) return r;
    if (pl->und) {
        rb_undistort_destroy(pl->und);
        pl->und = nullptr;
    }
    bool any = false;
    for (int i = 0; kc && i < 5; i++) any = any || kc[i] != 0.0;
    if (any && (r = rb_undistort_create(c, kc, &pl->und))) {
        if (pl->und) rb_undistort_destroy(pl->und);
        pl->und = nullptr;
        return r;
    }
    drop_graphs(pl);   // the captured batches contain the other gray kernel (both input formats)
    return RB_OK;
}
extern "C" int rb_pipeline_set_mirror(rb_pipeline *pl, int on) {
    if (!pl || on < 0 || on > 2) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    int r = set_begin(pl, "set_mirror");
    if (r) return r;
    const size_t stride = ((size_t)c->kcap * sizeof(rb_keyline) + 255) & ~(size_t)255;   // (sized for the larger record)
    if (on && !pl->mirror.stream) RB_CUDA(cudaStreamCreateWithFlags(&pl->mirror.stream, cudaStreamNonBlocking));
    if (on != pl->mirror.on) drop_graphs(pl);   // the captured batches contain (or not) the pack kernels
    pl->mirror.on = on;
    pl->mirror.rec = on == 2 ? 15 : sizeof(rb_keyline);
    pl->mirror.stride = stride;
    pl->mirror.n = 0;
    return grow_outputs(pl);
}
extern "C" int rb_pipeline_set_depth(rb_pipeline *pl, const rb_depth_params *p) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    int r = set_begin(pl, "set_depth");
    if (r) return r;
    if (!p) {
        if (pl->depth.on) drop_graphs(pl);   // the captured batches contain the pack and fill kernels
        pl->depth.on = 0;
        pl->depth.n = 0;
        pl->dimg.n = 0;
        return RB_OK;
    }
    DepthPlan plan;
    if ((r = rb_depth_plan(c, p, &plan))) {
        snprintf(c->err, sizeof(c->err), "set_depth: invalid parameters");
        return r;
    }
    if (!pl->depth.stage) {
        pl->depth.rec_stride = ((size_t)c->kcap * 15 + 255) & ~(size_t)255;
        RB_CUDA(cudaMalloc(&pl->depth.stage, (size_t)pl->max_batch * pl->depth.rec_stride));
        // lowest priority: a fill CTA may hold a whole SM's shared memory, which the tracker's kernels get first
        // (env REBVO_B200_DEPTH_PRIO=1: the tracker's own priority, for tools/bench_depth.py's comparison)
        int lo = 0, hi = 0;
        RB_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
        const char *dp = getenv("REBVO_B200_DEPTH_PRIO");
        for (int k = 0; k < RB_DEPTH_STREAMS; k++)
            RB_CUDA(cudaStreamCreateWithPriority(&pl->depth.stream[k], cudaStreamNonBlocking, (dp && atoi(dp) == 1) ? hi : lo));
    }
    const size_t ws_bytes = rb_depth_ws_bytes(plan, c->kcap);
    if (ws_bytes > pl->depth.ws_bytes) {
        cudaFree(pl->depth.ws);
        pl->depth.ws = nullptr;
        pl->depth.ws_bytes = 0;
        RB_CUDA(cudaMalloc(&pl->depth.ws, ws_bytes * RB_DEPTH_STREAMS));
        pl->depth.ws_bytes = ws_bytes;
    }
    if (pl->dimg.mode && (r = rb_depth_image_plan(c, plan.g, pl->dimg.mode, &pl->dimg.plan))) return r;
    drop_graphs(pl);   // the captured batches hold the fill's geometry
    pl->depth.plan = plan;
    pl->depth.on = 1;
    pl->depth.n = 0;
    pl->dimg.n = 0;
    return grow_outputs(pl);
}
extern "C" int rb_pipeline_depth(rb_pipeline *pl, int i, const rb_depth_cell **cells, int *gw, int *gh, double *min_dist) {
    if (!pl || !cells) return RB_ERR_ARG;
    if (pl->out_dev) return RB_ERR_STATE;
    if (!pl->depth.on || i < 0 || i >= pl->depth.n) return RB_ERR_ARG;
    const DepthGeom &g = pl->depth.plan.g;
    const unsigned char *slot = pl->view->depth_host + (size_t)i * pl->depth.plan.cells_bytes;
    *cells = reinterpret_cast<const rb_depth_cell *>(slot);
    if (gw) *gw = g.gw;
    if (gh) *gh = g.gh;
    if (min_dist) *min_dist = *reinterpret_cast<const double *>(slot + (size_t)g.gw * g.gh * sizeof(rb_depth_cell));
    return RB_OK;
}
extern "C" int rb_pipeline_set_depth_image(rb_pipeline *pl, int mode) {
    if (!pl || mode < 0 || mode > 2) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    int r = set_begin(pl, "set_depth_image");
    if (r) return r;
    if (mode) {
        const size_t plane = ((size_t)c->N + 63) & ~(size_t)63, stride = (size_t)mode * plane * sizeof(float);
        if (pl->depth.on && (r = rb_depth_image_plan(c, pl->depth.plan.g, mode, &pl->dimg.plan))) return r;
        pl->dimg.plane = plane;
        pl->dimg.stride = stride;
    }
    if (mode != pl->dimg.mode) drop_graphs(pl);   // the captured batches contain (or not) the image pass
    pl->dimg.mode = mode;
    pl->dimg.n = 0;
    return grow_outputs(pl);
}
extern "C" int rb_pipeline_depth_image(rb_pipeline *pl, int i, const float **rho, const float **s_rho) {
    if (!pl || !rho) return RB_ERR_ARG;
    if (pl->out_dev) return RB_ERR_STATE;
    if (i < 0 || i >= pl->dimg.n) return RB_ERR_ARG;
    const float *p = reinterpret_cast<const float *>(pl->view->dimg_host + (size_t)i * pl->dimg.stride);
    *rho = p;
    if (s_rho) *s_rho = pl->dimg.mode == 2 ? p + pl->dimg.plane : nullptr;
    return RB_OK;
}
extern "C" int rb_pipeline_set_odometry(rb_pipeline *pl, int on) {
    if (!pl || on < 0 || on > 1) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    int r = set_begin(pl, nullptr);
    if (r) return r;
    if (on && !pl->odom.dev) RB_CUDA(cudaMalloc(&pl->odom.dev, sizeof(rb_odometry) * pl->max_batch));
    if (on != pl->odom.on) drop_graphs(pl);   // the captured batches pass (or not) the record slots to their kernels
    pl->odom.on = on;
    pl->odom.n = 0;
    return grow_outputs(pl);
}
extern "C" int rb_pipeline_odometry(rb_pipeline *pl, const rb_odometry **recs, int *n) {
    if (!pl || !recs || !n) return RB_ERR_ARG;
    if (!pl->odom.n) return RB_ERR_STATE;
    *recs = pl->view->odom;
    *n = pl->odom.n;
    return RB_OK;
}
extern "C" int rb_pipeline_mirror(rb_pipeline *pl, int i, const void **records, int *n) {
    if (!pl || !records || !n) return RB_ERR_ARG;
    if (pl->out_dev) return RB_ERR_STATE;
    if (!pl->mirror.on || i < 0 || i >= pl->mirror.n) return RB_ERR_ARG;
    *records = pl->view->mirror_host + (size_t)i * pl->mirror.stride;
    *n = pl->view->nav[i].kn;
    return RB_OK;
}

extern "C" int rb_pipeline_set_output_memory(rb_pipeline *pl, int where) {
    if (!pl || where < 0 || where > 1) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    int r = set_begin(pl, "set_output_memory");
    if (r) return r;
    if (where == pl->out_dev) return RB_OK;
    // the buffers of the products that are on, in the new place; the other place's stay for a switch back
    const int was = pl->out_dev;
    pl->out_dev = where;
    if ((r = grow_outputs(pl))) {
        pl->out_dev = was;
        return r;
    }
    drop_graphs(pl);   // the captured batches contain (or not) k_mirror_to_host and its join
    pl->mirror.n = pl->depth.n = pl->dimg.n = 0;
    return RB_OK;
}
extern "C" int rb_pipeline_set_consumer_stream(rb_pipeline *pl, void *stream) {
    if (!pl) return RB_ERR_ARG;
    RB_ENTER(pl->c);
    if (refuse_busy(pl, "set_consumer_stream")) return RB_ERR_STATE;
    pl->consumer = (cudaStream_t)stream;
    return RB_OK;
}
extern "C" int rb_pipeline_mirror_dev(rb_pipeline *pl, int i, const void **records, int *n) {
    if (!pl || !records || !n) return RB_ERR_ARG;
    if (!pl->out_dev) return RB_ERR_STATE;
    if (!pl->mirror.on || i < 0 || i >= pl->mirror.n) return RB_ERR_ARG;
    *records = pl->view->mirror_dev + (size_t)i * pl->mirror.stride;
    *n = pl->view->nav[i].kn;
    return RB_OK;
}
extern "C" int rb_pipeline_depth_dev(rb_pipeline *pl, int i, const rb_depth_cell **cells, int *gw, int *gh,
                                     const double **min_dist) {
    if (!pl || !cells) return RB_ERR_ARG;
    if (!pl->out_dev) return RB_ERR_STATE;
    if (!pl->depth.on || i < 0 || i >= pl->depth.n) return RB_ERR_ARG;
    const DepthGeom &g = pl->depth.plan.g;
    const unsigned char *slot = pl->view->depth_dev + (size_t)i * pl->depth.plan.cells_bytes;
    *cells = reinterpret_cast<const rb_depth_cell *>(slot);
    if (gw) *gw = g.gw;
    if (gh) *gh = g.gh;
    if (min_dist) *min_dist = reinterpret_cast<const double *>(slot + (size_t)g.gw * g.gh * sizeof(rb_depth_cell));
    return RB_OK;
}
extern "C" int rb_pipeline_depth_image_dev(rb_pipeline *pl, int i, const float **rho, const float **s_rho) {
    if (!pl || !rho) return RB_ERR_ARG;
    if (!pl->out_dev) return RB_ERR_STATE;
    if (i < 0 || i >= pl->dimg.n) return RB_ERR_ARG;
    const float *p = reinterpret_cast<const float *>(pl->view->dimg_dev + (size_t)i * pl->dimg.stride);
    *rho = p;
    if (s_rho) *s_rho = pl->dimg.mode == 2 ? p + pl->dimg.plane : nullptr;
    return RB_OK;
}

// the synchronous pushes' C entry points: push_in's checks, then push_impl
static int push(rb_pipeline *pl, const char *what, PushIn in, rb_nav *nav_out) {
    if (!pl) return RB_ERR_ARG;
    const int r = push_in(pl, what, in);
    return r ? r : push_impl(pl, in, nav_out);
}
extern "C" int rb_pipeline_push(rb_pipeline *pl, const uint8_t *rgb, const double *ts, int n, rb_nav *nav_out) {
    return push(pl, "push", {rgb, nullptr, RB_FRAME_RGB24, false, false, nullptr, ts, n}, nav_out);
}
extern "C" int rb_pipeline_push_dev(rb_pipeline *pl, const uint8_t *rgb_dev, const double *ts, int n,
                                    rb_nav *nav_out) {
    return push(pl, "push_dev", {rgb_dev, nullptr, RB_FRAME_RGB24, true, false, nullptr, ts, n}, nav_out);
}
extern "C" int rb_pipeline_push_mono(rb_pipeline *pl, const uint8_t *mono, const double *ts, int n, rb_nav *nav_out) {
    return push(pl, "push_mono", {mono, nullptr, RB_FRAME_MONO8, false, false, nullptr, ts, n}, nav_out);
}
extern "C" int rb_pipeline_push_mono_dev(rb_pipeline *pl, const uint8_t *mono_dev, const double *ts, int n,
                                         rb_nav *nav_out) {
    return push(pl, "push_mono_dev", {mono_dev, nullptr, RB_FRAME_MONO8, true, false, nullptr, ts, n}, nav_out);
}
extern "C" int rb_pipeline_push_frames(rb_pipeline *pl, int format, const rb_frame *frames, const double *ts, int n,
                                       rb_nav *nav_out) {
    return push(pl, "push_frames", {nullptr, frames, format, false, false, nullptr, ts, n}, nav_out);
}
extern "C" int rb_pipeline_push_frames_dev(rb_pipeline *pl, int format, const rb_frame *frames, const double *ts, int n,
                                           rb_nav *nav_out) {
    return push(pl, "push_frames", {nullptr, frames, format, true, false, nullptr, ts, n}, nav_out);
}

// ---- detection masks (DESIGN.md §5) --------------------------------------------------------------------------------------
extern "C" int rb_pipeline_set_detect_mask(rb_pipeline *pl, const uint8_t *mask, int64_t step, int on_device) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    if (mask && step < c->w) {
        snprintf(c->err, sizeof(c->err), "set_detect_mask: step %lld is shorter than a row (%d bytes)", (long long)step, c->w);
        return RB_ERR_ARG;
    }
    int r = set_begin(pl, nullptr);
    if (r) return r;
    // (no captured batch changes: masked pushes read the fixed mask through det_mask_dev, unmasked ones never see it)
    pl->det_fixed_on = false;
    if (!mask) return RB_OK;
    if (!pl->det_fixed) RB_CUDA(cudaMalloc(&pl->det_fixed, (size_t)c->N));
    RB_CUDA(cudaMemcpy2DAsync(pl->det_fixed, (size_t)c->w, mask, (size_t)step, (size_t)c->w, c->h,
                              on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    pl->det_fixed_on = true;
    return RB_OK;
}
extern "C" int rb_pipeline_push_masked(rb_pipeline *pl, int format, int on_device, const rb_frame *frames,
                                       const rb_frame *masks, const double *ts, int n, rb_nav *nav_out) {
    return push(pl, "push_masked", {nullptr, frames, format, on_device != 0, true, masks, ts, n}, nav_out);
}

// ---- asynchronous pushes (DESIGN.md §5) ----------------------------------------------------------------------------------
extern "C" int rb_pipeline_set_async(rb_pipeline *pl, int depth) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    if (depth < 0 || depth > 8) {
        snprintf(c->err, sizeof(c->err), "set_async: depth %d is outside 0..8", depth);
        return RB_ERR_ARG;
    }
    int r = set_begin(pl, "set_async");
    if (r) return r;
    async_free(pl);
    if (depth && (r = async_alloc(pl, depth))) async_free(pl);
    return r;
}

// one ticket of input that push_in has checked: the front on the front stream into workspace k % 2, the back on the tracker
// stream into output slot k % depth
static int enqueue_impl(rb_pipeline *pl, const PushIn &in, int64_t *ticket) {
    rb_ctx *c = pl->c;
    AsyncRing *ar = pl->ar;
    if (!ar || pl->imu) {
        snprintf(c->err, sizeof(c->err), "enqueue: %s", pl->imu ? "not available in IMU mode"
                                                                  : "asynchronous pushes are off (rb_pipeline_set_async)");
        return RB_ERR_ARG;
    }
    if (!ticket) return RB_ERR_ARG;
    if (pl->tk_next - pl->tk_retired >= ar->depth) {
        snprintf(c->err, sizeof(c->err), "enqueue: %d tickets are outstanding, the depth of rb_pipeline_set_async: wait first",
                 ar->depth);
        return RB_ERR_STATE;
    }
    RB_CUDA(cudaSetDevice(c->device));
    const int n = in.n, fmt = in.fmt;
    const long long k = pl->tk_next;
    OutSlot &s = ar->slot[k % ar->depth];
    const int par = (int)(k & 1);
    DogWS *ws = par ? &ar->ws1 : &pl->ws;
    int r;
    write_args(pl, s, in.ts, n);
    // front: once the back of ticket k - 2 (the last to read this workspace) is done, the frames into its staging (host
    // input) or its frame table (strided device input), then gray and scale space
    cudaStream_t fs = ar->front, main_stream = c->stream;
    RB_CUDA(cudaStreamWaitEvent(fs, ar->ev_free[par], 0));
    if (!in.on_device && (r = stage_host_frames(pl, in, 0, n, fs, ws))) return r;
    s.tbl[0].src = in.on_device ? (const void *)in.data : (const void *)ws->rgb;   // (strided: unused)
    RB_CUDA(cudaMemcpyAsync(ar->front_dev[par], &s.tbl[0], sizeof(SubBatchPtrs), cudaMemcpyHostToDevice, fs));
    if (in_strided(fmt)) {
        memcpy(s.frames, in.frames, sizeof(rb_frame) * n);
        RB_CUDA(cudaMemcpyAsync(ar->frames_dev[par], s.frames, sizeof(rb_frame) * n, cudaMemcpyHostToDevice, fs));
    }
    auto front = [&]() {
        c->stream = fs;
        const int e = enqueue_front(pl, ws, ar->front_dev[par], ar->frames_dev[par], fmt, n, false);
        c->stream = main_stream;
        return e;
    };
    const int fkey = afront_slot(pl, fmt, par, n);
    if (!pl->use_graph) {
        if ((r = front())) return r;
    } else if ((r = graph_launch(pl, ar->front_graphs, fs, fkey, 1, [&](int) { return fkey; }, [&](int) { return front(); }))) {
        return r;
    }
    RB_CUDA(cudaEventRecord(ar->ev_front[par], fs));
    // back: after the consumer's reads of the outputs this slot held (device mode) and this ticket's front, behind the back
    // of ticket k - 1 on the tracker stream
    if (pl->out_dev && pl->consumer != c->stream && (r = stream_wait(pl, pl->consumer, c->stream))) return r;
    RB_CUDA(cudaStreamWaitEvent(c->stream, ar->ev_front[par], 0));
    RB_CUDA(cudaMemcpyAsync(pl->fa_dev, s.fa, sizeof(FrameArgs) * n, cudaMemcpyHostToDevice, c->stream));
    // (the slot's sources: its previous ticket, their last reader, has been waited)
    const bool masked = fill_masks(pl, in.masks, n, s);
    if ((r = write_tables(pl, s, 1, nullptr, 0, n, masked))) return r;
    if (!pl->use_graph || s.first == 0) {
        if ((r = enqueue_back(pl, ws, n, s.first, masked))) return r;
    } else {   // (every workspace and ring phase of this size at once, as the synchronous batches)
        auto sib_key = [&](int i) { return aback_slot(pl, masked, i / RB_NMAPS, i % RB_NMAPS, n); };
        auto sib_body = [&](int i) {
            const int ph = i % RB_NMAPS;
            return enqueue_back(pl, i / RB_NMAPS ? &ar->ws1 : &pl->ws, n, ph == 0 ? RB_NMAPS : ph, masked);
        };
        if ((r = graph_launch(pl, ar->back_graphs, c->stream, sib_key(par * RB_NMAPS + (int)(s.first % RB_NMAPS)),
                              2 * RB_NMAPS, sib_key, sib_body)))
            return r;
    }
    RB_CUDA(cudaEventRecord(ar->ev_free[par], c->stream));
    RB_CUDA(cudaMemcpyAsync(s.nav, pl->nav_dev, sizeof(rb_nav) * n, cudaMemcpyDeviceToHost, c->stream));
    if (pl->odom.on)
        RB_CUDA(cudaMemcpyAsync(s.odom, pl->odom.dev, sizeof(rb_odometry) * n, cudaMemcpyDeviceToHost, c->stream));
    // the abort flags of this ticket alone: read, then cleared for the next ticket (a push clears them when it finds one set)
    for (int m = 0; m < RB_NMAPS; m++) {
        int *flag = &pl->maps[m]->ts_host.ctl->abort;
        RB_CUDA(cudaMemcpyAsync(&s.abort[m], flag, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        RB_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), c->stream));
    }
    RB_CUDA(cudaEventRecord(s.done, c->stream));
    pl->tk_next = k + 1;
    pl->n_pushed += n;
    pl->t_prev = in.ts[n - 1];
    pl->restored = false;
    pl->last_sub = 0;   // (the workspaces are the tickets': rb_pipeline_batch_plane has nothing to show)
    *ticket = k;
    return RB_OK;
}
// the asynchronous pushes' C entry points: push_in's checks, then enqueue_impl
static int enqueue(rb_pipeline *pl, const char *what, PushIn in, int64_t *ticket) {
    if (!pl) return RB_ERR_ARG;
    const int r = push_in(pl, what, in);
    return r ? r : enqueue_impl(pl, in, ticket);
}
extern "C" int rb_pipeline_enqueue(rb_pipeline *pl, int format, int on_device, const uint8_t *data, const double *ts, int n,
                                   int64_t *ticket) {
    return enqueue(pl, "enqueue", {data, nullptr, format, on_device != 0, false, nullptr, ts, n}, ticket);
}
extern "C" int rb_pipeline_enqueue_frames(rb_pipeline *pl, int format, int on_device, const rb_frame *frames, const double *ts,
                                          int n, int64_t *ticket) {
    return enqueue(pl, "enqueue_frames", {nullptr, frames, format, on_device != 0, false, nullptr, ts, n}, ticket);
}
extern "C" int rb_pipeline_masked_enqueue(rb_pipeline *pl, int format, int on_device, const rb_frame *frames,
                                          const rb_frame *masks, const double *ts, int n, int64_t *ticket) {
    return enqueue(pl, "masked_enqueue", {nullptr, frames, format, on_device != 0, true, masks, ts, n}, ticket);
}

extern "C" int rb_pipeline_wait(rb_pipeline *pl, int64_t ticket, rb_nav *nav_out) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    if (ticket < pl->tk_retired || ticket >= pl->tk_next) {
        snprintf(c->err, sizeof(c->err), "wait: ticket %lld is %s", (long long)ticket,
                 ticket >= pl->tk_next ? "not issued" : "already retired");
        return RB_ERR_ARG;
    }
    RB_CUDA(cudaSetDevice(c->device));
    AsyncRing *ar = pl->ar;
    int r = RB_OK;
    while (pl->tk_retired <= ticket) {   // (in ticket order)
        OutSlot &s = ar->slot[pl->tk_retired % ar->depth];
        RB_CUDA(cudaEventSynchronize(s.done));
        const int e = retire(pl, s);
        if (!r) r = e;
        pl->tk_retired++;
    }
    const OutSlot &s = ar->slot[ticket % ar->depth];
    show(pl, s, s.n);
    if (nav_out) memcpy(nav_out, s.nav, sizeof(rb_nav) * s.n);
    return r;
}
extern "C" int rb_pipeline_poll(rb_pipeline *pl, int64_t *newest_complete) {
    if (!pl || !newest_complete) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    long long t = pl->tk_retired - 1;   // (retired tickets are complete; the tracker stream completes them in order)
    while (t + 1 < pl->tk_next) {
        const cudaError_t e = cudaEventQuery(pl->ar->slot[(t + 1) % pl->ar->depth].done);
        if (e == cudaErrorNotReady) {
            if (cudaPeekAtLastError() == cudaErrorNotReady) cudaGetLastError();   // (not an error of a later launch)
            break;
        }
        RB_CUDA(e);
        t++;
    }
    *newest_complete = t;
    return RB_OK;
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
// the batch's planes stay in the workspace until the next push: the detector and the side streams only read img0 / dog, and
// the mirror and depth passes write buffers of their own
extern "C" int rb_pipeline_batch_plane(rb_pipeline *pl, int slot, int which, float *out) {
    if (!pl || !out) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    if (refuse_busy(pl, "batch_plane")) return RB_ERR_STATE;
    if (slot < 0 || slot >= pl->last_sub || (which != 0 && which != 2 && which != 5)) return RB_ERR_ARG;
    const float *src = (which == 0 ? pl->ws.img0 : which == 2 ? pl->ws.dog : pl->ws.gray) + (size_t)slot * c->NP;
    // the pitched plane without its padding columns: w * h floats (as rb_map_get_plane)
    RB_CUDA(cudaMemcpy2DAsync(out, (size_t)4 * c->w, src, (size_t)4 * c->pitch, (size_t)4 * c->w, c->h,
                              cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

extern "C" int rb_pipeline_bench_pass(rb_pipeline *pl, int pass_id, int nimg, int iters, float *ms_per_launch,
                                      double *bytes_per_launch) {
    rb_ctx *c = pl->c;
    if (nimg < 1 || nimg > pl->max_batch || iters < 1) return RB_ERR_ARG;
    if (refuse_busy(pl, "bench_pass")) return RB_ERR_STATE;
    int r;
    double bytes = 0;
    // passes 4-7: the gray pass on the workspace's frames, 4 and 5 from RGB24, 6 and 7 from mono8; 5 and 7 with the
    // undistortion fused in (needs rb_pipeline_set_undistort; the frames are read through sb_dev->src).  Algorithmic bytes:
    // 3N (RGB) / N (mono) in + 4N out per frame, + the 32N-byte map once per launch
    const bool gray = pass_id >= 4 && pass_id <= 7, mono = pass_id >= 6, und_pass = pass_id == 5 || pass_id == 7;
    if (und_pass && !pl->und) return RB_ERR_STATE;
    pl->last_sub = 0;   // (the passes overwrite the workspace's planes: rb_pipeline_batch_plane has nothing to show)
    auto one = [&]() -> int {
        if (!gray) return rb_dog_single_pass(c, &pl->ws, pass_id, nimg, &bytes);
        bytes = (mono ? 5.0 : 7.0) * c->N * nimg + (und_pass ? 32.0 * c->N : 0.0);
        return rb_gray_enqueue(c, &pl->ws, und_pass ? pl->und : nullptr, mono, und_pass ? &pl->sb_dev->src : nullptr, nullptr,
                               nimg);
    };
    if (und_pass) {
        pl->out.tbl[0].src = pl->ws.rgb;
        RB_CUDA(cudaMemcpyAsync(pl->sb_dev, pl->out.tbl, sizeof(SubBatchPtrs), cudaMemcpyHostToDevice, c->stream));
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

// ---- session checkpoints (rb_pipeline_save_state / rb_pipeline_load_state; blob layout: state.cuh, DESIGN.md §5) ----------
static int state_mode(const rb_pipeline *pl) {
    return !pl->imu ? RB_STATE_VISION : pl->imu->live ? RB_STATE_IMU_LIVE : RB_STATE_IMU_DATASET;
}
// live ring: the samples pushed and not released yet, s[read_inx + 1 ..] up to write_inx
static int live_pending(const rbimu::ImuBuffer &b) { return (b.write_inx - b.read_inx - 1 + 2 * b.size) % b.size; }
// host section: t_prev, odometry's rkp_last; in IMU mode then ImuSession, the ring's read position (dataset mode), t_last and
// the count of pending samples (live mode), and those samples
#define RB_STATE_HOST_VISION 16
static size_t state_host_bytes(int mode, long long n_pending) {
    if (mode == RB_STATE_VISION) return RB_STATE_HOST_VISION;
    return RB_STATE_HOST_VISION + state_align8(sizeof(ImuSession)) + 24 + sizeof(rbimu::ImuSample) * (size_t)n_pending;
}
static uint64_t imu_samples_checksum(const ImuFlow &f) {
    return state_checksum(f.samples.data(), sizeof(rbimu::ImuSample) * f.samples.size());
}

extern "C" int rb_pipeline_save_state(rb_pipeline *pl, void *buf, size_t cap, size_t *written) {
    if (!pl || !written || (cap && !buf)) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    if (refuse_busy(pl, "save_state")) return RB_ERR_STATE;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    rb_map *m = pl->n_pushed > 0 ? pl->maps[(pl->n_pushed - 1) % RB_NMAPS] : nullptr;
    MapState ms;
    memset(&ms, 0, sizeof(ms));
    int r;
    if (m && (r = rb_read_map_state(m, &ms))) return r;
    const int mode = state_mode(pl);
    const int pending = mode == RB_STATE_IMU_LIVE ? live_pending(pl->imu->buf) : 0;
    const size_t dev_b = state_dev_bytes(ms.kn), off_host = sizeof(StateHeader) + dev_b;
    const size_t total = off_host + state_host_bytes(mode, pending);
    *written = total;
    if (cap < total) {
        snprintf(c->err, sizeof(c->err), "save_state: the blob needs %zu bytes, the buffer holds %zu", total, cap);
        return RB_ERR_ARG;
    }
    // the device section: one kernel writes the live prefix straight into mapped pinned memory
    if ((r = grow_mapped(c, &pl->state_host, &pl->state_host_bytes, dev_b))) return r;
    if ((r = rb_state_pack_enqueue(c, m, pl->fs, pl->chain, pl->state_host))) return r;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    unsigned char *out = static_cast<unsigned char *>(buf);
    memcpy(out + sizeof(StateHeader), pl->state_host, dev_b);
    unsigned char *q = out + off_host;
    memset(q, 0, total - off_host);
    memcpy(q, &pl->t_prev, 8);
    memcpy(q + 8, &pl->odom.rkp_last, 8);
    StateHeader h;
    memset(&h, 0, sizeof(h));
    if (pl->imu) {
        const ImuFlow &f = *pl->imu;
        q += RB_STATE_HOST_VISION;
        memcpy(q, static_cast<const ImuSession *>(&f), sizeof(ImuSession));
        q += state_align8(sizeof(ImuSession));
        const int64_t read_inx = f.live ? -1 : f.buf.read_inx, npend = pending;
        const double t_last = f.live ? f.t_last : 0.0;
        memcpy(q, &read_inx, 8);
        memcpy(q + 8, &t_last, 8);
        memcpy(q + 16, &npend, 8);
        q += 24;
        for (int k = 0; k < pending; k++)
            memcpy(q + sizeof(rbimu::ImuSample) * k, &f.buf.s[(f.buf.read_inx + 1 + k) % f.buf.size], sizeof(rbimu::ImuSample));
        if (!f.live) {
            h.imu_count = f.samples.size();
            h.imu_checksum = imu_samples_checksum(f);
        }
    }
    memcpy(h.magic, RB_STATE_MAGIC, 8);
    h.version = RB_STATE_VERSION;
    h.header_bytes = sizeof(StateHeader);
    h.total_bytes = total;
    h.cam = c->cam;
    h.kl_capacity = c->kcap;
    h.mode = mode;
    h.sigma0 = c->sigma0;
    h.ksigma = c->ksigma;
    h.n_pushed = pl->n_pushed;
    h.kn = ms.kn;
    h.det_r = m ? m->det_r : 0;
    h.off_dev = sizeof(StateHeader);
    h.off_host = off_host;
    memcpy(out, &h, sizeof(h));
    h.checksum = state_checksum(out + RB_STATE_SUMMED, total - RB_STATE_SUMMED);
    memcpy(out, &h, sizeof(h));
    return RB_OK;
}

extern "C" int rb_pipeline_load_state(rb_pipeline *pl, const void *buf, size_t n) {
    if (!pl) return RB_ERR_ARG;
    rb_ctx *c = pl->c;
    RB_ENTER(c);
    if (refuse_busy(pl, "load_state")) return RB_ERR_STATE;
    int r = rb_state_check(buf, n, c->err, sizeof(c->err));
    if (r) return r;
    const unsigned char *b = static_cast<const unsigned char *>(buf);
    StateHeader h;
    memcpy(&h, b, sizeof(h));
#define REFUSE(...)                                         \
    do {                                                    \
        snprintf(c->err, sizeof(c->err), __VA_ARGS__);      \
        return RB_ERR_ARG;                                  \
    } while (0)
    // everything is checked before anything of the pipeline changes
    if (memcmp(&h.cam, &c->cam, sizeof(rb_camera)) != 0 || h.sigma0 != c->sigma0 || h.ksigma != c->ksigma ||
        h.kl_capacity != c->kcap)
        REFUSE("load_state: the blob's camera, Sigma0, KSigma or kl_capacity are not this pipeline's");
    const int mode = state_mode(pl);
    if (h.mode != mode) REFUSE("load_state: a blob of mode %d, the pipeline runs mode %d", h.mode, mode);
    if (h.det_r < 0 || h.det_r > RB_PLANE_FIT_MAX || h.off_host - h.off_dev != state_dev_bytes(h.kn))
        REFUSE("load_state: inconsistent device section");
    MapState ms;
    memcpy(&ms, b + h.off_dev + state_align8(sizeof(FrameState)) + state_align8(sizeof(DetChain)), sizeof(ms));
    if (ms.kn != h.kn) REFUSE("load_state: inconsistent keyline count");
    const size_t host_b = n - h.off_host;
    if (host_b < RB_STATE_HOST_VISION) REFUSE("load_state: truncated host section");
    const unsigned char *q = b + h.off_host;
    int64_t read_inx = -1, npend = 0;
    double t_last = 0;
    const unsigned char *imu_q = q + RB_STATE_HOST_VISION;
    if (pl->imu) {
        const ImuFlow &f = *pl->imu;
        if (host_b < state_host_bytes(mode, 0)) REFUSE("load_state: truncated IMU section");
        const unsigned char *t = imu_q + state_align8(sizeof(ImuSession));
        memcpy(&read_inx, t, 8);
        memcpy(&t_last, t + 8, 8);
        memcpy(&npend, t + 16, 8);
        if (!f.live) {
            if (h.imu_count != f.samples.size() || h.imu_checksum != imu_samples_checksum(f))
                REFUSE("load_state: the pipeline's IMU samples are not those of the blob's session");
            if (read_inx < 0 || read_inx >= f.buf.size || npend != 0) REFUSE("load_state: inconsistent IMU ring position");
        } else if (npend < 0 || npend > f.buf.size - 1) {
            REFUSE("load_state: %lld samples pending, the pipeline's ring holds %d", (long long)npend, f.buf.size - 1);
        }
    }
    if (host_b != state_host_bytes(mode, npend)) REFUSE("load_state: inconsistent host section");
#undef REFUSE
    // the device section through mapped pinned memory into the slot of the restored newest frame
    RB_CUDA(cudaStreamSynchronize(c->stream));
    const size_t dev_b = h.off_host - h.off_dev;
    if ((r = grow_mapped(c, &pl->state_host, &pl->state_host_bytes, dev_b))) return r;
    memcpy(pl->state_host, b + h.off_dev, dev_b);
    rb_map *m = h.n_pushed > 0 ? pl->maps[(h.n_pushed - 1) % RB_NMAPS] : nullptr;
    // the other ring maps as rb_pipeline_reset leaves them: each frame detects its own map before it reads one
    for (int k = 0; k < RB_NMAPS; k++) {
        RB_CUDA(cudaMemsetAsync(&pl->maps[k]->ts_host.ctl->abort, 0, sizeof(int), c->stream));
        if (pl->maps[k] != m) RB_CUDA(cudaMemsetAsync(&pl->maps[k]->st->frame_count, 0, sizeof(unsigned int), c->stream));
        pl->out.abort[k] = 0;
    }
    if ((r = rb_state_unpack_enqueue(c, m, pl->fs, pl->chain, pl->state_host, h.kn))) return r;
    RB_CUDA(cudaStreamSynchronize(c->stream));
    if (m) m->det_r = h.det_r;
    pl->n_pushed = h.n_pushed;
    pl->restored = true;
    memcpy(&pl->t_prev, q, 8);
    memcpy(&pl->odom.rkp_last, q + 8, 8);
    if (pl->imu) {
        ImuFlow &f = *pl->imu;
        memcpy(static_cast<ImuSession *>(&f), imu_q, sizeof(ImuSession));
        if (!f.live) {
            f.buf.read_inx = (int)read_inx;
        } else {   // the pending samples, oldest first, at the start of the ring
            const unsigned char *s = imu_q + state_align8(sizeof(ImuSession)) + 24;
            for (int k = 0; k < (int)npend; k++) memcpy(&f.samples[k], s + sizeof(rbimu::ImuSample) * k, sizeof(rbimu::ImuSample));
            f.buf.write_inx = (int)npend;
            f.buf.read_inx = f.buf.size - 1;
            f.buf.n = (int)npend;
            f.t_last = t_last;
        }
    }
    // the outputs of the last push are not this session's
    show(pl, pl->out, 0);
    pl->last_sub = 0;
    return RB_OK;
}

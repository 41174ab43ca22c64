// state.cuh -- the session state blob of rb_pipeline_save_state / rb_pipeline_load_state (layout: DESIGN.md §5).
// The header and the host-side checks are host code; k_state_pack / k_state_unpack (state.cu) move the device part.
#pragma once
#include "common.cuh"
#include "frame.cuh"

#define RB_STATE_MAGIC "RBB2STAT"
#define RB_STATE_VERSION 1u
// the checksum covers every byte from this offset to the end: everything but magic, version, the two sizes and itself
#define RB_STATE_SUMMED 32

// 128 bytes, little-endian, at the start of every blob
struct StateHeader {
    char magic[8];
    uint32_t version;
    uint32_t header_bytes;        // sizeof(StateHeader)
    uint64_t total_bytes;         // the whole blob
    uint64_t checksum;            // state_checksum of bytes [RB_STATE_SUMMED, total_bytes)
    rb_camera cam;                // (offset 32)
    int32_t kl_capacity;
    int32_t mode;                 // RB_STATE_VISION / RB_STATE_IMU_DATASET / RB_STATE_IMU_LIVE
    double sigma0, ksigma;
    int64_t n_pushed;
    int32_t kn;                   // keylines of the newest map (0 when n_pushed == 0)
    int32_t det_r;                // its plane-fit radius
    uint64_t imu_count;           // dataset mode: the samples of rb_pipeline_set_imu and their checksum; 0 otherwise
    uint64_t imu_checksum;
    uint64_t off_dev;             // device section: FrameState, DetChain, MapState, then the keyline arrays
    uint64_t off_host;            // host section: t_prev, rkp_last, then the IMU state in IMU mode
};
static_assert(sizeof(StateHeader) == 128, "StateHeader is 128 bytes");

// bytes of one keyline in the device section: 5 double, 6 float2, 1 float and 6 int arrays
#define RB_STATE_KL_BYTES (5 * 8 + 6 * 8 + 4 + 6 * 4)
__host__ __device__ inline size_t state_align8(size_t b) { return (b + 7) & ~(size_t)7; }
// the fixed part of the device section
__host__ __device__ inline size_t state_dev_fixed() {
    return state_align8(sizeof(FrameState)) + state_align8(sizeof(DetChain)) + state_align8(sizeof(MapState));
}
__host__ __device__ inline size_t state_dev_bytes(int kn) { return state_dev_fixed() + state_align8((size_t)RB_STATE_KL_BYTES * kn); }

// FNV-1a over 64-bit little-endian words (then the bytes of a tail shorter than a word): h = (h ^ word) * 0x100000001b3,
// from h = 0xcbf29ce484222325.  Word steps: eight times fewer dependent multiplies than the byte form.
static inline uint64_t state_checksum(const void *p, size_t n) {
    const unsigned char *b = static_cast<const unsigned char *>(p);
    uint64_t h = 0xcbf29ce484222325ull;
    size_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w;
        memcpy(&w, b + i, 8);
        h = (h ^ w) * 0x100000001b3ull;
    }
    for (; i < n; i++) h = (h ^ b[i]) * 0x100000001b3ull;
    return h;
}

// The header's own consistency (magic, version, sizes, section offsets, kn) and the checksum; RB_OK or RB_ERR_ARG with the
// reason in err.  Geometry and mode are the caller's to compare.
int rb_state_check(const void *buf, size_t n, char *err, size_t err_cap);

// map == nullptr: no map yet (n_pushed == 0), a zero MapState and no keylines.  dst: the device section, kn keylines, in
// memory the device can write (mapped pinned host memory)
int rb_state_pack_enqueue(rb_ctx *c, const rb_map *m, const FrameState *fs, const DetChain *ch, unsigned char *dst);
// the reverse, into map m (nullptr: FrameState and DetChain only), and m's keyline mask rebuilt from p_inx
int rb_state_unpack_enqueue(rb_ctx *c, rb_map *m, FrameState *fs, DetChain *ch, const unsigned char *src, int kn);

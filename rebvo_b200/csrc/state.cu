// state.cu -- the device side of the session state blob (rb_pipeline_save_state / rb_pipeline_load_state, pipeline.cu)
// and its host-only header check (rb_state_info).
//
// The blob holds the newest ring map only: the next frame reads maps f and f-1, and f+1 is detected fresh.  Of that map it
// holds the first kn entries of every KLSoA array a later frame or a stage-level read observes, and its MapState.  The
// keyline mask (4 bytes per pixel) is not stored: after a detect it is -1 everywhere but at the keylines' pixels, so the
// load rebuilds it from p_inx.  The minimiser's per-keyline records `pack` are rebuilt from m_m, c_p, u_m and n_m (as
// rb_map_load_keylines does); the distance field is not stored, the next frame builds its own map's field before it reads
// one.
#include "state.cuh"

// Keyline arrays of the device section, each kn entries long and in this order: rho, s_rho, rho0, s_rho0, n_m0 (double),
// m_m, u_m, c_p, p_m, p_m_0, m_m0 (float2), n_m (float), p_inx, m_id, m_id_f, m_num, p_id, n_id (int32)
struct KlSections {
    double *d[5];
    float2 *f2[6];
    float *n_m;
    int *i[6];
};
__device__ __forceinline__ KlSections kl_sections(unsigned char *base, int kn) {
    KlSections s;
    size_t o = 0;
    for (int k = 0; k < 5; k++, o += 8 * (size_t)kn) s.d[k] = reinterpret_cast<double *>(base + o);
    for (int k = 0; k < 6; k++, o += 8 * (size_t)kn) s.f2[k] = reinterpret_cast<float2 *>(base + o);
    s.n_m = reinterpret_cast<float *>(base + o);
    o += 4 * (size_t)kn;
    for (int k = 0; k < 6; k++, o += 4 * (size_t)kn) s.i[k] = reinterpret_cast<int *>(base + o);
    return s;
}

// n8 8-byte words (src == nullptr: zeros)
__device__ __forceinline__ void copy_words(unsigned long long *dst, const unsigned long long *src, int n8) {
    for (int k = threadIdx.x; k < n8; k += blockDim.x) dst[k] = src ? src[k] : 0ull;
}

// map -> blob.  kn is read here, on the device: only the live prefix of every array is written (straight into mapped
// pinned host memory), however large the capacity.
__global__ void __launch_bounds__(256) k_state_pack(KLSoA kl, const MapState *st, const FrameState *fs, const DetChain *ch,
                                                    unsigned char *dst) {
    const int kn = st ? st->kn : 0;
    unsigned char *p = dst;
    if (blockIdx.x == 0) {
        copy_words(reinterpret_cast<unsigned long long *>(p), reinterpret_cast<const unsigned long long *>(fs),
                   (int)(sizeof(FrameState) / 8));
        p += state_align8(sizeof(FrameState));
        copy_words(reinterpret_cast<unsigned long long *>(p), reinterpret_cast<const unsigned long long *>(ch),
                   (int)(sizeof(DetChain) / 8));
        p += state_align8(sizeof(DetChain));
        copy_words(reinterpret_cast<unsigned long long *>(p), reinterpret_cast<const unsigned long long *>(st),
                   (int)(sizeof(MapState) / 8));
    }
    const KlSections s = kl_sections(dst + state_dev_fixed(), kn);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kn; i += gridDim.x * blockDim.x) {
        s.d[0][i] = kl.rho[i];
        s.d[1][i] = kl.s_rho[i];
        s.d[2][i] = kl.rho0[i];
        s.d[3][i] = kl.s_rho0[i];
        s.d[4][i] = kl.n_m0[i];
        s.f2[0][i] = kl.m_m[i];
        s.f2[1][i] = kl.u_m[i];
        s.f2[2][i] = kl.c_p[i];
        s.f2[3][i] = kl.p_m[i];
        s.f2[4][i] = kl.p_m_0[i];
        s.f2[5][i] = kl.m_m0[i];
        s.n_m[i] = kl.n_m[i];
        s.i[0][i] = kl.p_inx[i];
        s.i[1][i] = kl.m_id[i];
        s.i[2][i] = kl.m_id_f[i];
        s.i[3][i] = kl.m_num[i];
        s.i[4][i] = kl.p_id[i];
        s.i[5][i] = kl.n_id[i];
    }
}

// blob -> map (st == nullptr: FrameState and DetChain only).  The mask was filled with -1 before: each keyline marks its
// pixel, as the detector left it (k_detect_b).  A p_inx outside the image marks nothing.
__global__ void __launch_bounds__(256) k_state_unpack(KLSoA kl, MapState *st, FrameState *fs, DetChain *ch, int *mask,
                                                      int npix, const unsigned char *src, int kn) {
    const unsigned char *p = src;
    if (blockIdx.x == 0) {
        copy_words(reinterpret_cast<unsigned long long *>(fs), reinterpret_cast<const unsigned long long *>(p),
                   (int)(sizeof(FrameState) / 8));
        p += state_align8(sizeof(FrameState));
        copy_words(reinterpret_cast<unsigned long long *>(ch), reinterpret_cast<const unsigned long long *>(p),
                   (int)(sizeof(DetChain) / 8));
        p += state_align8(sizeof(DetChain));
        if (st)
            copy_words(reinterpret_cast<unsigned long long *>(st), reinterpret_cast<const unsigned long long *>(p),
                       (int)(sizeof(MapState) / 8));
    }
    if (!st) return;
    const KlSections s = kl_sections(const_cast<unsigned char *>(src) + state_dev_fixed(), kn);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kn; i += gridDim.x * blockDim.x) {
        kl.rho[i] = s.d[0][i];
        kl.s_rho[i] = s.d[1][i];
        kl.rho0[i] = s.d[2][i];
        kl.s_rho0[i] = s.d[3][i];
        kl.n_m0[i] = s.d[4][i];
        const float2 m = s.f2[0][i], u = s.f2[1][i], cp = s.f2[2][i];
        kl.m_m[i] = m;
        kl.u_m[i] = u;
        kl.c_p[i] = cp;
        kl.p_m[i] = s.f2[3][i];
        kl.p_m_0[i] = s.f2[4][i];
        kl.m_m0[i] = s.f2[5][i];
        const float n_m = s.n_m[i];
        kl.n_m[i] = n_m;
        const int pix = s.i[0][i];
        kl.p_inx[i] = pix;
        kl.m_id[i] = s.i[1][i];
        kl.m_id_f[i] = s.i[2][i];
        kl.m_num[i] = s.i[3][i];
        kl.p_id[i] = s.i[4][i];
        kl.n_id[i] = s.i[5][i];
        kl.pack[2 * i] = make_float4(m.x, m.y, cp.x, cp.y);
        kl.pack[2 * i + 1] = make_float4(u.x, u.y, n_m, 0.f);
        if ((unsigned)pix < (unsigned)npix) mask[pix] = i;
    }
}

static int state_grid(const rb_ctx *c) {
    const int g = rb_div_up(c->kcap, 256), cap = 2 * (c->sm_count > 0 ? c->sm_count : 1);
    return g < cap ? g : cap;
}

int rb_state_pack_enqueue(rb_ctx *c, const rb_map *m, const FrameState *fs, const DetChain *ch, unsigned char *dst) {
    KLSoA kl;
    memset(&kl, 0, sizeof(kl));
    if (m) kl = m->kl;
    k_state_pack<<<state_grid(c), 256, 0, c->stream>>>(kl, m ? m->st : nullptr, fs, ch, dst);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

int rb_state_unpack_enqueue(rb_ctx *c, rb_map *m, FrameState *fs, DetChain *ch, const unsigned char *src, int kn) {
    KLSoA kl;
    memset(&kl, 0, sizeof(kl));
    if (m) {
        kl = m->kl;
        RB_CUDA(cudaMemsetAsync(m->mask, 0xff, sizeof(int) * (size_t)c->N, c->stream));   // img_mask_kl.Reset(-1)
    }
    k_state_unpack<<<state_grid(c), 256, 0, c->stream>>>(kl, m ? m->st : nullptr, fs, ch, m ? m->mask : nullptr, c->N, src,
                                                         m ? kn : 0);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// ---- host: the header ----------------------------------------------------------------------------------------------------
int rb_state_check(const void *buf, size_t n, char *err, size_t err_cap) {
#define REFUSE(...)                                          \
    do {                                                     \
        if (err && err_cap) snprintf(err, err_cap, __VA_ARGS__); \
        return RB_ERR_ARG;                                   \
    } while (0)
    if (!buf || n < sizeof(StateHeader)) REFUSE("state blob: %zu bytes, shorter than its %zu-byte header", n, sizeof(StateHeader));
    StateHeader h;
    memcpy(&h, buf, sizeof(h));
    if (memcmp(h.magic, RB_STATE_MAGIC, 8) != 0) REFUSE("state blob: bad magic");
    if (h.version != RB_STATE_VERSION)
        REFUSE("state blob: version %u, this library reads version %u", h.version, RB_STATE_VERSION);
    if (h.header_bytes != sizeof(StateHeader)) REFUSE("state blob: header of %u bytes", h.header_bytes);
    if (h.total_bytes != n) REFUSE("state blob: %zu bytes given, the header says %llu", n, (unsigned long long)h.total_bytes);
    const unsigned char *b = static_cast<const unsigned char *>(buf);
    if (state_checksum(b + RB_STATE_SUMMED, n - RB_STATE_SUMMED) != h.checksum) REFUSE("state blob: checksum mismatch");
    if (h.mode < RB_STATE_VISION || h.mode > RB_STATE_IMU_LIVE) REFUSE("state blob: mode %d", h.mode);
    if (h.kl_capacity < 1 || h.kl_capacity > RB_KCAP_MAX || h.kn < 0 || h.kn > h.kl_capacity || h.n_pushed < 0 ||
        (h.n_pushed == 0 && h.kn != 0))
        REFUSE("state blob: inconsistent counts (kn %d, capacity %d, frames %lld)", h.kn, h.kl_capacity, (long long)h.n_pushed);
    if (h.off_dev != sizeof(StateHeader) || h.off_host < h.off_dev || h.off_host > n ||
        h.off_host - h.off_dev < (uint64_t)RB_STATE_KL_BYTES * (uint64_t)h.kn || (h.off_dev | h.off_host) % 8)
        REFUSE("state blob: inconsistent section offsets");
    return RB_OK;
#undef REFUSE
}

extern "C" int rb_state_info(const void *buf, size_t n, struct rb_state_info *out) {
    if (!out) return RB_ERR_ARG;
    int r = rb_state_check(buf, n, nullptr, 0);
    if (r) return r;
    StateHeader h;
    memcpy(&h, buf, sizeof(h));
    memset(out, 0, sizeof(*out));
    out->version = h.version;
    out->mode = h.mode;
    out->bytes = h.total_bytes;
    out->cam = h.cam;
    out->Sigma0 = h.sigma0;
    out->KSigma = h.ksigma;
    out->kl_capacity = h.kl_capacity;
    out->kn = h.kn;
    out->n_pushed = h.n_pushed;
    return RB_OK;
}

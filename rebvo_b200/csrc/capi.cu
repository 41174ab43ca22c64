// capi.cu -- the C ABI of librebvo_b200 (include/rebvo_b200.h): context / edge-map lifetime, uploads,
// scalar read-back and the AoS <-> SoA keyline conversion for host consumers.
#include <math.h>
#include <stdlib.h>
#include <new>

#include "common.cuh"
#include "tracker.cuh"

int rb_detect_upload_pinv(rb_ctx *c, const double *tab);

// ---- host-side set-up math -----------------------------------------------------------------------
// iigauss::iigauss (src/mtracklib/iigauss.cpp:43-81): Kovesi box sizes for a target sigma
static void box_plan_one(double sigma, int box_n, int *box_d, double *sigma_r) {
    const double wideal = sqrt(12 * sigma * sigma / box_n + 1);
    int wl = (int)wideal;
    const int tmp = wl / 2;
    if (tmp * 2 == wl) wl--;
    const int m = (int)round((3 * box_n + 4 * box_n * wl + box_n * wl * wl - 12 * sigma * sigma) / (4 + 4 * wl));
    int i = 0;
    for (; i < m && i < box_n; i++) box_d[i] = wl;
    for (; i < box_n; i++) box_d[i] = wl + 2;
    *sigma_r = sqrt((m * wl * wl + (box_n - m) * (wl + 2.0) * (wl + 2.0) - box_n) / 12.0);
}

// plane-fit pseudo inverse PInv = Matrix3x3Inv(Phi^T Phi) * Phi^T (edge_finder.cpp:83-100,
// include/UtilLib/toon_util.h:32-41) of half-width ws: out[r * n + k], n = (2 ws + 1)^2
static void plane_fit_pinv(int ws, double *out) {
    const int n = (2 * ws + 1) * (2 * ws + 1);
    double Phi[(2 * RB_PLANE_FIT_MAX + 1) * (2 * RB_PLANE_FIT_MAX + 1)][3];
    int k = 0;
    for (int i = -ws; i <= ws; i++)
        for (int j = -ws; j <= ws; j++, k++) {
            Phi[k][0] = j;
            Phi[k][1] = i;
            Phi[k][2] = 1;
        }
    double A[3][3];
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) {
            double s = 0;
            for (k = 0; k < n; k++) s += Phi[k][r] * Phi[k][c];
            A[r][c] = s;
        }
    double B[3][3];
    B[0][0] = A[2][2] * A[1][1] - A[2][1] * A[1][2];
    B[0][1] = -(A[2][2] * A[0][1] - A[2][1] * A[0][2]);
    B[0][2] = A[1][2] * A[0][1] - A[1][1] * A[0][2];
    B[1][0] = -(A[2][2] * A[1][0] - A[2][0] * A[1][2]);
    B[1][1] = A[2][2] * A[0][0] - A[2][0] * A[0][2];
    B[1][2] = -(A[1][2] * A[0][0] - A[1][0] * A[0][2]);
    B[2][0] = A[2][1] * A[1][0] - A[2][0] * A[1][1];
    B[2][1] = -(A[2][1] * A[0][0] - A[2][0] * A[0][1]);
    B[2][2] = A[1][1] * A[0][0] - A[1][0] * A[0][1];
    const double det = A[0][0] * (A[1][1] * A[2][2] - A[1][2] * A[2][1]) -
                       A[0][1] * (A[1][0] * A[2][2] - A[1][2] * A[2][0]) +
                       A[0][2] * (A[1][0] * A[2][1] - A[1][1] * A[2][0]);
    for (int r = 0; r < 3; r++)
        for (int c = 0; c < 3; c++) B[r][c] = B[r][c] / det;
    for (int r = 0; r < 3; r++)
        for (k = 0; k < n; k++) {
            double s = 0;
            for (int c = 0; c < 3; c++) s += B[r][c] * Phi[k][c];
            out[r * n + k] = s;
        }
}

// the pseudo inverses of every supported radius, packed at rb_pinv_offset(r); they depend on the radius only, so all
// contexts upload the same table
static const double *plane_fit_tables() {
    static double tab[RB_PINV_DOUBLES];
    static std::once_flag once;
    std::call_once(once, [] {
        for (int r = 1; r <= RB_PLANE_FIT_MAX; r++) plane_fit_pinv(r, tab + rb_pinv_offset(r));
    });
    return tab;
}

// ---- AoS <-> SoA ----------------------------------------------------------------------------------
__device__ __forceinline__ void pack_one(const KLSoA &kl, int i, rb_keyline *dst) {
    rb_keyline k;
    k.p_inx = kl.p_inx[i];
    float2 v = kl.m_m[i];
    k.m_m[0] = v.x; k.m_m[1] = v.y;
    v = kl.u_m[i];
    k.u_m[0] = v.x; k.u_m[1] = v.y;
    k.n_m = kl.n_m[i];
    k.score = 0.f;
    v = kl.c_p[i];
    k.c_p[0] = v.x; k.c_p[1] = v.y;
    k._pad0 = 0;
    k.rho = kl.rho[i];
    k.s_rho = kl.s_rho[i];
    k.rho_nr = RB_RHO_INIT;      // never updated by the reference (complex_regularization=false)
    k.s_rho_nr = RB_RHO_MAX;
    k.rho0 = kl.rho0[i];
    k.s_rho0 = kl.s_rho0[i];
    v = kl.p_m[i];
    k.p_m[0] = v.x; k.p_m[1] = v.y;
    v = kl.p_m_0[i];
    k.p_m_0[0] = v.x; k.p_m_0[1] = v.y;
    k.m_id = kl.m_id[i];
    k.m_id_f = kl.m_id_f[i];
    k.m_id_kf = -1;
    k.m_num = kl.m_num[i];
    v = kl.m_m0[i];
    k.m_m0[0] = v.x; k.m_m0[1] = v.y;
    k.n_m0 = kl.n_m0[i];
    k.p_id = kl.p_id[i];
    k.n_id = kl.n_id[i];
    k.net_id = -1;
    k.stereo_m_id = -1;
    k.stereo_rho = RB_RHO_INIT;
    k.stereo_s_rho = RB_RHO_MAX;
    *dst = k;
}
__global__ void k_pack_aos(KLSoA kl, const MapState *st, rb_keyline *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st->kn) return;
    pack_one(kl, i, out + i);
}

// pipeline mirror: the destination comes through a device pointer, so that one captured graph serves every staging buffer.
// The records of a block are assembled in shared memory and leave as contiguous 8-byte stores (a thread writing its own
// 168-byte record straight to global memory scatters 42 four-byte stores per lane).
__global__ void __launch_bounds__(128) k_pack_aos_ind(KLSoA kl, const MapState *st, unsigned char *const *base, size_t offset) {
    __shared__ __align__(16) rb_keyline rec[128];
    const int kn = st->kn;
    const int i0 = blockIdx.x * 128;
    if (i0 >= kn) return;
    const int i = i0 + threadIdx.x;
    if (i < kn) pack_one(kl, i, &rec[threadIdx.x]);
    __syncthreads();
    const int nrec = kn - i0 < 128 ? kn - i0 : 128;
    const int n8 = nrec * (int)(sizeof(rb_keyline) / 8);   // 168 = 21 x 8
    uint2 *dst = reinterpret_cast<uint2 *>(*base + offset) + (size_t)i0 * (sizeof(rb_keyline) / 8);
    const uint2 *src = reinterpret_cast<const uint2 *>(rec);
    for (int k = threadIdx.x; k < n8; k += 128) dst[k] = src[k];
}
int rb_map_pack_aos_enqueue(rb_ctx *c, rb_map *m, unsigned char *const *base, size_t offset) {
    k_pack_aos_ind<<<rb_div_up(c->kcap, 128), 128, 0, c->stream>>>(m->kl, m->st, base, offset);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

__global__ void k_unpack_aos(KLSoA kl, MapState *st, const rb_keyline *in, int kn) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) st->kn = kn;
    if (i >= kn) return;
    const rb_keyline k = in[i];
    kl.p_inx[i] = k.p_inx;
    kl.m_m[i] = make_float2(k.m_m[0], k.m_m[1]);
    kl.u_m[i] = make_float2(k.u_m[0], k.u_m[1]);
    kl.n_m[i] = k.n_m;
    kl.c_p[i] = make_float2(k.c_p[0], k.c_p[1]);
    kl.rho[i] = k.rho;
    kl.s_rho[i] = k.s_rho;
    kl.rho0[i] = k.rho0;
    kl.s_rho0[i] = k.s_rho0;
    kl.p_m[i] = make_float2(k.p_m[0], k.p_m[1]);
    kl.p_m_0[i] = make_float2(k.p_m_0[0], k.p_m_0[1]);
    kl.m_id[i] = k.m_id;
    kl.m_id_f[i] = k.m_id_f;
    kl.m_num[i] = k.m_num;
    kl.m_m0[i] = make_float2(k.m_m0[0], k.m_m0[1]);
    kl.n_m0[i] = k.n_m0;
    kl.p_id[i] = k.p_id;
    kl.n_id[i] = k.n_id;
    kl.pack[2 * i] = make_float4(k.m_m[0], k.m_m[1], k.c_p[0], k.c_p[1]);
    kl.pack[2 * i + 1] = make_float4(k.u_m[0], k.u_m[1], k.n_m, 0.f);
}

__global__ void k_fill_int(int *p, int v, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

// ---- context --------------------------------------------------------------------------------------
extern "C" int rb_ctx_create(rb_ctx **out, int device, const rb_camera *cam, double sigma0, double ksigma,
                             int kl_capacity) {
    if (!out || !cam) return RB_ERR_ARG;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device >= ndev) return RB_ERR_NO_DEVICE;
    if (cam->w < 32 || cam->h < 32 || kl_capacity < 1 || kl_capacity > RB_KCAP_MAX) return RB_ERR_ARG;
    rb_ctx *c = new (std::nothrow) rb_ctx;
    if (!c) return RB_ERR_ARG;
    memset(c, 0, sizeof(*c));
    c->mtx = new (std::nothrow) std::recursive_mutex;
    if (!c->mtx) {
        delete c;
        return RB_ERR_ARG;
    }
    c->device = device;
    c->cam = *cam;
    c->w = cam->w;
    c->h = cam->h;
    c->N = cam->w * cam->h;
    c->pitch = (cam->w + 3) & ~3;
    c->NP = c->pitch * cam->h;
    c->ppx = cam->ppx;
    c->ppy = cam->ppy;
    c->zfm = (double)((cam->zfx + cam->zfy) / 2);  // cam_model: zfm((focal_dist.x+focal_dist.y)/2) in float
    c->sigma0 = sigma0;
    c->ksigma = ksigma;
    c->kcap = kl_capacity;
    {
        const char *pd = getenv("REBVO_B200_PDL");
        c->pdl = !(pd && atoi(pd) == 0);
    }
    // sspace::sspace (sspace.cpp:36-46): filter1 sigma = filter0.sigma_r * k_sigma
    box_plan_one(sigma0, 3, c->plan.d[0], &c->plan.sigma_r[0]);
    box_plan_one(c->plan.sigma_r[0] * ksigma, 3, c->plan.d[1], &c->plan.sigma_r[1]);
    int r = RB_OK;
    auto fail = [&](int code) {
        *out = c;  // keep the context so that the caller can read rb_last_error()
        return code;
    };
#define CK(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e__ = (call);                                                                 \
        if (e__ != cudaSuccess) {                                                                 \
            snprintf(c->err, sizeof(c->err), "%s:%d %s: %s", __FILE__, __LINE__, #call,           \
                     cudaGetErrorString(e__));                                                    \
            return fail(RB_ERR_CUDA);                                                             \
        }                                                                                         \
    } while (0)
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    if ((r = rb_minimizer_cluster_setup(c))) return fail(r);
    {   // the context's stream carries the latency-critical tracker chain: highest priority, so that its kernels get SM slots
        // before the queued blocks of the detector / mirror streams (env REBVO_B200_PRIO=0: default priority)
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        const char *pe = getenv("REBVO_B200_PRIO");
        CK(cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, (pe && atoi(pe) == 0) ? lo : hi));
    }
    c->nseg = c->h * rb_div_up(c->w, 32);
    CK(cudaMalloc(&c->seg_cnt, sizeof(int) * c->nseg));
    CK(cudaMalloc(&c->cand, sizeof(float4) * (size_t)c->N));
    c->red_cap = 1024;
    CK(cudaMalloc(&c->red_part, sizeof(double) * 32 * c->red_cap));
    CK(cudaMalloc(&c->ticket, sizeof(unsigned int) * 16));
    CK(cudaMemset(c->ticket, 0, sizeof(unsigned int) * 16));
    CK(cudaMallocHost(&c->pinned, 1 << 16));
    CK(cudaMalloc(&c->dev_small, 1 << 16));
    CK(cudaMemset(c->dev_small, 0, 1 << 16));
    {
        const int mm_init[2] = {-1, 0x7f7fffff};   // reEstimateThresh scratch: max bits, min bits (re-armed by k_nm_histo)
        CK(cudaMemcpy((char *)c->dev_small + RB_DS_REEST, mm_init, sizeof(mm_init), cudaMemcpyHostToDevice));
    }
    if ((r = rb_detect_upload_pinv(c, plane_fit_tables()))) return fail(r);
    if ((r = rb_dog_make_tables(c))) return fail(r);
#undef CK
    *out = c;
    return RB_OK;
}

extern "C" void rb_ctx_destroy(rb_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) {
        cudaStreamSynchronize(c->stream);
        cudaStreamDestroy(c->stream);
    }
    cudaFree(c->seg_cnt);
    cudaFree(c->cand);
    cudaFree(c->red_part);
    cudaFree(c->ticket);
    cudaFree(c->dev_small);
    cudaFree(c->boxtab);
    cudaFree(c->depth_ws);
    if (c->pinned) cudaFreeHost(c->pinned);
    delete c->mtx;
    delete c;
}

extern "C" const char *rb_last_error(const rb_ctx *c) { return c ? c->err : "null context"; }

extern "C" int rb_ctx_sync(rb_ctx *c) {
    if (!c) return RB_ERR_ARG;
    RB_ENTER(c);
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

extern "C" int rb_ctx_box_plan(const rb_ctx *c, int *out_d, double *out_sigma_r) {
    for (int f = 0; f < 2; f++) {
        for (int i = 0; i < 3; i++) out_d[f * 3 + i] = c->plan.d[f][i];
        out_sigma_r[f] = c->plan.sigma_r[f];
    }
    return RB_OK;
}

extern "C" int64_t rb_ctx_launch_count(const rb_ctx *c) { return c->launches; }
extern "C" int rb_ctx_minimizer_clusters(const rb_ctx *c) { return c->min_cluster_g; }

// ---- map ------------------------------------------------------------------------------------------
int rb_map_alloc(rb_ctx *c, rb_map **out, bool with_ws) {
    rb_map *m = new (std::nothrow) rb_map;
    if (!m) return RB_ERR_ARG;
    memset(m, 0, sizeof(*m));
    m->c = c;
    *out = m;
    const size_t N = c->N, K = c->kcap + 32;
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaMalloc(&m->mask, sizeof(int) * N));
    RB_CUDA(cudaMalloc(&m->field, sizeof(unsigned long long) * N));
    RB_CUDA(cudaMemsetAsync(m->field, 0xff, sizeof(unsigned long long) * N, c->stream));
    k_fill_int<<<(unsigned)((N + 255) / 256), 256, 0, c->stream>>>(m->mask, -1, N);  // img_mask_kl.Reset(-1)
    RB_LAUNCH_CHECK();
    KLSoA &k = m->kl;
    RB_CUDA(cudaMalloc(&k.p_inx, sizeof(int) * K));
    RB_CUDA(cudaMalloc(&k.m_m, sizeof(float2) * K));
    RB_CUDA(cudaMalloc(&k.u_m, sizeof(float2) * K));
    RB_CUDA(cudaMalloc(&k.c_p, sizeof(float2) * K));
    RB_CUDA(cudaMalloc(&k.p_m, sizeof(float2) * K));
    RB_CUDA(cudaMalloc(&k.p_m_0, sizeof(float2) * K));
    RB_CUDA(cudaMalloc(&k.m_m0, sizeof(float2) * K));
    RB_CUDA(cudaMalloc(&k.n_m, sizeof(float) * K));
    RB_CUDA(cudaMalloc(&k.rho, sizeof(double) * K));
    RB_CUDA(cudaMalloc(&k.s_rho, sizeof(double) * K));
    RB_CUDA(cudaMalloc(&k.rho0, sizeof(double) * K));
    RB_CUDA(cudaMalloc(&k.s_rho0, sizeof(double) * K));
    RB_CUDA(cudaMalloc(&k.n_m0, sizeof(double) * K));
    RB_CUDA(cudaMalloc(&k.m_id, sizeof(int) * K));
    RB_CUDA(cudaMalloc(&k.m_id_f, sizeof(int) * K));
    RB_CUDA(cudaMalloc(&k.m_num, sizeof(int) * K));
    RB_CUDA(cudaMalloc(&k.p_id, sizeof(int) * K));
    RB_CUDA(cudaMalloc(&k.n_id, sizeof(int) * K));
    RB_CUDA(cudaMalloc(&k.pack, sizeof(float4) * 2 * K));
    RB_CUDA(cudaMalloc(&m->st, sizeof(MapState)));
    RB_CUDA(cudaMemsetAsync(m->st, 0, sizeof(MapState), c->stream));
    for (int i = 0; i < 3; i++) {
        RB_CUDA(cudaMalloc(&m->res[i], sizeof(double) * K));
        RB_CUDA(cudaMemsetAsync(m->res[i], 0, sizeof(double) * K, c->stream));
        RB_CUDA(cudaMalloc(&m->carry_flag[i], K));
        RB_CUDA(cudaMemsetAsync(m->carry_flag[i], 0, K, c->stream));
    }
    int r = rb_track_state_alloc(c, m);
    if (r) return r;
    if (with_ws) {
        if ((r = rb_dogws_alloc(c, &m->ws, 1))) return r;
        m->owns_ws = true;
        m->img0 = m->ws.img0;
        m->dog = m->ws.dog;
    }
    return RB_OK;
}

extern "C" int rb_map_create(rb_ctx *c, rb_map **out) {
    if (!c) return RB_ERR_ARG;
    RB_ENTER(c);
    if (!c || !out) return RB_ERR_ARG;
    return rb_map_alloc(c, out, true);
}

// edge_finder(const edge_finder&) + global_tracker(const global_tracker&) (edge_finder.cpp:42-52,
// global_tracker.cpp:42-47): a new ring-slot-like object holding a copy of the keylines, the id mask, the match field
// (+ its search radius) and FrameCount.  Device-to-device copies on the context's stream; scale-space planes and the
// minimiser scratch are not part of the reference's copy either.
extern "C" void rb_map_destroy(rb_map *m);
extern "C" int rb_map_clone(const rb_map *src, rb_map **out) {
    if (!src) return RB_ERR_ARG;
    RB_ENTER(src->c);
    if (!src || !out) return RB_ERR_ARG;
    rb_ctx *c = src->c;
    int r = rb_map_alloc(c, out, false);
    if (r) return r;
    rb_map *m = *out;
    const size_t N = c->N, K = c->kcap + 32;
    const KLSoA &a = src->kl;
    KLSoA &b = m->kl;
    // on a failed copy the half-initialised map is destroyed here and *out is nulled
#define CP(dst, srcp, bytes)                                                                                 \
    do {                                                                                                     \
        cudaError_t e__ = cudaMemcpyAsync(dst, srcp, bytes, cudaMemcpyDeviceToDevice, c->stream);            \
        if (e__ != cudaSuccess) {                                                                            \
            snprintf(c->err, sizeof(c->err), "rb_map_clone: %s", cudaGetErrorString(e__));                   \
            rb_map_destroy(m);                                                                               \
            *out = nullptr;                                                                                  \
            return RB_ERR_CUDA;                                                                              \
        }                                                                                                    \
    } while (0)
    CP(m->mask, src->mask, sizeof(int) * N);
    CP(m->field, src->field, sizeof(unsigned long long) * N);
    CP(b.p_inx, a.p_inx, sizeof(int) * K);
    CP(b.m_m, a.m_m, sizeof(float2) * K);
    CP(b.u_m, a.u_m, sizeof(float2) * K);
    CP(b.c_p, a.c_p, sizeof(float2) * K);
    CP(b.p_m, a.p_m, sizeof(float2) * K);
    CP(b.p_m_0, a.p_m_0, sizeof(float2) * K);
    CP(b.m_m0, a.m_m0, sizeof(float2) * K);
    CP(b.n_m, a.n_m, sizeof(float) * K);
    CP(b.rho, a.rho, sizeof(double) * K);
    CP(b.s_rho, a.s_rho, sizeof(double) * K);
    CP(b.rho0, a.rho0, sizeof(double) * K);
    CP(b.s_rho0, a.s_rho0, sizeof(double) * K);
    CP(b.n_m0, a.n_m0, sizeof(double) * K);
    CP(b.m_id, a.m_id, sizeof(int) * K);
    CP(b.m_id_f, a.m_id_f, sizeof(int) * K);
    CP(b.m_num, a.m_num, sizeof(int) * K);
    CP(b.p_id, a.p_id, sizeof(int) * K);
    CP(b.n_id, a.n_id, sizeof(int) * K);
    CP(b.pack, a.pack, sizeof(float4) * 2 * K);
    CP(m->st, src->st, sizeof(MapState));
#undef CP
    m->field_radius = src->field_radius;
    m->det_r = src->det_r;
    if (cudaStreamSynchronize(c->stream) != cudaSuccess) {
        snprintf(c->err, sizeof(c->err), "rb_map_clone: copy failed");
        rb_map_destroy(m);
        *out = nullptr;
        return RB_ERR_CUDA;
    }
    return RB_OK;
}

extern "C" void rb_map_destroy(rb_map *m) {
    if (!m) return;
    rb_ctx *c = m->c;
    RB_ENTER(c);
    cudaStreamSynchronize(c->stream);
    if (m->owns_ws) rb_dogws_free(&m->ws);
    cudaFree(m->mask);
    cudaFree(m->field);
    KLSoA &k = m->kl;
    void *ptrs[] = {k.p_inx, k.m_m, k.u_m, k.c_p, k.p_m, k.p_m_0, k.m_m0, k.n_m, k.rho, k.s_rho, k.rho0,
                    k.s_rho0, k.n_m0, k.m_id, k.m_id_f, k.m_num, k.p_id, k.n_id, k.pack, m->st};
    for (void *p : ptrs) cudaFree(p);
    for (int i = 0; i < 3; i++) {
        cudaFree(m->res[i]);
        cudaFree(m->carry_flag[i]);
    }
    rb_track_state_free(m);
    delete m;
}

extern "C" int rb_map_upload_rgb(rb_map *m, const uint8_t *rgb) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    if (!m->owns_ws) return RB_ERR_STATE;
    RB_CUDA(cudaMemcpyAsync(m->ws.rgb, rgb, (size_t)3 * c->N, cudaMemcpyHostToDevice, c->stream));
    return rb_gray_enqueue(c, &m->ws, nullptr, false, nullptr, nullptr, 1);
}

extern "C" int rb_map_upload_mono(rb_map *m, const uint8_t *mono) {
    if (!m || !mono) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    if (!m->owns_ws) return RB_ERR_STATE;
    RB_CUDA(cudaMemcpyAsync(m->ws.rgb, mono, (size_t)c->N, cudaMemcpyHostToDevice, c->stream));
    return rb_gray_enqueue(c, &m->ws, nullptr, true, nullptr, nullptr, 1);
}

extern "C" int rb_map_upload_gray(rb_map *m, const float *gray) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    if (!m->owns_ws) return RB_ERR_STATE;
    // w * h floats in, rows of the pitched plane out (its padding columns keep their zeros)
    RB_CUDA(cudaMemcpy2DAsync(m->ws.gray, (size_t)4 * c->pitch, gray, (size_t)4 * c->w, (size_t)4 * c->w, c->h,
                              cudaMemcpyHostToDevice, c->stream));
    return RB_OK;
}

extern "C" int rb_map_dog_build(rb_map *m) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    if (!m->owns_ws) return RB_ERR_STATE;
    return rb_dog_build_batch(m->c, &m->ws, 1);
}

extern "C" int rb_map_get_plane(rb_map *m, int which, float *out) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    if (!m->owns_ws || which < 0 || which > 5) return RB_ERR_ARG;
    const float *src = nullptr;
    if (which == 0) src = m->ws.img0;
    else if (which == 2) src = m->ws.dog;
    else if (which == 5) src = m->ws.gray;
    else {
        int r = rb_dog_aux_planes(c, &m->ws, 0);
        if (r) return r;
        src = m->ws.aux + (size_t)(which == 1 ? 0 : which == 3 ? 1 : 2) * c->NP;
    }
    // the pitched plane without its padding columns: w * h floats
    RB_CUDA(cudaMemcpy2DAsync(out, (size_t)4 * c->w, src, (size_t)4 * c->pitch, (size_t)4 * c->w, c->h,
                              cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

static int read_state(rb_map *m, MapState *host) {
    rb_ctx *c = m->c;
    RB_CUDA(cudaMemcpyAsync(c->pinned, m->st, sizeof(MapState), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    memcpy(host, c->pinned, sizeof(MapState));
    return RB_OK;
}

extern "C" int rb_map_detect_ss(rb_map *m, rb_map *ss, const rb_detect_params *p, double *tresh, int *l_kl_num,
                                int *kn_out);
extern "C" int rb_map_detect(rb_map *m, const rb_detect_params *p, double *tresh, int *l_kl_num, int *kn_out) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    return rb_map_detect_ss(m, m, p, tresh, l_kl_num, kn_out);
}
// rb_map_detect_ss with the detection masks at mask_dev (nullptr: the unmasked detector)
static int detect_ss(rb_map *m, rb_map *ss, const rb_detect_params *p, double *tresh, int *l_kl_num, int *kn_out,
                     const DetMask *mask_dev) {
    rb_ctx *c = m->c;
    DetChain *ch_dev = (DetChain *)((char *)c->dev_small + RB_DS_CHAIN);
    DetChain *ch_host = (DetChain *)((char *)c->pinned + RB_DS_CHAIN);
    ch_host->tresh = *tresh;
    ch_host->l_kl_num = *l_kl_num;
    ch_host->pad = 0;
    RB_CUDA(cudaMemcpyAsync(ch_dev, ch_host, sizeof(DetChain), cudaMemcpyHostToDevice, c->stream));
    int r = rb_detect_enqueue(c, m, ss->img0, ss->dog, p, ch_dev, mask_dev);
    if (r) return r;
    RB_CUDA(cudaMemcpyAsync(ch_host, ch_dev, sizeof(DetChain), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    *tresh = ch_host->tresh;
    *l_kl_num = ch_host->l_kl_num;
    if (kn_out) *kn_out = ch_host->l_kl_num;
    return RB_OK;
}
extern "C" int rb_map_detect_ss(rb_map *m, rb_map *ss, const rb_detect_params *p, double *tresh, int *l_kl_num,
                                int *kn_out) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    if (!m || !ss) return RB_ERR_ARG;
    rb_ctx *c = m->c;
    if (!ss->img0 || ss->c != c || !p || !tresh || !l_kl_num) return RB_ERR_ARG;
    return detect_ss(m, ss, p, tresh, l_kl_num, kn_out, nullptr);
}
// the host mask is copied into a device buffer of this call (a stage-level entry point: tests and tools)
extern "C" int rb_map_detect_masked(rb_map *m, rb_map *ss, const rb_detect_params *p, const uint8_t *mask, int64_t step,
                                    double *tresh, int *l_kl_num, int *kn_out) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    if (!ss) return RB_ERR_ARG;
    rb_ctx *c = m->c;
    if (!ss->img0 || ss->c != c || !p || !tresh || !l_kl_num || !mask || step < c->w) return RB_ERR_ARG;
    unsigned char *buf = nullptr;
    const size_t off = ((size_t)c->N + 255) & ~(size_t)255;
    RB_CUDA(cudaMalloc(&buf, off + sizeof(DetMask)));
    DetMask dm;
    dm.fixed = nullptr;
    dm.fixed_step = 0;
    dm.frame = buf;
    dm.frame_step = c->w;
    cudaError_t e = cudaMemcpy2DAsync(buf, (size_t)c->w, mask, (size_t)step, (size_t)c->w, c->h, cudaMemcpyHostToDevice,
                                      c->stream);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(buf + off, &dm, sizeof(dm), cudaMemcpyHostToDevice, c->stream);
    int r = RB_OK;
    if (e != cudaSuccess) {
        snprintf(c->err, sizeof(c->err), "detect_masked: %s", cudaGetErrorString(e));
        r = RB_ERR_CUDA;
    } else {
        r = detect_ss(m, ss, p, tresh, l_kl_num, kn_out, reinterpret_cast<const DetMask *>(buf + off));
    }
    cudaStreamSynchronize(c->stream);
    cudaFree(buf);
    return r;
}

extern "C" int rb_map_reestimate_thresh(rb_map *m, int knum, int nbins, float *out_thresh) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    int r = rb_reestimate_enqueue(m->c, m, knum, nbins);
    if (r) return r;
    MapState s;
    if ((r = read_state(m, &s))) return r;
    if (out_thresh) *out_thresh = s.retuned;
    return RB_OK;
}

extern "C" int rb_map_knum(rb_map *m, int *kn) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    MapState s;
    int r = read_state(m, &s);
    if (r) return r;
    *kn = s.kn;
    return RB_OK;
}

extern "C" int rb_map_counters(rb_map *m, int out[3]) {
    if (!m || !out) return RB_ERR_ARG;
    RB_ENTER(m->c);
    MapState s;
    int r = read_state(m, &s);
    if (r) return r;
    out[0] = s.fwd_match;
    out[1] = s.nmatch;
    out[2] = s.reg_num;
    return RB_OK;
}

extern "C" int rb_map_sync_host_keylines(rb_map *m, rb_keyline *dst, int capacity, int *kn) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    MapState s;
    int r = read_state(m, &s);
    if (r) return r;
    if (kn) *kn = s.kn;
    if (s.kn == 0) return RB_OK;
    if (!dst || capacity < s.kn) return RB_ERR_ARG;
    rb_keyline *tmp = nullptr;
    RB_CUDA(cudaMalloc(&tmp, sizeof(rb_keyline) * (size_t)s.kn));
    k_pack_aos<<<rb_div_up(s.kn, 128), 128, 0, c->stream>>>(m->kl, m->st, tmp);
    c->launches++;
    cudaError_t e = cudaMemcpyAsync(dst, tmp, sizeof(rb_keyline) * (size_t)s.kn, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    cudaFree(tmp);
    if (e != cudaSuccess) {
        snprintf(c->err, sizeof(c->err), "sync_host_keylines: %s", cudaGetErrorString(e));
        return RB_ERR_CUDA;
    }
    return RB_OK;
}

extern "C" int rb_map_load_keylines(rb_map *m, const rb_keyline *src, int kn, const int32_t *mask) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    if (kn < 0 || kn > c->kcap) return RB_ERR_ARG;
    rb_keyline *tmp = nullptr;
    if (kn > 0) {
        RB_CUDA(cudaMalloc(&tmp, sizeof(rb_keyline) * (size_t)kn));
        cudaError_t e = cudaMemcpyAsync(tmp, src, sizeof(rb_keyline) * (size_t)kn, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) {
            cudaFree(tmp);
            snprintf(c->err, sizeof(c->err), "load_keylines: %s", cudaGetErrorString(e));
            return RB_ERR_CUDA;
        }
    }
    k_unpack_aos<<<rb_div_up(kn > 0 ? kn : 1, 128), 128, 0, c->stream>>>(m->kl, m->st, tmp, kn);
    c->launches++;
    cudaError_t e = cudaSuccess;
    if (mask) e = cudaMemcpyAsync(m->mask, mask, sizeof(int) * (size_t)c->N, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    cudaFree(tmp);
    if (e != cudaSuccess) {
        snprintf(c->err, sizeof(c->err), "load_keylines: %s", cudaGetErrorString(e));
        return RB_ERR_CUDA;
    }
    return RB_OK;
}

extern "C" int rb_map_get_mask(rb_map *m, int32_t *out) {
    if (!m) return RB_ERR_ARG;
    RB_ENTER(m->c);
    rb_ctx *c = m->c;
    RB_CUDA(cudaMemcpyAsync(out, m->mask, sizeof(int) * (size_t)c->N, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

int rb_read_map_state(rb_map *m, MapState *host) { return read_state(m, host); }

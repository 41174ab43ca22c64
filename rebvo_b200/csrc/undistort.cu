// undistort.cu -- SURVEY.md section 8(f) rank 1: image_undistort::undistort<true> on RGB24, the step right before
// the DoG on every EuRoC frame (UseUndistort=1, src/rebvo/rebvo_first_t.cpp:231).
//
//   map   : image_undistort::image_undistort (src/VideoLib/image_undistort.cpp:29-94) -- per output pixel up to four
//           source indices and 16.16 fixed-point bilinear weights, from the rad-tan model
//           cam_model::distortHom2Hom (include/UtilLib/cam_model.h:72-84).  Built once on the host in the
//           reference's float/double mix.
//   apply : biInterp(Image<RGB24Pixel>&) (include/VideoLib/image_undistort.h:63-78): integer multiply-accumulate,
//           >> 16.  Integer-exact, so bit parity is trivial.
// Device layout: int4 inx / int4 iw per pixel; unused taps carry weight 0 on index 0, which makes the kernel
// branch-free.  Algorithmic bytes per frame: 3N in + 3N out + 32N map.
#include <math.h>

#include <new>
#include <vector>

#include "common.cuh"

struct rb_undistort {
    rb_ctx *c;
    int4 *inx, *iw;
    uint8_t *tmp_in, *tmp_out;   // staging for the host-pointer entry point
};

__global__ void __launch_bounds__(256) k_undistort_rgb(const uint8_t *__restrict__ in, uint8_t *__restrict__ out,
                                                       const int4 *__restrict__ inx, const int4 *__restrict__ iw,
                                                       int N, int nimg) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int img = blockIdx.y;
    if (i >= N || img >= nimg) return;
    const uint8_t *src = in + (size_t)img * 3 * N;
    const int4 ix = inx[i], w = iw[i];
    int r = 0, g = 0, b = 0;
#define TAP(IDX, WW)                         \
    {                                        \
        const uint8_t *p = src + 3 * (IDX);  \
        r += (WW) * (int)p[0];               \
        g += (WW) * (int)p[1];               \
        b += (WW) * (int)p[2];               \
    }
    TAP(ix.x, w.x)
    TAP(ix.y, w.y)
    TAP(ix.z, w.z)
    TAP(ix.w, w.w)
#undef TAP
    uint8_t *o = out + (size_t)img * 3 * N + 3 * (size_t)i;
    o[0] = (uint8_t)(r >> 16);
    o[1] = (uint8_t)(g >> 16);
    o[2] = (uint8_t)(b >> 16);
}

// Fused with Image<float>::ConvertRGB2BW for the per-frame pipeline (rebvo_first_t.cpp:231 then sspace::build's first
// step): gray = float(r + g + b) of the undistorted pixel, whose channels are the integer bilinear sums >> 16.  The
// undistorted colour image itself is only consumed by the encoder / viewer (out of scope), so it is never materialised: per
// frame 3N bytes of RGB in, 4N of gray out, the 32N-byte map stays L2-resident across the batch.  The RGB source is read
// through a device-resident pointer like k_rgb2gray.
// The taps are gathered as aligned 32-bit words (a pixel's three bytes start at any byte offset: two neighbouring words and a
// funnel shift; the two taps of a row are adjacent pixels almost everywhere, so three words serve both) instead of twelve
// byte loads per pixel, which bound the first version.
__device__ __forceinline__ unsigned int ug_px(const unsigned int *__restrict__ W, int byte_ofs, int last_word) {
    const int wi = byte_ofs >> 2;
    const unsigned int lo = __ldg(W + wi), hi = __ldg(W + (wi + 1 <= last_word ? wi + 1 : last_word));
    return __funnelshift_r(lo, hi, (byte_ofs & 3) * 8);   // bytes byte_ofs .. byte_ofs + 3
}
__device__ __forceinline__ void ug_acc(unsigned int v, int w, int &r, int &g, int &b) {
    r += w * (int)(v & 0xffu);
    g += w * (int)((v >> 8) & 0xffu);
    b += w * (int)((v >> 16) & 0xffu);
}
__device__ __forceinline__ float ug_pixel(const uint8_t *__restrict__ src, const int4 ix, const int4 w, int N) {
    int r = 0, g = 0, b = 0;
    if ((reinterpret_cast<uintptr_t>(src) & 3) == 0) {
        const unsigned int *W = reinterpret_cast<const unsigned int *>(src);
        const int last_word = (3 * N - 1) >> 2;
        if (ix.y == ix.x + 1 && ix.w == ix.z + 1) {   // two runs of two adjacent pixels: 6 bytes each, three words
#pragma unroll
            for (int row = 0; row < 2; row++) {
                const int ofs = 3 * (row ? ix.z : ix.x), wi = ofs >> 2, sh = (ofs & 3) * 8;
                const unsigned int w0 = __ldg(W + wi), w1 = __ldg(W + (wi + 1 <= last_word ? wi + 1 : last_word)),
                                   w2 = __ldg(W + (wi + 2 <= last_word ? wi + 2 : last_word));
                const unsigned int lo = __funnelshift_r(w0, w1, sh), hi = __funnelshift_r(w1, w2, sh);   // bytes ofs..+3, ofs+4..+7
                ug_acc(lo, row ? w.z : w.x, r, g, b);
                ug_acc(__funnelshift_r(lo, hi, 24), row ? w.w : w.y, r, g, b);                            // bytes ofs+3..+6
            }
        } else {
            ug_acc(ug_px(W, 3 * ix.x, last_word), w.x, r, g, b);
            ug_acc(ug_px(W, 3 * ix.y, last_word), w.y, r, g, b);
            ug_acc(ug_px(W, 3 * ix.z, last_word), w.z, r, g, b);
            ug_acc(ug_px(W, 3 * ix.w, last_word), w.w, r, g, b);
        }
    } else {   // (a caller's device buffer that is not 4-byte aligned)
#define TAP(IDX, WW)                         \
    {                                        \
        const uint8_t *p = src + 3 * (IDX);  \
        r += (WW) * (int)p[0];               \
        g += (WW) * (int)p[1];               \
        b += (WW) * (int)p[2];               \
    }
        TAP(ix.x, w.x)
        TAP(ix.y, w.y)
        TAP(ix.z, w.z)
        TAP(ix.w, w.w)
#undef TAP
    }
    const unsigned int s = (unsigned int)((uint8_t)(r >> 16)) + (unsigned int)((uint8_t)(g >> 16)) + (unsigned int)((uint8_t)(b >> 16));
    return (float)s;
}
// IMGS frames per thread: the 32-byte map entry of a pixel (L2-resident, but 739 MB of L2 reads per 64-frame launch when every
// frame fetches it again) is loaded once for IMGS frames
template <int IMGS>
__global__ void __launch_bounds__(256) k_undistort_gray(const uint8_t *const *__restrict__ src_pp, float *__restrict__ gray,
                                                        const int4 *__restrict__ inx, const int4 *__restrict__ iw, int N,
                                                        int nimg) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int img0 = blockIdx.y * IMGS;
    if (i >= N) return;
    const int4 ix = inx[i], w = iw[i];
    const uint8_t *src = *src_pp + (size_t)img0 * 3 * N;
    float v[IMGS];
#pragma unroll
    for (int k = 0; k < IMGS; k++) v[k] = img0 + k < nimg ? ug_pixel(src + (size_t)k * 3 * N, ix, w, N) : 0.f;
#pragma unroll
    for (int k = 0; k < IMGS; k++)
        if (img0 + k < nimg) gray[(size_t)(img0 + k) * N + i] = v[k];
}
int rb_undistort_gray_enqueue(rb_undistort *u, const void *const *src_pp, float *gray, int nimg) {
    rb_ctx *c = u->c;
    static const int imgs_env = getenv("REBVO_B200_UG_IMGS") ? atoi(getenv("REBVO_B200_UG_IMGS")) : 4;
    const int imgs = nimg >= 4 ? imgs_env : 1;
#define UG_LAUNCH(K)                                                                                                       \
    k_undistort_gray<K><<<dim3(rb_div_up(c->N, 256), rb_div_up(nimg, K)), 256, 0, c->stream>>>((const uint8_t *const *)src_pp, \
                                                                                           gray, u->inx, u->iw, c->N, nimg)
    if (imgs >= 8) UG_LAUNCH(8);
    else if (imgs >= 4) UG_LAUNCH(4);
    else if (imgs >= 2) UG_LAUNCH(2);
    else UG_LAUNCH(1);
#undef UG_LAUNCH
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// Mono twin of ug_pixel (rb_pipeline_push_mono): a mono frame m stands for the RGB24 frame (m, m, m), whose three channel
// sums are all s = sum_k iw_k * m_k, so the RGB pass's (u8)(r>>16) + (u8)(g>>16) + (u8)(b>>16) is 3 * (u8)(s>>16), with the
// same truncation.  One byte per tap.  The two taps of a row are adjacent bytes almost everywhere: one aligned word, plus
// the next one only when the pair straddles a word boundary, and one funnel shift.  The source is 4-byte aligned (a frame
// is N bytes with N % 4 == 0, and rb_pipeline_push_mono_dev refuses unaligned buffers).
__device__ __forceinline__ float ug_pixel_mono(const uint8_t *__restrict__ src, const int4 ix, const int4 w) {
    int s;
    if (ix.y == ix.x + 1 && ix.w == ix.z + 1) {
        const unsigned int *W = reinterpret_cast<const unsigned int *>(src);
        s = 0;
#pragma unroll
        for (int row = 0; row < 2; row++) {
            const int ofs = row ? ix.z : ix.x, wi = ofs >> 2;
            // (ofs % 4 == 3: byte ofs + 1 <= N - 1 is in the next word, which therefore exists)
            const unsigned int w0 = __ldg(W + wi), w1 = (ofs & 3) == 3 ? __ldg(W + wi + 1) : w0;
            const unsigned int v = __funnelshift_r(w0, w1, (ofs & 3) * 8);   // bytes ofs, ofs + 1 in the low half
            s += (row ? w.z : w.x) * (int)(v & 0xffu) + (row ? w.w : w.y) * (int)((v >> 8) & 0xffu);
        }
    } else {
        s = w.x * (int)__ldg(src + ix.x) + w.y * (int)__ldg(src + ix.y) + w.z * (int)__ldg(src + ix.z) +
            w.w * (int)__ldg(src + ix.w);
    }
    return (float)(3u * (unsigned int)(uint8_t)(s >> 16));
}
template <int IMGS>
__global__ void __launch_bounds__(256) k_undistort_gray_mono(const uint8_t *const *__restrict__ src_pp,
                                                             float *__restrict__ gray, const int4 *__restrict__ inx,
                                                             const int4 *__restrict__ iw, int N, int nimg) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int img0 = blockIdx.y * IMGS;
    if (i >= N) return;
    const int4 ix = inx[i], w = iw[i];
    const uint8_t *src = *src_pp + (size_t)img0 * N;
    float v[IMGS];
#pragma unroll
    for (int k = 0; k < IMGS; k++) v[k] = img0 + k < nimg ? ug_pixel_mono(src + (size_t)k * N, ix, w) : 0.f;
#pragma unroll
    for (int k = 0; k < IMGS; k++)
        if (img0 + k < nimg) gray[(size_t)(img0 + k) * N + i] = v[k];
}
int rb_undistort_gray_mono_enqueue(rb_undistort *u, const void *const *src_pp, float *gray, int nimg) {
    rb_ctx *c = u->c;
    static const int imgs_env = getenv("REBVO_B200_UG_IMGS") ? atoi(getenv("REBVO_B200_UG_IMGS")) : 4;
    const int imgs = nimg >= 4 ? imgs_env : 1;
#define UGM_LAUNCH(K)                                                                                              \
    k_undistort_gray_mono<K><<<dim3(rb_div_up(c->N, 256), rb_div_up(nimg, K)), 256, 0, c->stream>>>(              \
        (const uint8_t *const *)src_pp, gray, u->inx, u->iw, c->N, nimg)
    if (imgs >= 8) UGM_LAUNCH(8);
    else if (imgs >= 4) UGM_LAUNCH(4);
    else if (imgs >= 2) UGM_LAUNCH(2);
    else UGM_LAUNCH(1);
#undef UGM_LAUNCH
    RB_LAUNCH_CHECK();
    return RB_OK;
}

static inline bool inx_valid_f(float fx, float fy, int w, int h) {
    // Image::isInxValid takes `const uint&`: the float is converted to unsigned (x86-64: through a 64-bit
    // truncation, so negatives wrap to huge values and fail the upper bound)
    const unsigned int x = (unsigned int)(long long)fx, y = (unsigned int)(long long)fy;
    return x < (unsigned int)w && y < (unsigned int)h;
}
static inline int index_rc(float x, float y, int w, int h) {  // Image::GetIndexRC (image.h:121-126)
    const int xi = (int)round(x), yi = (int)round(y);
    if (xi >= w || yi >= h || xi < 0 || yi < 0) return -1;
    return yi * w + xi;
}

extern "C" int rb_undistort_create(rb_ctx *c, const double kc[5], rb_undistort **out) {
    if (!c || !kc || !out) return RB_ERR_ARG;
    *out = nullptr;
    rb_undistort *u = new (std::nothrow) rb_undistort;
    if (!u) return RB_ERR_ARG;
    memset(u, 0, sizeof(*u));
    u->c = c;
    const int w = c->w, h = c->h, N = c->N;
    const double Kc2 = kc[0], Kc4 = kc[1], Kc6 = kc[2], P1 = kc[3], P2 = kc[4];
    const float ppx = c->cam.ppx, ppy = c->cam.ppy, zfx = c->cam.zfx, zfy = c->cam.zfy;
    const double zfm = c->zfm;
    std::vector<int4> hinx(N), hiw(N);
    const float i_mult = (float)(1 << 16);
    for (int x = 0; x < w; x++)
        for (int y = 0; y < h; y++) {
            float qx = (float)x - ppx, qy = (float)y - ppy;           // cam.Img2Hom(Point2D<float>(x,y))
            {                                                          // cam.distortHom2Hom(qd)
                const double xp = qx / zfm, yp = qy / zfm;
                const double r2 = xp * xp + yp * yp;
                const double xpp = xp * (1 + r2 * (Kc2 + r2 * (Kc4 + r2 * Kc6))) + 2 * P1 * xp * yp + P2 * (r2 + 2 * xp * xp);
                const double ypp = yp * (1 + r2 * (Kc2 + r2 * (Kc4 + r2 * Kc6))) + P1 * (r2 + 2 * yp * yp) + 2 * P2 * xp * yp;
                qx = xpp * zfx;
                qy = ypp * zfy;
            }
            const float idx = qx + ppx, idy = qy + ppy;               // cam.Hom2Img(qd)
            const float p00x = floor(idx), p00y = floor(idy), p11x = floor(idx) + 1, p11y = floor(idy) + 1;
            const float p01x = p11x, p01y = p00y, p10x = p00x, p10y = p11y;
            int num = 0, inx[4] = {0, 0, 0, 0}, iw[4] = {0, 0, 0, 0};
            float wgt[4] = {0, 0, 0, 0};
            if (inx_valid_f(p00x, p00y, w, h)) {
                wgt[num] = (p11x - idx) * (p11y - idy);
                inx[num++] = index_rc(p00x, p00y, w, h);
            }
            if (inx_valid_f(p01x, p01y, w, h)) {
                wgt[num] = (idx - p00x) * (p11y - idy);
                inx[num++] = index_rc(p01x, p01y, w, h);
            }
            if (inx_valid_f(p10x, p10y, w, h)) {
                wgt[num] = (p11x - idx) * (idy - p00y);
                inx[num++] = index_rc(p10x, p10y, w, h);
            }
            if (inx_valid_f(p11x, p11y, w, h)) {
                wgt[num] = (idx - p00x) * (idy - p00y);
                inx[num++] = index_rc(p11x, p11y, w, h);
            }
            if (num > 0) {
                float sum_w = 0;
                for (int i = 0; i < num; i++) sum_w += wgt[i];
                for (int i = 0; i < num; i++) {
                    wgt[i] /= sum_w;
                    iw[i] = (int)(wgt[i] * i_mult);
                }
            }
            for (int i = num; i < 4; i++) {
                inx[i] = 0;
                iw[i] = 0;
            }
            for (int i = 0; i < num; i++)
                if (inx[i] < 0) {   // cannot happen for a valid tap; keep the kernel in bounds regardless
                    inx[i] = 0;
                    iw[i] = 0;
                }
            const int o = y * w + x;                                  // umap(x,y)
            hinx[o] = make_int4(inx[0], inx[1], inx[2], inx[3]);
            hiw[o] = make_int4(iw[0], iw[1], iw[2], iw[3]);
        }
    *out = u;
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaMalloc(&u->inx, sizeof(int4) * (size_t)N));
    RB_CUDA(cudaMalloc(&u->iw, sizeof(int4) * (size_t)N));
    RB_CUDA(cudaMalloc(&u->tmp_in, (size_t)3 * N));
    RB_CUDA(cudaMalloc(&u->tmp_out, (size_t)3 * N));
    RB_CUDA(cudaMemcpy(u->inx, hinx.data(), sizeof(int4) * (size_t)N, cudaMemcpyHostToDevice));
    RB_CUDA(cudaMemcpy(u->iw, hiw.data(), sizeof(int4) * (size_t)N, cudaMemcpyHostToDevice));
    return RB_OK;
}

extern "C" void rb_undistort_destroy(rb_undistort *u) {
    if (!u) return;
    cudaSetDevice(u->c->device);
    cudaStreamSynchronize(u->c->stream);
    cudaFree(u->inx);
    cudaFree(u->iw);
    cudaFree(u->tmp_in);
    cudaFree(u->tmp_out);
    delete u;
}

// device -> device, nimg frames, on the context's stream (no synchronisation)
int rb_undistort_enqueue(rb_undistort *u, const uint8_t *in_dev, uint8_t *out_dev, int nimg) {
    rb_ctx *c = u->c;
    dim3 grid(rb_div_up(c->N, 256), nimg);
    k_undistort_rgb<<<grid, 256, 0, c->stream>>>(in_dev, out_dev, u->inx, u->iw, c->N, nimg);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

extern "C" int rb_undistort_rgb_dev(rb_undistort *u, const uint8_t *in_dev, uint8_t *out_dev, int nimg) {
    if (!u || !in_dev || !out_dev || nimg < 1 || in_dev == out_dev) return RB_ERR_ARG;
    RB_ENTER(u->c);
    return rb_undistort_enqueue(u, in_dev, out_dev, nimg);
}

// host -> host convenience (one frame), synchronous
extern "C" int rb_undistort_rgb(rb_undistort *u, const uint8_t *in, uint8_t *out) {
    if (!u || !in || !out) return RB_ERR_ARG;
    rb_ctx *c = u->c;
    RB_ENTER(c);
    RB_CUDA(cudaMemcpyAsync(u->tmp_in, in, (size_t)3 * c->N, cudaMemcpyHostToDevice, c->stream));
    int r = rb_undistort_enqueue(u, u->tmp_in, u->tmp_out, 1);
    if (r) return r;
    RB_CUDA(cudaMemcpyAsync(out, u->tmp_out, (size_t)3 * c->N, cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

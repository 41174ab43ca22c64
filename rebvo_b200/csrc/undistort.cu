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
// branch-free.  Algorithmic bytes per frame: 3N in + 3N out + 32N map.  The pipeline's undistortion is fused into its gray
// pass (gray.cu), which reads this map.
#include <math.h>

#include <new>
#include <vector>

#include "undistort.cuh"

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
    std::vector<int4> hinx(N), hiw(N), hxy(N);
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
            int xy[4];
            for (int i = 0; i < 4; i++) xy[i] = (int)((unsigned int)(inx[i] % w) | (unsigned int)(inx[i] / w) << 16);
            hxy[o] = make_int4(xy[0], xy[1], xy[2], xy[3]);
        }
    *out = u;
    RB_CUDA(cudaSetDevice(c->device));
    RB_CUDA(cudaMalloc(&u->inx, sizeof(int4) * (size_t)N));
    RB_CUDA(cudaMalloc(&u->iw, sizeof(int4) * (size_t)N));
    RB_CUDA(cudaMalloc(&u->ixy, sizeof(int4) * (size_t)N));
    RB_CUDA(cudaMalloc(&u->tmp_in, (size_t)3 * N));
    RB_CUDA(cudaMalloc(&u->tmp_out, (size_t)3 * N));
    RB_CUDA(cudaMemcpy(u->inx, hinx.data(), sizeof(int4) * (size_t)N, cudaMemcpyHostToDevice));
    RB_CUDA(cudaMemcpy(u->iw, hiw.data(), sizeof(int4) * (size_t)N, cudaMemcpyHostToDevice));
    RB_CUDA(cudaMemcpy(u->ixy, hxy.data(), sizeof(int4) * (size_t)N, cudaMemcpyHostToDevice));
    return RB_OK;
}

extern "C" void rb_undistort_destroy(rb_undistort *u) {
    if (!u) return;
    cudaSetDevice(u->c->device);
    cudaStreamSynchronize(u->c->stream);
    cudaFree(u->inx);
    cudaFree(u->iw);
    cudaFree(u->ixy);
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

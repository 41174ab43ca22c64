// dog.cu -- scale space: bit-exact float32 integral-image box blurs, DoG and gradient.
//
// Replaces sspace::build (src/mtracklib/sspace.cpp:52-85) = 2 x iigauss::smooth (iigauss.cpp:91-101),
// each 3 x { iimage::load (iimage.cpp:53-71) ; iimage::average (iimage.cpp:86-128) }.
//
// Parity constraint (SURVEY.md section 0 item 5): the reference's integral images are float32 and exceed
// 2^24, so every add must happen in the reference's order: each row left->right, then each column
// top->bottom.  The kernels therefore keep one sequential chain per row / per column and get their
// parallelism from rows x columns x images of a batch; the library is compiled with -fmad=false so no
// mul+add is ever contracted.
//
// Pass structure per box stage (B images x 2 filters in one launch):
//   k_rowscan<AVG> : S(x,y)  = sum_{i<=x} avg(I_prev)(i,y)   warp per 32-row band, smem-transposed tiles
//   k_colscan      : I(x,y)  = sum_{j<=y} S(x,j)              thread per 4 columns, float4 streams
// and a final k_blur_dog that evaluates the last box of both filters, Img(0) and the DoG.
#include <stdlib.h>
#include <new>

#include "common.cuh"

// ---------------------------------------------------------------------------------------------------
// iimage::average for one pixel (iimage.cpp:86-128).  The nine regions of the reference collapse to:
// taps A=I(xr,yb) B=I(xl,yb) C=I(xr,yt) D=I(xl,yt) with xr=min(x+d2,w-1), yb=min(y+d2,h-1), xl=x-d2-1,
// yt=y-d2-1; a tap whose xl / yt is negative is absent; the subtraction order is A-B-C+D except in the
// bottom band (y >= h-d2) where the reference writes A-C-B+D; the factor is a=1.0/(d*d) in the centre
// region and the per-pixel reciprocal box area of iimage::build_average (iimage.cpp:134-179) elsewhere.
//
// The code is branch-free on purpose: the four loads are unconditional (an absent tap reads a clamped address and
// is dropped by a select) and the factor comes from a (d2+1)x(d2+1) table of the reciprocal clipped areas
// tab[(cy-d2-1)*8 + (cx-d2-1)] = (float)(1.0/(double)(float)(cx*cy)) (host-computed, staged in shared memory; its
// centre entry cx=cy=d equals a).  With branches around each pixel the compiler cannot hoist the loads of the
// next pixels, and a 32x32 tile degenerates into 32 dependent L2 round trips.
#define BOX_TAB_W 8
#define BOX_TAB_N (BOX_TAB_W * BOX_TAB_W)
__device__ __forceinline__ float box_avg(const float *__restrict__ I, int x, int y, int w, int h, int d,
                                         int d2, const float *__restrict__ tab) {
    const bool left = x < d2 + 1, right = x >= w - d2;
    const bool top = y < d2 + 1, bottom = y >= h - d2;
    const int xr = right ? w - 1 : x + d2;
    const int yb = bottom ? h - 1 : y + d2;
    const int xl = left ? 0 : x - d2 - 1, yt = top ? 0 : y - d2 - 1;
    const float A = I[yb * w + xr], B = I[yb * w + xl], C = I[yt * w + xr], D = I[yt * w + xl];
    const float t1 = bottom ? C : B, t2 = bottom ? B : C;   // bottom band: A-C-B+D, elsewhere A-B-C+D
    const bool h1 = bottom ? !top : !left, h2 = bottom ? !left : !top;
    float r = A;
    r = h1 ? r - t1 : r;
    r = h2 ? r - t2 : r;
    r = (!top && !left) ? r + D : r;
    const int cx = left ? x + d2 + 1 : (right ? w - x + d2 : d);   // clipped box extents (build_average)
    const int cy = top ? y + d2 + 1 : (bottom ? h - y + d2 : d);
    return r * tab[(cy - d2 - 1) * BOX_TAB_W + (cx - d2 - 1)];
}

// Image<float>::ConvertRGB2BW (image.h:197-203): b+g+r as float, 4 pixels per thread
// src_pp (optional): the RGB source is read through a device-resident pointer, so that one captured graph serves
// whichever staging region / caller buffer a push uses (rb_pipeline)
__global__ void __launch_bounds__(256) k_rgb2gray(const uint32_t *__restrict__ rgb_fixed,
                                                  const uint32_t *const *__restrict__ src_pp,
                                                  float4 *__restrict__ gray, size_t n4) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const uint32_t *__restrict__ rgb = src_pp ? *src_pp : rgb_fixed;
    uint32_t a = rgb[3 * i], b = rgb[3 * i + 1], c = rgb[3 * i + 2];
    // bytes: a = p0.0 p0.1 p0.2 p1.0 | b = p1.1 p1.2 p2.0 p2.1 | c = p2.2 p3.0 p3.1 p3.2
    float4 o;
    o.x = (float)((a & 0xff) + ((a >> 8) & 0xff) + ((a >> 16) & 0xff));
    o.y = (float)((a >> 24) + (b & 0xff) + ((b >> 8) & 0xff));
    o.z = (float)(((b >> 16) & 0xff) + (b >> 24) + (c & 0xff));
    o.w = (float)(((c >> 8) & 0xff) + ((c >> 16) & 0xff) + (c >> 24));
    gray[i] = o;
}

// The same for 8-bit grayscale input (rb_pipeline_push_mono): a mono frame m stands for the RGB24 frame (m, m, m), so a
// pixel's b+g+r is the integer 3v and the plane is bit-identical to k_rgb2gray's on the replicated frame.  4 pixels per
// thread: one 32-bit load, one float4 store; the source is read through src_pp like k_rgb2gray's.
__global__ void __launch_bounds__(256) k_mono2gray(const uint32_t *__restrict__ mono_fixed,
                                                   const uint32_t *const *__restrict__ src_pp,
                                                   float4 *__restrict__ gray, size_t n4) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    const uint32_t *__restrict__ mono = src_pp ? *src_pp : mono_fixed;
    const uint32_t a = mono[i];
    float4 o;
    o.x = (float)(3u * (a & 0xff));
    o.y = (float)(3u * ((a >> 8) & 0xff));
    o.z = (float)(3u * ((a >> 16) & 0xff));
    o.w = (float)(3u * (a >> 24));
    gray[i] = o;
}

// Row pass: warp per band of 32 rows of one image.  Tiles of 32x32 are produced coalesced (optionally
// through box_avg of the previous integral image), transposed through shared memory so that each lane
// owns one row, scanned sequentially (the reference's add order), and stored coalesced.
template <bool AVG>
__global__ void __launch_bounds__(128) k_rowscan(const float *__restrict__ in, float *__restrict__ out,
                                                 int w, int h, int nimg, int in_mod, int nper, int d_f0,
                                                 int d_f1, const float *__restrict__ tab_f0,
                                                 const float *__restrict__ tab_f1) {
    __shared__ float tile[4][32][33];
    __shared__ float stab[4][BOX_TAB_N];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * 4 + warp;
    const int bands = (h + 31) >> 5;
    const int img = gw / bands, band = gw - img * bands;
    if (img >= nimg) return;
    const size_t N = (size_t)w * h;
    const float *__restrict__ I = in + (size_t)(img % in_mod) * N;
    float *__restrict__ O = out + (size_t)img * N;
    const bool f1 = (img / nper) != 0;
    const int d = f1 ? d_f1 : d_f0;
    const int d2 = d / 2;
    if (AVG) {
        const float *__restrict__ tg = f1 ? tab_f1 : tab_f0;
        stab[warp][lane] = tg[lane];
        stab[warp][lane + 32] = tg[lane + 32];
        __syncwarp();
    }
    const float *tab = stab[warp];
    const int y0 = band * 32;
    float v[32];
    float carry = 0.f;

    // branch-free tile production: clamped coordinates + select, so that all loads of a tile are in flight at once
#define LOAD_TILE(X0)                                                           \
    {                                                                           \
        const int x = (X0) + lane;                                              \
        const int xc = x < w ? x : w - 1;                                       \
        _Pragma("unroll") for (int r = 0; r < 32; r++) {                        \
            const int y = y0 + r;                                               \
            const int yc = y < h ? y : h - 1;                                   \
            const float t = AVG ? box_avg(I, xc, yc, w, h, d, d2, tab) : I[(size_t)yc * w + xc]; \
            v[r] = (y < h && x < w) ? t : 0.f;                                  \
        }                                                                       \
    }
    LOAD_TILE(0);
    for (int x0 = 0; x0 < w; x0 += 32) {
#pragma unroll
        for (int r = 0; r < 32; r++) tile[warp][r][lane] = v[r];
        __syncwarp();
        if (x0 + 32 < w) LOAD_TILE(x0 + 32);  // next tile's loads overlap the dependent add chain
        float *row = tile[warp][lane];
#pragma unroll
        for (int cidx = 0; cidx < 32; cidx++) {
            carry = carry + row[cidx];  // I(x,y) = I(x-1,y) + in(x,y), iimage.cpp:56-60
            row[cidx] = carry;
        }
        __syncwarp();
        const int x = x0 + lane;
        if (x < w) {
#pragma unroll
            for (int r = 0; r < 32; r++) {
                const int y = y0 + r;
                if (y < h) O[(size_t)y * w + x] = tile[warp][r][lane];
            }
        }
        __syncwarp();
    }
#undef LOAD_TILE
}

// Column pass: thread per 4 adjacent columns; I(x,y) += I(x,y-1) top->bottom (iimage.cpp:62-66)
__global__ void __launch_bounds__(64) k_colscan(const float4 *__restrict__ in, float4 *__restrict__ out,
                                                int w4, int h, int nimg) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int img = idx / w4, cx = idx - img * w4;
    if (img >= nimg) return;
    const float4 *__restrict__ I = in + (size_t)img * w4 * h + cx;
    float4 *__restrict__ O = out + (size_t)img * w4 * h + cx;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    constexpr int U = 16;
    for (int y = 0; y < h; y += U) {
        float4 v[U];
#pragma unroll
        for (int k = 0; k < U; k++)
            if (y + k < h) v[k] = __ldcs(&I[(size_t)(y + k) * w4]);
#pragma unroll
        for (int k = 0; k < U; k++)
            if (y + k < h) {
                acc.x = v[k].x + acc.x;
                acc.y = v[k].y + acc.y;
                acc.z = v[k].z + acc.z;
                acc.w = v[k].w + acc.w;
                O[(size_t)(y + k) * w4] = acc;
            }
    }
}

// Column pass, software-pipelined: VW adjacent columns per thread, the next U rows are in flight while the current U are added
// and stored (the add chain per column is the reference's: top to bottom, one float add per row)
template <int VW> struct ColVec;
template <> struct ColVec<4> { typedef float4 T; };
__device__ __forceinline__ void col_acc(float4 &a, const float4 &v) { a.x = v.x + a.x; a.y = v.y + a.y; a.z = v.z + a.z; a.w = v.w + a.w; }
template <int VW, int U>
__global__ void __launch_bounds__(64) k_colscan_pipe(const typename ColVec<VW>::T *__restrict__ in,
                                                     typename ColVec<VW>::T *__restrict__ out, int wv, int h, int nimg) {
    typedef typename ColVec<VW>::T V;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int img = idx / wv, cx = idx - img * wv;
    if (img >= nimg) return;
    const V *__restrict__ I = in + (size_t)img * wv * h + cx;
    V *__restrict__ O = out + (size_t)img * wv * h + cx;
    V acc;
    memset(&acc, 0, sizeof(acc));
    V a[U], b[U];
#pragma unroll
    for (int k = 0; k < U; k++)
        if (k < h) a[k] = __ldcs(&I[(size_t)k * wv]);
    for (int y = 0; y < h; y += 2 * U) {
#pragma unroll
        for (int k = 0; k < U; k++)
            if (y + U + k < h) b[k] = __ldcs(&I[(size_t)(y + U + k) * wv]);
#pragma unroll
        for (int k = 0; k < U; k++)
            if (y + k < h) {
                col_acc(acc, a[k]);
                O[(size_t)(y + k) * wv] = acc;
            }
#pragma unroll
        for (int k = 0; k < U; k++)
            if (y + 2 * U + k < h) a[k] = __ldcs(&I[(size_t)(y + 2 * U + k) * wv]);
#pragma unroll
        for (int k = 0; k < U; k++)
            if (y + U + k < h) {
                col_acc(acc, b[k]);
                O[(size_t)(y + U + k) * wv] = acc;
            }
    }
}

// Last box of both filters + sspace::build_dog (sspace.cpp:63-70): img0, dog = img1 - img0
#define BLUR_RY 4
__global__ void __launch_bounds__(256) k_blur_dog(const float *__restrict__ I, float *__restrict__ img0,
                                                  float *__restrict__ dog, float *__restrict__ img1_opt,
                                                  int w, int h, int B, int d0, int d1,
                                                  const float *__restrict__ tab0, const float *__restrict__ tab1) {
    __shared__ float st0[BOX_TAB_N], st1[BOX_TAB_N];
    if (threadIdx.x < BOX_TAB_N) st0[threadIdx.x] = tab0[threadIdx.x];
    else if (threadIdx.x < 2 * BOX_TAB_N) st1[threadIdx.x - BOX_TAB_N] = tab1[threadIdx.x - BOX_TAB_N];
    __syncthreads();
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y0 = blockIdx.y * BLUR_RY;
    const int b = blockIdx.z;
    if (x >= w) return;
    const size_t N = (size_t)w * h;
    const float *I0 = I + (size_t)b * N, *I1 = I + (size_t)(B + b) * N;
    // BLUR_RY rows per thread, unrolled: 8 x BLUR_RY independent taps in flight per thread (one row per thread left
    // the pass latency-bound: 92k tiny blocks, each paying the table load and a barrier for 8 loads per thread)
    float v0[BLUR_RY], v1[BLUR_RY];
#pragma unroll
    for (int r = 0; r < BLUR_RY; r++) {
        const int y = min(y0 + r, h - 1);
        v0[r] = box_avg(I0, x, y, w, h, d0, d0 / 2, st0);
        v1[r] = box_avg(I1, x, y, w, h, d1, d1 / 2, st1);
    }
#pragma unroll
    for (int r = 0; r < BLUR_RY; r++) {
        const int y = y0 + r;
        if (y < h) {
            const size_t o = (size_t)b * N + (size_t)y * w + x;
            img0[o] = v0[r];
            dog[o] = v1[r] - v0[r];
            if (img1_opt) img1_opt[(size_t)y * w + x] = v1[r];
        }
    }
}


// ---------------------------------------------------------------------------------------------------
// Last box + DoG with TMA-staged tiles.  k_blur_dog above reads its 2 x 4 taps per pixel through L1 with unaligned,
// overlapping row segments.  Here a CTA owns a 64 x 32 output tile: ONE elected thread issues two
// cp.async.bulk.tensor loads (the (64+d) x (32+d) windows of the two filters' integral images, out-of-image parts
// zero-filled by the TMA unit, completion counted on an mbarrier), every thread evaluates iimage::average from shared
// memory with box_avg's exact arithmetic, and the two result tiles leave through TMA stores (the unit clips the tiles
// that stick out of the image).  No per-thread address arithmetic or predication for the window, each integral value is
// fetched once per tile.
#include <cuda.h>
#define BT_W 64
#define BT_H 32
#define BT_BW 76            // window width in floats: 64 + 9 (largest box) rounded up to a multiple of 4 (16-byte rows)
#define BT_BH 41            // 32 + 9
#define BT_THREADS 256
struct BlurTmaSmem {       // 64 x 32 tiles: more resident CTAs rather than a persistent two-stage version of this kernel
    alignas(128) float win0[BT_BH][BT_BW];   // (every TMA source / destination tile is 128-byte aligned)
    alignas(128) float win1[BT_BH][BT_BW];
    alignas(128) float o0[BT_H][BT_W];
    alignas(128) float o1[BT_H][BT_W];
    alignas(8) unsigned long long bar;
    float tab[2][BOX_TAB_N];
};
__global__ void __launch_bounds__(BT_THREADS) k_blur_dog_tma(const __grid_constant__ CUtensorMap tm_in,
                                                             const __grid_constant__ CUtensorMap tm_img0,
                                                             const __grid_constant__ CUtensorMap tm_dog, int w, int h,
                                                             int nimg, int out_slot, int d0, int d1,
                                                             const float *__restrict__ tab0, const float *__restrict__ tab1,
                                                             int *fail) {
    extern __shared__ __align__(128) unsigned char bt_raw[];
    BlurTmaSmem &sm = *reinterpret_cast<BlurTmaSmem *>((reinterpret_cast<uintptr_t>(bt_raw) + 127) & ~(uintptr_t)127);
    const int tid = threadIdx.x;
    const int x0 = blockIdx.x * BT_W, y0 = blockIdx.y * BT_H, b = blockIdx.z;
    const int d20 = d0 / 2, d21 = d1 / 2;
    // window origin: the TMA unit wants the first element of a box row 16-byte aligned in global memory, so the windows start
    // 8 columns left of the tile (left halo <= 5 for the largest box) and are 8 + 64 + 4 = 76 wide
    const int wx0[2] = {x0 - 8, x0 - 8}, wy0[2] = {y0 - d20 - 1, y0 - d21 - 1};
    const unsigned int bar = (unsigned int)__cvta_generic_to_shared(&sm.bar);
    if (tid < BOX_TAB_N) sm.tab[0][tid] = tab0[tid];
    else if (tid < 2 * BOX_TAB_N) sm.tab[1][tid - BOX_TAB_N] = tab1[tid - BOX_TAB_N];
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == 0) {
        const unsigned int bytes = 2u * BT_BH * BT_BW * 4u;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
#pragma unroll
        for (int f = 0; f < 2; f++) {
            const unsigned int dst = (unsigned int)__cvta_generic_to_shared(f ? &sm.win1[0][0] : &sm.win0[0][0]);
            const int z = f * nimg + b;
            asm volatile(
                "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                ::"r"(dst), "l"(&tm_in), "r"(wx0[f]), "r"(wy0[f]), "r"(z), "r"(bar)
                : "memory");
        }
    }
    {   // wait for the two windows (bounded: a broken copy flags an error instead of hanging the device)
        unsigned int ok = 0;
        const long long t0 = clock64();
        while (!ok) {
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                         : "=r"(ok) : "r"(bar) : "memory");
            if (!ok && clock64() - t0 > (1ll << 28)) {
                if (tid == 0) *fail = 1;
                break;
            }
        }
    }
    // 64 x 32 pixels, 256 threads: thread = column (tid & 63), rows (tid >> 6) + 4k
    const int lx = tid & 63, ly0 = tid >> 6;
    const int x = x0 + lx;
    const int dm = d20 > d21 ? d20 : d21;
    if (x0 >= dm + 1 && x0 + BT_W - 1 < w - dm && y0 >= dm + 1 && y0 + BT_H - 1 < h - dm) {
        // centre region of iimage::average for the whole tile and both filters: constant tap offsets, no selects
        const float a0 = sm.tab[0][d20 * BOX_TAB_W + d20], a1 = sm.tab[1][d21 * BOX_TAB_W + d21];
        const float *r0 = &sm.win0[0][lx + 8 + d20], *l0 = &sm.win0[0][lx + 8 - d20 - 1];
        const float *r1 = &sm.win1[0][lx + 8 + d21], *l1 = &sm.win1[0][lx + 8 - d21 - 1];
#pragma unroll
        for (int k = 0; k < BT_H / 4; k++) {
            const int ly = ly0 + 4 * k;
            float v0 = r0[(ly + d0) * BT_BW] - l0[(ly + d0) * BT_BW];   // A - B
            v0 = v0 - r0[ly * BT_BW];                                   //   - C
            v0 = v0 + l0[ly * BT_BW];                                   //   + D
            float v1 = r1[(ly + d1) * BT_BW] - l1[(ly + d1) * BT_BW];
            v1 = v1 - r1[ly * BT_BW];
            v1 = v1 + l1[ly * BT_BW];
            v0 *= a0;
            v1 *= a1;
            sm.o0[ly][lx] = v0;
            sm.o1[ly][lx] = v1 - v0;
        }
    } else {
        // border tiles: the dropped terms are the taps on column / row -1, zero-filled by the tensor map (see k_rowscan_tma_avg)
        const float *rr[2], *ll[2], *tc[2];
        int jbmax[2];
#pragma unroll
        for (int f = 0; f < 2; f++) {
            const int d = f ? d1 : d0, d2 = f ? d21 : d20;
            const float(*W)[BT_BW] = f ? sm.win1 : sm.win0;
            const int xr = (x + d2 < w - 1 ? x + d2 : w - 1) - wx0[f], xl = x - d2 - 1 - wx0[f];
            const bool left = x < d2 + 1, right = x >= w - d2;
            int cxi = (left ? x + d2 + 1 : (right ? w - x + d2 : d)) - d2 - 1;
            cxi = cxi < 0 ? 0 : cxi;   // (columns >= w: clipped by the store)
            rr[f] = &W[0][xr];
            ll[f] = &W[0][xl];
            tc[f] = sm.tab[f] + cxi;
            jbmax[f] = h - 1 - wy0[f];
        }
#pragma unroll 2
        for (int k = 0; k < BT_H / 4; k++) {
            const int ly = ly0 + 4 * k, y = y0 + ly;
            float v[2];
#pragma unroll
            for (int f = 0; f < 2; f++) {
                const int d = f ? d1 : d0, d2 = f ? d21 : d20;
                const bool top = y < d2 + 1, bottom = y >= h - d2;
                const int jb = ly + d < jbmax[f] ? ly + d : jbmax[f];
                int cyi = (top ? y + d2 + 1 : (bottom ? h - y + d2 : d)) - d2 - 1;
                cyi = cyi < 0 ? 0 : cyi;   // (rows >= h: clipped by the store)
                const float A = rr[f][jb * BT_BW], B = ll[f][jb * BT_BW], C = rr[f][ly * BT_BW], D = ll[f][ly * BT_BW];
                const float t1 = bottom ? C : B, t2 = bottom ? B : C;   // bottom band: A-C-B+D, elsewhere A-B-C+D
                float r = A - t1;
                r = r - t2;
                r = r + D;
                v[f] = r * tc[f][cyi * BOX_TAB_W];
            }
            sm.o0[ly][lx] = v[0];
            sm.o1[ly][lx] = v[1] - v[0];
        }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the TMA unit
    __syncthreads();
    if (tid == 0) {
        const unsigned int s0 = (unsigned int)__cvta_generic_to_shared(&sm.o0[0][0]);
        const unsigned int s1 = (unsigned int)__cvta_generic_to_shared(&sm.o1[0][0]);
        const int z = out_slot + b;
        asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(&tm_img0),
                     "r"(x0), "r"(y0), "r"(z), "r"(s0)
                     : "memory");
        asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(&tm_dog), "r"(x0),
                     "r"(y0), "r"(z), "r"(s1)
                     : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // shared memory may be released
    }
}

// tensor maps of a workspace (driver entry point fetched at run time: the library does not link libcuda)
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                        const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static bool make_tmap3(CUtensorMap *tm, float *base, int w, int h, int nimg, int bw, int bh, bool swizzle128 = false) {
    static PFN_tmapEncodeTiled enc = nullptr;
    if (!enc) {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn) return false;
        enc = (PFN_tmapEncodeTiled)fn;
    }
    const cuuint64_t dims[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)nimg};
    const cuuint64_t strides[2] = {(cuuint64_t)w * 4, (cuuint64_t)w * h * 4};
    const cuuint32_t box[3] = {(cuuint32_t)bw, (cuuint32_t)bh, 1};
    const cuuint32_t es[3] = {1, 1, 1};
    return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
               swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
// tensor map slots of a workspace
enum { TM_I_BLUR = 0, TM_IMG0, TM_DOG, TM_GRAY, TM_S, TM_I0_F0, TM_I0_F1, TM_I_F0, TM_I_F1, TM_COUNT };
int rb_dog_make_tmaps(rb_ctx *c, DogWS *ws) {
    ws->tma_ok = false;
    ws->tma_row_ok = false;
    const char *e = getenv("REBVO_B200_BLUR_TMA");
    const char *er = getenv("REBVO_B200_ROW_TMA");
    const bool want_blur = !(e && atoi(e) == 0), want_row = !(er && atoi(er) == 0);
    if (!want_blur && !want_row) return RB_OK;
    if ((c->w * 4) % 16) return RB_OK;
    CUtensorMap *t = new (std::nothrow) CUtensorMap[TM_COUNT];
    if (!t) return RB_OK;
    ws->tmaps = t;
    if (want_blur) {
        bool ok = make_tmap3(&t[TM_I_BLUR], ws->I, c->w, c->h, 2 * ws->B, BT_BW, BT_BH) &&
                  make_tmap3(&t[TM_IMG0], ws->img0, c->w, c->h, ws->B, BT_W, BT_H) &&
                  make_tmap3(&t[TM_DOG], ws->dog, c->w, c->h, ws->B, BT_W, BT_H);
        ok = ok && cudaFuncSetAttribute(k_blur_dog_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BlurTmaSmem) + 128) == cudaSuccess;
        if (!ok) cudaGetLastError();
        ws->tma_ok = ok;
    }
    if (want_row) {
        // row pass: 32 x 32 tiles, 128-byte swizzle on the tiles the sequential scan walks row-wise (gray in, S out); the
        // box-average inputs are (32 + d) x 32 windows read column-wise (no swizzle)
        const int (*d)[3] = c->plan.d;
        bool ok = make_tmap3(&t[TM_GRAY], ws->gray, c->w, c->h, ws->B, 32, 32, true) &&
                  make_tmap3(&t[TM_S], ws->S, c->w, c->h, 2 * ws->B, 32, 32, true) &&
                  make_tmap3(&t[TM_I0_F0], ws->I0, c->w, c->h, ws->B, 32, 32 + d[0][0]) &&
                  make_tmap3(&t[TM_I0_F1], ws->I0, c->w, c->h, ws->B, 32, 32 + d[1][0]) &&
                  make_tmap3(&t[TM_I_F0], ws->I, c->w, c->h, 2 * ws->B, 32, 32 + d[0][1]) &&
                  make_tmap3(&t[TM_I_F1], ws->I, c->w, c->h, 2 * ws->B, 32, 32 + d[1][1]);
        if (!ok) cudaGetLastError();
        ws->tma_row_ok = ok;
        ws->tma_row_mask = er ? atoi(er) : 1;   // 1 = both row passes, 2 = plain only, 3 = box average only (diagnosis)
    }
    return RB_OK;
}

// sspace::calc_gradient (sspace.cpp:75-85), materialised only for the debug accessor; borders = 0
__global__ void k_gradient(const float *__restrict__ img0, float *__restrict__ dx, float *__restrict__ dy,
                           int w, int h) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= w) return;
    float gx = 0.f, gy = 0.f;
    if (x >= 1 && x < w - 1 && y >= 1 && y < h - 1) {
        gx = img0[y * w + x + 1] - img0[y * w + x - 1];
        gy = img0[(y + 1) * w + x] - img0[(y - 1) * w + x];
    }
    dx[y * w + x] = gx;
    dy[y * w + x] = gy;
}

// ---------------------------------------------------------------------------------------------------
int rb_dogws_alloc(rb_ctx *c, DogWS *ws, int B) {
    memset(ws, 0, sizeof(*ws));
    ws->B = B;
    const size_t N = c->N;
    RB_CUDA(cudaMalloc(&ws->rgb, (size_t)B * 3 * N));
    RB_CUDA(cudaMalloc(&ws->gray, (size_t)B * N * 4));
    RB_CUDA(cudaMalloc(&ws->S, (size_t)2 * B * N * 4));
    RB_CUDA(cudaMalloc(&ws->I0, (size_t)B * N * 4));
    RB_CUDA(cudaMalloc(&ws->I, (size_t)2 * B * N * 4));
    RB_CUDA(cudaMalloc(&ws->img0, (size_t)B * N * 4));
    RB_CUDA(cudaMalloc(&ws->dog, (size_t)B * N * 4));
    RB_CUDA(cudaMalloc(&ws->aux, (size_t)3 * N * 4));
    return rb_dog_make_tmaps(c, ws);
}

void rb_dogws_free(DogWS *ws) {
    cudaFree(ws->rgb);
    cudaFree(ws->gray);
    cudaFree(ws->S);
    cudaFree(ws->I0);
    cudaFree(ws->I);
    cudaFree(ws->img0);
    cudaFree(ws->dog);
    cudaFree(ws->aux);
    delete[] (CUtensorMap *)ws->tmaps;
    memset(ws, 0, sizeof(*ws));
}

int rb_dog_gray(rb_ctx *c, DogWS *ws, int nimg, const void *const *src_pp) {
    const size_t n4 = (size_t)nimg * c->N / 4;
    k_rgb2gray<<<(unsigned)((n4 + 255) / 256), 256, 0, c->stream>>>((const uint32_t *)ws->rgb,
                                                                   (const uint32_t *const *)src_pp,
                                                                   (float4 *)ws->gray, n4);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// mono -> gray: nimg frames of N bytes (the source must be 4-byte aligned; N is a multiple of 4)
int rb_dog_gray_mono(rb_ctx *c, DogWS *ws, int nimg, const void *const *src_pp) {
    const size_t n4 = (size_t)nimg * c->N / 4;
    k_mono2gray<<<(unsigned)((n4 + 255) / 256), 256, 0, c->stream>>>((const uint32_t *)ws->rgb,
                                                                    (const uint32_t *const *)src_pp,
                                                                    (float4 *)ws->gray, n4);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// ---------------------------------------------------------------------------------------------------
// Row pass, asynchronous version: the raw input of a band is streamed into a per-warp shared-memory ring of
// 32-column chunks with cp.async (16 B per lane, no registers, NS-3 chunks in flight ahead of the consumer), so the
// sequential scan never waits for a DRAM round trip.  Tile t of a box-averaged pass needs the columns
// [32t-d2-1, 32t+31+d2], i.e. chunks t-1, t, t+1 of the rows [y0-d2-1, y0+31+d2]; every integral value is fetched
// from memory once and the four taps of iimage::average come from shared memory.  Same arithmetic and add order as
// k_rowscan (bit-identical output).
#define RING_NS 4          // ring slots: 3 live chunks + 1 in flight
#define RING_WARPS 4
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc, int src_bytes) {
    const unsigned int s = (unsigned int)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gsrc), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

template <bool AVG>
__global__ void __launch_bounds__(32 * RING_WARPS) k_rowscan_ring(const float *__restrict__ in, float *__restrict__ out,
                                                                  int w, int h, int nimg, int in_mod, int nper, int d_f0,
                                                                  int d_f1, const float *__restrict__ tab_f0,
                                                                  const float *__restrict__ tab_f1, int rmax) {
    extern __shared__ __align__(16) float smem_ring[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * RING_WARPS + warp;
    const int bands = (h + 31) >> 5;
    const int img = gw / bands, band = gw - img * bands;
    if (img >= nimg) return;
    // per-warp carve-up: ring [RING_NS][rmax][32], tile [32][33], table [64]
    float *ring = smem_ring + (size_t)warp * (RING_NS * rmax * 32 + 32 * 33 + BOX_TAB_N);
    float(*tile)[33] = reinterpret_cast<float(*)[33]>(ring + RING_NS * rmax * 32);
    float *tab = ring + RING_NS * rmax * 32 + 32 * 33;
    const size_t N = (size_t)w * h;
    const float *__restrict__ I = in + (size_t)(img % in_mod) * N;
    float *__restrict__ O = out + (size_t)img * N;
    const bool f1 = (img / nper) != 0;
    const int d = AVG ? (f1 ? d_f1 : d_f0) : 1;
    const int d2 = AVG ? d / 2 : 0;
    const int R = AVG ? 32 + d : 32;                 // rows staged per chunk
    const int yb0 = AVG ? band * 32 - d2 - 1 : band * 32;   // image row of ring row 0
    if (AVG) {
        const float *__restrict__ tg = f1 ? tab_f1 : tab_f0;
        tab[lane] = tg[lane];
        tab[lane + 32] = tg[lane + 32];
    }
    const int y0 = band * 32;
    const bool band_interior = AVG && (y0 >= d2 + 1) && (y0 + 31 < h - d2);
    const int nchunk = (w + 31) >> 5;
    const int sub = lane >> 3, piece = lane & 7;   // 8 lanes x 16 B cover one 32-float row; 4 rows per instruction

    auto issue_chunk = [&](int ci) {
        if (ci >= 0 && ci < nchunk) {
            float *dst0 = ring + (size_t)(ci % RING_NS) * rmax * 32;
            const int gx = ci * 32 + piece * 4;
            int bytes = (w - gx) * 4;
            bytes = bytes < 0 ? 0 : (bytes > 16 ? 16 : bytes);
            const int gxc = gx < w ? gx : 0;
            for (int j = sub; j < R; j += 4) {
                int gy = yb0 + j;
                gy = gy < 0 ? 0 : (gy > h - 1 ? h - 1 : gy);
                cp_async16(dst0 + j * 32 + piece * 4, I + (size_t)gy * w + gxc, bytes);
            }
        }
        cp_async_commit();
    };
    // prologue: chunks 0 .. RING_NS-2
#pragma unroll
    for (int ci = 0; ci < RING_NS - 1; ci++) issue_chunk(ci);

    float carry = 0.f;
    for (int t = 0; t < nchunk; t++) {
        cp_async_wait<RING_NS - 3>();   // chunks <= t+1 have landed (this lane's copies)
        __syncwarp();                   // ... and everybody else's
        const int x = t * 32 + lane;
        const int xc = x < w ? x : w - 1;
        if (AVG && band_interior && t * 32 >= d2 + 1 && t * 32 + 31 < w - d2) {
            // centre region of iimage::average for the whole tile (80 % of the tiles): constant tap offsets, no selects
            const int xr = x + d2, xl = x - d2 - 1;
            const float *colr = ring + (size_t)((xr >> 5) % RING_NS) * rmax * 32 + (xr & 31);
            const float *coll = ring + (size_t)((xl >> 5) % RING_NS) * rmax * 32 + (xl & 31);
            const float *colr_b = colr + d * 32, *coll_b = coll + d * 32;   // bottom taps: ring row r + d
            const float a = tab[d2 * BOX_TAB_W + d2];
#pragma unroll
            for (int r = 0; r < 32; r++) {
                float v = colr_b[r * 32] - coll_b[r * 32];   // A - B
                v = v - colr[r * 32];                        //   - C
                v = v + coll[r * 32];                        //   + D
                tile[r][lane] = v * a;
            }
        } else if (AVG) {
            const bool left = xc < d2 + 1, right = xc >= w - d2;
            const int xr = right ? w - 1 : xc + d2, xl = left ? 0 : xc - d2 - 1;
            const int cx = left ? xc + d2 + 1 : (right ? w - xc + d2 : d);
            const float *colr = ring + (size_t)((xr >> 5) % RING_NS) * rmax * 32 + (xr & 31);
            const float *coll = ring + (size_t)((xl >> 5) % RING_NS) * rmax * 32 + (xl & 31);
            const float *tcol = tab + (cx - d2 - 1);
#pragma unroll 8
            for (int r = 0; r < 32; r++) {
                const int y = y0 + r;
                const int yc = y < h ? y : h - 1;
                const bool top = yc < d2 + 1, bottom = yc >= h - d2;
                const int jb = (bottom ? h - 1 : yc + d2) - yb0, jt = top ? 0 : yc - d2 - 1 - yb0;
                const float A = colr[jb * 32], B = coll[jb * 32], C = colr[jt * 32], Dd = coll[jt * 32];
                const float t1 = bottom ? C : B, t2 = bottom ? B : C;   // bottom band: A-C-B+D, elsewhere A-B-C+D
                const bool h1 = bottom ? !top : !left, h2 = bottom ? !left : !top;
                float v = A;
                v = h1 ? v - t1 : v;
                v = h2 ? v - t2 : v;
                v = (!top && !left) ? v + Dd : v;
                const int cy = top ? yc + d2 + 1 : (bottom ? h - yc + d2 : d);
                v = v * tcol[(cy - d2 - 1) * BOX_TAB_W];
                tile[r][lane] = (y < h && x < w) ? v : 0.f;
            }
        } else {
            const float *col = ring + (size_t)(t % RING_NS) * rmax * 32 + lane;
#pragma unroll 8
            for (int r = 0; r < 32; r++) {
                const float v = col[r * 32];
                tile[r][lane] = (y0 + r < h && x < w) ? v : 0.f;
            }
        }
        __syncwarp();
        // the chunk t-1 (AVG) / t (plain) is no longer needed: refill its slot with the chunk RING_NS-1 ahead
        issue_chunk(AVG ? t - 1 + RING_NS : t + RING_NS - 1);
        float *row = tile[lane];
#pragma unroll
        for (int cidx = 0; cidx < 32; cidx++) {
            carry = carry + row[cidx];  // I(x,y) = I(x-1,y) + in(x,y), iimage.cpp:56-60
            row[cidx] = carry;
        }
        __syncwarp();
        if (x < w) {
#pragma unroll 8
            for (int r = 0; r < 32; r++)
                if (y0 + r < h) O[(size_t)(y0 + r) * w + x] = tile[r][lane];
        }
        __syncwarp();
    }
    cp_async_wait<0>();
}

// ---------------------------------------------------------------------------------------------------
// Row pass on TMA tiles.  One warp = one 32-row band of one image (the sequential float add chain of iimage.cpp:56-60 runs
// along x, one row per lane), one warp per CTA so that the CTAs spread evenly over the SMs.  The cp.async ring version is
// warp-latency-bound (many instructions per 32 x 32 chunk, few warps active), not memory-bound; here a chunk costs ~80 (plain) / ~370 (box average) instructions:
//   * one lane issues one cp.async.bulk.tensor load per chunk on an mbarrier ring, RT_NS - 1 chunks ahead;
//   * the tile the scan walks row-wise lives in shared memory in the 128-byte swizzle of the tensor map, so that a lane reads
//     and writes its row as eight conflict-free 16-byte accesses (unit k of row r sits at unit k ^ (r & 7));
//   * the scanned tile leaves with one cp.async.bulk.tensor store; bounds are the tensor map's business (zero fill on the
//     way in, clipping on the way out).
// Same arithmetic and add order as k_rowscan (bit-identical output).
__device__ __forceinline__ unsigned int rt_s32(const void *p) { return (unsigned int)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void rt_load3(unsigned int dst, const CUtensorMap *tm, int x, int y, int z, unsigned int bar,
                                         unsigned int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(dst), "l"(tm), "r"(x), "r"(y), "r"(z), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void rt_store3(const CUtensorMap *tm, int x, int y, int z, unsigned int src) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(tm), "r"(x), "r"(y),
                 "r"(z), "r"(src)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ bool rt_wait(unsigned int bar, unsigned int parity, int *fail) {
    unsigned int ok = 0;
    const long long t0 = clock64();
    while (true) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) return true;
        if (clock64() - t0 > (1ll << 28)) {   // a broken copy flags an error instead of hanging the device
            *fail = 1;
            return false;
        }
    }
}
// in-place scan of a swizzled 32 x 32 tile (shared-space address), lane = row
__device__ __forceinline__ float rt_scan_tile(unsigned int tile_s, int lane, float carry) {
    const unsigned int rowp = tile_s + (unsigned int)((lane * 128) ^ ((lane & 7) << 4));
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const unsigned int a = rowp ^ (unsigned int)(k << 4);
        float4 v;
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
        carry = carry + v.x;   // I(x,y) = I(x-1,y) + in(x,y), iimage.cpp:56-60
        v.x = carry;
        carry = carry + v.y;
        v.y = carry;
        carry = carry + v.z;
        v.z = carry;
        carry = carry + v.w;
        v.w = carry;
        asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
    }
    return carry;
}

template <int RT_NS>
__global__ void __launch_bounds__(32) k_rowscan_tma_plain(const __grid_constant__ CUtensorMap tm_in,
                                                          const __grid_constant__ CUtensorMap tm_out, int w, int h,
                                                          int zin0, int *fail) {
    extern __shared__ unsigned char rt_raw[];
    unsigned char *base = rt_raw + ((1024u - (rt_s32(rt_raw) & 1023u)) & 1023u);   // 1024-byte aligned (swizzle atom)
    unsigned long long *full = reinterpret_cast<unsigned long long *>(base + RT_NS * 4096);
    const int lane = threadIdx.x;
    const int bands = (h + 31) >> 5;
    const int img = blockIdx.x / bands, band = blockIdx.x - img * bands;
    const int y0 = band * 32;
    const int nchunk = (w + 31) >> 5;
    const unsigned int ring_s = rt_s32(base), full_s = rt_s32(full);
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < RT_NS; k++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full_s + 8 * k) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#pragma unroll
        for (int ci = 0; ci < RT_NS - 1; ci++)
            if (ci < nchunk) rt_load3(ring_s + ci * 4096, &tm_in, 32 * ci, y0, zin0 + img, full_s + 8 * ci, 4096);
    }
    __syncwarp();
    float carry = 0.f;
    for (int t = 0; t < nchunk; t++) {
        const int slot = t % RT_NS;
        if (!rt_wait(full_s + 8 * slot, (unsigned int)(t / RT_NS) & 1u, fail)) break;
        carry = rt_scan_tile(ring_s + slot * 4096, lane, carry);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the TMA unit
        __syncwarp();
        if (lane == 0) {
            rt_store3(&tm_out, 32 * t, y0, img, ring_s + slot * 4096);
            // the slot of chunk t-1 (its store has been read out) takes the chunk RT_NS-1 ahead
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            const int cn = t + RT_NS - 1;
            if (cn < nchunk)
                rt_load3(ring_s + (cn % RT_NS) * 4096, &tm_in, 32 * cn, y0, zin0 + img, full_s + 8 * (cn % RT_NS), 4096);
        }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// Box average + row scan: chunk c of the input holds the columns [32c - 16, 32c + 16), so that the taps of the output tile t
// (columns [32t, 32t + 32), |offset| <= d2 + 1 <= 16) come from the chunks t and t+1 only: two chunks live, two in flight.
// Windows are (32 + d) x 32, read column-wise (lane = column, dense rows, no swizzle); the output tile is written column-wise
// into the swizzled layout and scanned in place.  (Output tiles shifted by 16 columns instead fault in the TMA store.)
template <int RT_NS>
__global__ void __launch_bounds__(32) k_rowscan_tma_avg(const __grid_constant__ CUtensorMap tm_in0,
                                                        const __grid_constant__ CUtensorMap tm_in1,
                                                        const __grid_constant__ CUtensorMap tm_out, int w, int h,
                                                        int in_mod, int nper, int d_f0, int d_f1,
                                                        const float *__restrict__ tab_f0, const float *__restrict__ tab_f1,
                                                        int rmax, int *fail) {
    extern __shared__ unsigned char rt_raw[];
    unsigned char *base = rt_raw + ((1024u - (rt_s32(rt_raw) & 1023u)) & 1023u);   // 1024-byte aligned (swizzle atom)
    unsigned char *otile = base;                                        // [2][4096]
    float *ring = reinterpret_cast<float *>(base + 2 * 4096);           // [RT_NS][rmax][32]
    unsigned long long *full = reinterpret_cast<unsigned long long *>(base + 2 * 4096 + (size_t)RT_NS * rmax * 128);
    float *tab = reinterpret_cast<float *>(full + RT_NS);
    const int lane = threadIdx.x;
    const int bands = (h + 31) >> 5;
    const int img = blockIdx.x / bands, band = blockIdx.x - img * bands;
    const bool f1 = (img / nper) != 0;
    const int d = f1 ? d_f1 : d_f0, d2 = d / 2;
    const int y0 = band * 32, yb0 = y0 - d2 - 1;    // image row of window row 0
    const int zin = img % in_mod;
    const CUtensorMap *tm = f1 ? &tm_in1 : &tm_in0;
    const unsigned int wbytes = (unsigned int)(32 + d) * 128u;
    const int ntile = (w + 31) >> 5, nchunk = (w + 16 + 31) >> 5;
    const unsigned int ring_s = rt_s32(ring), full_s = rt_s32(full), ot_s = rt_s32(otile);
    const unsigned int slot_bytes = (unsigned int)rmax * 128u;
    {
        const float *__restrict__ tg = f1 ? tab_f1 : tab_f0;
        tab[lane] = tg[lane];
        tab[lane + 32] = tg[lane + 32];
    }
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < RT_NS; k++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(full_s + 8 * k) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#pragma unroll
        for (int ci = 0; ci < RT_NS - 1; ci++)
            if (ci < nchunk) rt_load3(ring_s + ci * slot_bytes, tm, 32 * ci - 16, yb0, zin, full_s + 8 * ci, wbytes);
    }
    __syncwarp();
    const bool band_interior = (y0 >= d2 + 1) && (y0 + 31 < h - d2);
    // column-wise store offsets into the swizzled output tile: element (r, lane) at r * 128 + so[r & 7]
    unsigned int so[8];
#pragma unroll
    for (int j = 0; j < 8; j++) so[j] = (unsigned int)((((lane >> 2) ^ j) << 4) | ((lane & 3) << 2));
    float carry = 0.f;
    bool ok = rt_wait(full_s, 0u, fail);   // chunk 0
    for (int t = 0; ok && t < ntile; t++) {
        if (lane == 0) {
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // the store of tile t-2 has left its buffer
            const int cn = t + RT_NS - 1;                                     // the slot of chunk t-1 is free since tile t-1
            if (cn < nchunk)
                rt_load3(ring_s + (cn % RT_NS) * slot_bytes, tm, 32 * cn - 16, yb0, zin, full_s + 8 * (cn % RT_NS), wbytes);
        }
        if (t + 1 < nchunk && !rt_wait(full_s + 8 * ((t + 1) % RT_NS), (unsigned int)((t + 1) / RT_NS) & 1u, fail)) break;
        __syncwarp();
        unsigned char *ot = otile + (t & 1) * 4096;
        const int x = t * 32 + lane;
        if (band_interior && t * 32 >= d2 + 1 && t * 32 + 31 < w - d2) {
            // centre region of iimage::average for the whole tile: constant tap offsets, no selects
            const int xr = x + d2 + 16, xl = x - d2 - 1 + 16;   // (+16: chunk c starts at column 32c - 16)
            const float *colr = ring + (size_t)((xr >> 5) % RT_NS) * rmax * 32 + (xr & 31);
            const float *coll = ring + (size_t)((xl >> 5) % RT_NS) * rmax * 32 + (xl & 31);
            const float *colr_b = colr + d * 32, *coll_b = coll + d * 32;   // bottom taps: window row r + d
            const float a = tab[d2 * BOX_TAB_W + d2];
#pragma unroll
            for (int r = 0; r < 32; r++) {
                float v = colr_b[r * 32] - coll_b[r * 32];   // A - B
                v = v - colr[r * 32];                        //   - C
                v = v + coll[r * 32];                        //   + D
                *reinterpret_cast<float *>(ot + r * 128 + so[r & 7]) = v * a;
            }
        } else {
            // border tiles.  The dropped terms of iimage::average (left: B and D, top: C and D) are the taps that fall on
            // column / row -1, which the tensor map fills with +0: subtracting or adding +0 is the identity here (an
            // integral value is never -0: the add chains start from +0), so only the clamps (right, bottom), the bottom
            // band's term order and the clipped-area factor remain.
            const int xr = (x + d2 < w - 1 ? x + d2 : w - 1) + 16, xl = x - d2 - 1 + 16;
            const bool left = x < d2 + 1, right = x >= w - d2;
            int cxi = (left ? x + d2 + 1 : (right ? w - x + d2 : d)) - d2 - 1;
            cxi = cxi < 0 ? 0 : cxi;   // (columns >= w: clipped by the store)
            const float *colr = ring + (size_t)((xr >> 5) % RT_NS) * rmax * 32 + (xr & 31);
            const float *coll = ring + (size_t)((xl >> 5) % RT_NS) * rmax * 32 + (xl & 31);
            const float *tcol = tab + cxi;
            const int jbmax = h - 1 - yb0;
#pragma unroll
            for (int r = 0; r < 32; r++) {
                const int y = y0 + r;   // (warp-uniform row quantities)
                const bool top = y < d2 + 1, bottom = y >= h - d2;
                const int jb = r + d < jbmax ? r + d : jbmax;
                int cyi = (top ? y + d2 + 1 : (bottom ? h - y + d2 : d)) - d2 - 1;
                cyi = cyi < 0 ? 0 : cyi;   // (rows >= h: clipped by the store)
                const float A = colr[jb * 32], B = coll[jb * 32], C = colr[r * 32], Dd = coll[r * 32];
                const float t1 = bottom ? C : B, t2 = bottom ? B : C;   // bottom band: A-C-B+D, elsewhere A-B-C+D
                float v = A - t1;
                v = v - t2;
                v = v + Dd;
                *reinterpret_cast<float *>(ot + r * 128 + so[r & 7]) = v * tcol[cyi * BOX_TAB_W];
            }
        }
        __syncwarp();
        carry = rt_scan_tile(ot_s + (t & 1) * 4096, lane, carry);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0) rt_store3(&tm_out, 32 * t, y0, img, ot_s + (t & 1) * 4096);
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

static int rowscan_tma(rb_ctx *c, DogWS *ws, int stage, const float *in, int nimg, int in_mod, int nper) {
    const CUtensorMap *t = (const CUtensorMap *)ws->tmaps;
    const int bands = (c->h + 31) / 32;
    int *fail = (int *)((char *)c->dev_small + RB_DS_TMA_FAIL);
    const int ns_env = c->row_ns;
    if (stage < 0) {
        const int zin0 = (int)((in - ws->gray) / (ptrdiff_t)c->N);
        const int ns = ns_env ? ns_env : 4;
#define RT_PLAIN(NS) k_rowscan_tma_plain<NS><<<nimg * bands, 32, NS * 4096 + 64 + 1024, c->stream>>>(t[TM_GRAY], t[TM_S], c->w, c->h, zin0, fail)
        if (ns >= 8) RT_PLAIN(8);
        else if (ns >= 6) RT_PLAIN(6);
        else RT_PLAIN(4);
#undef RT_PLAIN
    } else {
        const int d0 = c->plan.d[0][stage], d1 = c->plan.d[1][stage];
        const int rmax = 32 + (d0 > d1 ? d0 : d1);
        const int ns = ns_env ? ns_env : 4;
#define RT_AVG(NS)                                                                                                              \
    k_rowscan_tma_avg<NS><<<nimg * bands, 32, 2 * 4096 + (size_t)NS * rmax * 128 + 64 + BOX_TAB_N * 4 + 1024, c->stream>>>(     \
        t[stage == 0 ? TM_I0_F0 : TM_I_F0], t[stage == 0 ? TM_I0_F1 : TM_I_F1], t[TM_S], c->w, c->h, in_mod, nper, d0, d1,       \
        c->boxtab + (0 * 3 + stage) * BOX_TAB_N, c->boxtab + (1 * 3 + stage) * BOX_TAB_N, rmax, fail)
        if (ns >= 6) RT_AVG(6);
        else if (ns >= 5) RT_AVG(5);
        else if (ns == 3) RT_AVG(3);
        else RT_AVG(4);
#undef RT_AVG
    }
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// per-device opt-ins of this file's kernels (function attributes are per device: called from rb_ctx_create after
// cudaSetDevice, so that contexts on several GPUs of one process all get them)
int rb_dog_device_setup(rb_ctx *c) {
    RB_CUDA(cudaFuncSetAttribute(k_rowscan_tma_avg<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    RB_CUDA(cudaFuncSetAttribute(k_rowscan_ring<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    RB_CUDA(cudaFuncSetAttribute(k_rowscan_ring<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return RB_OK;
}

static int rowscan_ring(rb_ctx *c, int stage, const float *in, float *out, int nimg, int in_mod, int nper) {
    const int bands = (c->h + 31) / 32;
    const int blocks = rb_div_up(nimg * bands, RING_WARPS);
    const int dmax = stage >= 0 ? (c->plan.d[0][stage] > c->plan.d[1][stage] ? c->plan.d[0][stage] : c->plan.d[1][stage]) : 0;
    const int rmax = 32 + dmax;
    const size_t smem = (size_t)RING_WARPS * (RING_NS * rmax * 32 + 32 * 33 + BOX_TAB_N) * sizeof(float);
    if (stage >= 0) {
        k_rowscan_ring<true><<<blocks, 32 * RING_WARPS, smem, c->stream>>>(
            in, out, c->w, c->h, nimg, in_mod, nper, c->plan.d[0][stage], c->plan.d[1][stage],
            c->boxtab + (0 * 3 + stage) * BOX_TAB_N, c->boxtab + (1 * 3 + stage) * BOX_TAB_N, rmax);
    } else {
        k_rowscan_ring<false><<<blocks, 32 * RING_WARPS, smem, c->stream>>>(in, out, c->w, c->h, nimg, in_mod, nper, 1, 1,
                                                                          nullptr, nullptr, rmax);
    }
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// stage < 0: plain row scan of the input; stage 0..1: row scan of box `stage` of both filters
static int rowscan(rb_ctx *c, DogWS *ws, int stage, const float *in, float *out, int nimg, int in_mod, int nper) {
    if (ws->tma_row_ok && out == ws->S && stage <= 1 && (ws->tma_row_mask == 1 || ws->tma_row_mask == (stage < 0 ? 2 : 3)) &&
        (stage < 0 ? (in >= ws->gray && in < ws->gray + (size_t)ws->B * c->N) : in == (stage == 0 ? ws->I0 : ws->I)))
        return rowscan_tma(c, ws, stage, in, nimg, in_mod, nper);
    if (c->rowscan_mode == 2) return rowscan_ring(c, stage, in, out, nimg, in_mod, nper);
    const int bands = (c->h + 31) / 32;
    const int warps = nimg * bands;
    const int blocks = rb_div_up(warps, 4);
    if (stage >= 0)
        k_rowscan<true><<<blocks, 128, 0, c->stream>>>(in, out, c->w, c->h, nimg, in_mod, nper, c->plan.d[0][stage],
                                                       c->plan.d[1][stage], c->boxtab + (0 * 3 + stage) * BOX_TAB_N,
                                                       c->boxtab + (1 * 3 + stage) * BOX_TAB_N);
    else
        k_rowscan<false><<<blocks, 128, 0, c->stream>>>(in, out, c->w, c->h, nimg, in_mod, nper, 1, 1, nullptr, nullptr);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

static int blur_dog(rb_ctx *c, DogWS *ws, int nimg, float *img1_opt, int out_slot = 0) {
    if (ws->tma_ok && !img1_opt) {
        const CUtensorMap *t = (const CUtensorMap *)ws->tmaps;
        dim3 tg(rb_div_up(c->w, BT_W), rb_div_up(c->h, BT_H), nimg);
        k_blur_dog_tma<<<tg, BT_THREADS, sizeof(BlurTmaSmem) + 128, c->stream>>>(
            t[TM_I_BLUR], t[TM_IMG0], t[TM_DOG], c->w, c->h, nimg, out_slot, c->plan.d[0][2], c->plan.d[1][2],
            c->boxtab + (0 * 3 + 2) * BOX_TAB_N, c->boxtab + (1 * 3 + 2) * BOX_TAB_N, (int *)((char *)c->dev_small + RB_DS_TMA_FAIL));
        RB_LAUNCH_CHECK();
        return RB_OK;
    }
    dim3 grid(rb_div_up(c->w, 256), rb_div_up(c->h, BLUR_RY), nimg);
    const size_t off = (size_t)out_slot * c->N;
    k_blur_dog<<<grid, 256, 0, c->stream>>>(ws->I, ws->img0 + off, ws->dog + off, img1_opt, c->w, c->h, nimg,
                                            c->plan.d[0][2],
                                            c->plan.d[1][2], c->boxtab + (0 * 3 + 2) * BOX_TAB_N,
                                            c->boxtab + (1 * 3 + 2) * BOX_TAB_N);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// reciprocal clipped-area tables of iimage::build_average for the six boxes of the plan (see box_avg)
int rb_dog_make_tables(rb_ctx *c) {
    float host[6 * BOX_TAB_N];
    for (int f = 0; f < 2; f++)
        for (int i = 0; i < 3; i++) {
            const int d = c->plan.d[f][i], d2 = d / 2;
            if (d2 + 1 > BOX_TAB_W) {
                snprintf(c->err, sizeof(c->err), "box width %d too large for this build", d);
                return RB_ERR_ARG;
            }
            float *t = host + (f * 3 + i) * BOX_TAB_N;
            for (int k = 0; k < BOX_TAB_N; k++) t[k] = 0.f;
            for (int cy = d2 + 1; cy <= d; cy++)
                for (int cx = d2 + 1; cx <= d; cx++) {
                    const float area = (float)(cx * cy);   // div(x,y)=cx*cy stored in a float image, then 1.0/div
                    t[(cy - d2 - 1) * BOX_TAB_W + (cx - d2 - 1)] = (float)(1.0 / (double)area);
                }
        }
    RB_CUDA(cudaMalloc(&c->boxtab, sizeof(host)));
    RB_CUDA(cudaMemcpy(c->boxtab, host, sizeof(host), cudaMemcpyHostToDevice));
    return RB_OK;
}

static int colscan(rb_ctx *c, const float *in, float *out, int nimg) {
    // default: float4 x 16 rows pipelined; REBVO_B200_COLSCAN=1: the unpipelined float4 x 16 loop
    const int mode = c->colscan_mode;
#define COL_PIPE(VW, U)                                                                                                \
    k_colscan_pipe<VW, U><<<rb_div_up(nimg * (c->w / VW), 64), 64, 0, c->stream>>>(                                      \
        (const ColVec<VW>::T *)in, (ColVec<VW>::T *)out, c->w / VW, c->h, nimg)
    if (mode != 1) COL_PIPE(4, 16);
    else {
        const int w4 = c->w / 4;
        const int threads = nimg * w4;
        k_colscan<<<rb_div_up(threads, 64), 64, 0, c->stream>>>((const float4 *)in, (float4 *)out, w4, c->h, nimg);
    }
#undef COL_PIPE
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// sspace::build for the m images [f0, f0 + m) of the workspace (gray already present): img0 / dog of those slots.  The
// intermediate planes (S, I0, I) are scratch shared by all ranges: ranges must not run concurrently.
int rb_dog_build_range(rb_ctx *c, DogWS *ws, int f0, int m) {
    if (f0 < 0 || m < 1 || f0 + m > ws->B) return RB_ERR_ARG;
    int r;
    const size_t N = c->N;
    // iimage::load(in): identical for both filters -> computed once
    if ((r = rowscan(c, ws, -1, ws->gray + f0 * N, ws->S, m, m, m))) return r;
    if ((r = colscan(c, ws->S, ws->I0, m))) return r;
    // box 0 of both filters reads the shared integral; image index = filter * m + b
    if ((r = rowscan(c, ws, 0, ws->I0, ws->S, 2 * m, m, m))) return r;
    if ((r = colscan(c, ws->S, ws->I, 2 * m))) return r;
    // box 1
    if ((r = rowscan(c, ws, 1, ws->I, ws->S, 2 * m, 2 * m, m))) return r;
    if ((r = colscan(c, ws->S, ws->I, 2 * m))) return r;
    // box 2 + DoG.  Filter f of image b lives at I[(f*m + b)*N]
    return blur_dog(c, ws, m, nullptr, f0);
}

// sspace::build for nimg images of the workspace (gray already present)
int rb_dog_build_batch(rb_ctx *c, DogWS *ws, int nimg) {
    if (nimg < 1 || nimg > ws->B) return RB_ERR_ARG;
    int r;
    // REBVO_B200_DOG_SUB: sub-batches whose intermediate planes (S, I0, I: 20 N bytes per frame) fit in L2 (50 MB on H100)
    // (the passes are latency-, not capacity-bound); default: the whole batch in one go
    const int sub = c->dog_sub > 0 ? c->dog_sub : nimg;
    for (int s = 0; s < nimg; s += sub)
        if ((r = rb_dog_build_range(c, ws, s, nimg - s < sub ? nimg - s : sub))) return r;
    return RB_OK;
}

// Img(1), dx, dy of image `img` into ws->aux (debug accessor; needs ws->I from the last build with
// the same nimg = ws_last_nimg, passed through B of the call: only valid for nimg == 1 workspaces)
int rb_dog_aux_planes(rb_ctx *c, DogWS *ws, int img) {
    if (ws->B != 1 || img != 0) return RB_ERR_ARG;
    int r = blur_dog(c, ws, 1, ws->aux);
    if (r) return r;
    dim3 grid(rb_div_up(c->w, 256), c->h, 1);
    k_gradient<<<grid, 256, 0, c->stream>>>(ws->img0, ws->aux + c->N, ws->aux + 2 * (size_t)c->N, c->w,
                                            c->h);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// measurement hook used by rb_pipeline_bench_pass
int rb_dog_single_pass(rb_ctx *c, DogWS *ws, int pass_id, int nimg, double *bytes) {
    const double N = (double)c->N;
    switch (pass_id) {
        case 0:
            *bytes = 8.0 * N * nimg;   // read gray 4N, write S 4N
            return rowscan(c, ws, -1, ws->gray, ws->S, nimg, nimg, nimg);
        case 1:
            *bytes = 8.0 * N * 2 * nimg;   // read I 4N (each tap row is re-used from L1/L2), write S 4N
            return rowscan(c, ws, 1, ws->I, ws->S, 2 * nimg, 2 * nimg, nimg);
        case 2:
            *bytes = 8.0 * N * 2 * nimg;   // read S 4N, write I 4N
            return colscan(c, ws->S, ws->I, 2 * nimg);
        case 3:
            *bytes = 16.0 * N * nimg;      // read I of both filters 8N, write img0 + dog 8N
            return blur_dog(c, ws, nimg, nullptr);
        case 4:
            *bytes = 7.0 * N * nimg;       // read RGB 3N, write gray 4N
            return rb_dog_gray(c, ws, nimg);
        case 6:
            *bytes = 5.0 * N * nimg;       // read mono N, write gray 4N
            return rb_dog_gray_mono(c, ws, nimg);
        default:
            return RB_ERR_ARG;
    }
}

// gray.cu -- the gray pass: a batch of pushed frames -> the float gray plane of the scale space.
//
// Image<float>::ConvertRGB2BW (image.h:197-203): gray = b + g + r as float; with UseUndistort=1 the pass is fused with
// image_undistort::undistort<true> (src/VideoLib/image_undistort.cpp, rebvo_first_t.cpp:231), see k_undistort_gray.
// Two kernel templates cover every input, k_gray<MONO, L> and k_undistort_gray<IMGS, MONO, L>:
//   MONO : RGB24 (3 bytes per pixel) or mono8.  A mono frame m stands for the RGB24 frame (m, m, m), so a pixel's b+g+r is
//          the integer 3v and the plane is bit-identical to the RGB pass's on the replicated frame.
//   L    : the layout of the frames, GrayLayout.
// rb_gray_enqueue is the one entry point: it picks the instance from the layout, the format and the undistortion map.
#include "common.cuh"
#include "undistort.cuh"

// GRAY_ALIGNED : packed frames (3N or N bytes each, back to back) of a width w % 4 == 0.  The plane is unpitched and the
//                frames are word-aligned whenever the source is.
// GRAY_ANYW    : packed frames of any width.  The plane has rows of `pitch` floats (DogWS), and a row -- and, past the first,
//                a frame -- starts at any byte offset, in the staging buffer (the rest of a head / rest push starts
//                mid-buffer) and in a caller's device buffer alike.
// GRAY_STRIDED : strided frames (rb_pipeline_push_frames_dev): frame f of the batch starts at frames[f].data and its rows are
//                frames[f].step bytes apart, each frame read where it is.  The plane is pitched as for GRAY_ANYW (pitch == w:
//                unpitched).
// The packed layouts read the batch through a device-resident pointer *src_pp, so that one captured graph serves whichever
// staging region / caller buffer a push uses (rb_pipeline).
enum GrayLayout { GRAY_ALIGNED, GRAY_ANYW, GRAY_STRIDED };

// A word of the word array p0 (a source rounded down to 4 bytes), of which only the bytes [lo, hi) may be read: loaded whole
// when it lies inside them, else assembled from its bytes that do -- no load touches a byte outside the frames.
__device__ __forceinline__ uint32_t frame_word(const uint8_t *__restrict__ p0, long long wi, long long lo, long long hi) {
    const long long b = 4 * wi;
    if (b >= lo && b + 4 <= hi) return __ldg(reinterpret_cast<const uint32_t *>(p0) + wi);
    uint32_t v = 0;
#pragma unroll
    for (int k = 0; k < 4; k++)
        if (b + k >= lo && b + k < hi) v |= (uint32_t)__ldg(p0 + b + k) << (8 * k);
    return v;
}

// the gray values of 4 RGB24 pixels held by 3 words:
// bytes: a = p0.0 p0.1 p0.2 p1.0 | b = p1.1 p1.2 p2.0 p2.1 | c = p2.2 p3.0 p3.1 p3.2
__device__ __forceinline__ float4 rgb_gray4(uint32_t a, uint32_t b, uint32_t c) {
    float4 o;
    o.x = (float)((a & 0xff) + ((a >> 8) & 0xff) + ((a >> 16) & 0xff));
    o.y = (float)((a >> 24) + (b & 0xff) + ((b >> 8) & 0xff));
    o.z = (float)(((b >> 16) & 0xff) + (b >> 24) + (c & 0xff));
    o.w = (float)(((c >> 8) & 0xff) + ((c >> 16) & 0xff) + (c >> 24));
    return o;
}
// the gray values of 4 mono8 pixels held by 1 word
__device__ __forceinline__ float4 mono_gray4(uint32_t a) {
    float4 o;
    o.x = (float)(3u * (a & 0xff));
    o.y = (float)(3u * ((a >> 8) & 0xff));
    o.z = (float)(3u * ((a >> 16) & 0xff));
    o.w = (float)(3u * (a >> 24));
    return o;
}

// the float4 of the nv (1..4) pixels whose first byte is t of the word array p0, of which the bytes [lo, hi) may be read:
// the aligned words that hold its 12 (RGB) / 4 (mono) source bytes, and funnel shifts
template <bool MONO>
__device__ __forceinline__ float4 gray4(const uint8_t *__restrict__ p0, long long t, int nv, long long lo, long long hi) {
    const int cb = MONO ? 1 : 3;   // bytes per pixel
    const long long wi = t >> 2, we = (t + cb * nv - 1) >> 2;   // first / last word holding a wanted byte
    const int sh = (int)(t & 3) * 8;
    float4 o;
    if (MONO) {
        const uint32_t w0 = frame_word(p0, wi, lo, hi), w1 = we > wi ? frame_word(p0, wi + 1, lo, hi) : 0u;
        o = mono_gray4(__funnelshift_r(w0, w1, sh));   // bytes t .. t+3
    } else {
        uint32_t wd[4];
#pragma unroll
        for (int k = 0; k < 4; k++) wd[k] = wi + k <= we ? frame_word(p0, wi + k, lo, hi) : 0u;
        o = rgb_gray4(__funnelshift_r(wd[0], wd[1], sh), __funnelshift_r(wd[1], wd[2], sh),
                      __funnelshift_r(wd[2], wd[3], sh));   // bytes t .. t+11
    }
    // pixels past w came from the next row's bytes (or zeros): the padding columns get +0
    if (nv < 4) {
        o.w = 0.f;
        if (nv < 3) o.z = 0.f;
        if (nv < 2) o.y = 0.f;
    }
    return o;
}

// 4 pixels per thread, one float4 of the plane.  The packed layouts read *src_pp, or src_fixed when src_pp is null.
//   GRAY_ALIGNED : float4 i of the n4 of the batch from 3 (RGB) / 1 (mono) aligned words; an RGB source that is not
//   4-byte aligned through gray4 instead.
//   GRAY_ANYW, GRAY_STRIDED : the float4 of 4 pixels of one pitched row (gray4, zeros in the padding columns).  Word indices
//   count from the batch's source (GRAY_ANYW) / the frame's own first byte (GRAY_STRIDED) rounded down to 4, and loads are
//   bounded by the batch's bytes / the frame's span [data, data + (h-1)*step + w*bpp): the row padding and the bytes around a
//   frame are never read.
template <bool MONO, GrayLayout L>
__global__ void __launch_bounds__(256) k_gray(const uint8_t *__restrict__ src_fixed, const uint8_t *const *__restrict__ src_pp,
                                              const rb_frame *__restrict__ frames, float4 *__restrict__ gray, size_t n4,
                                              int w, int h, int pitch, int nimg) {
    if constexpr (L == GRAY_ALIGNED) {
        size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
        if (i >= n4) return;
        const uint8_t *s = src_pp ? *src_pp : src_fixed;
        const uint32_t *__restrict__ src = reinterpret_cast<const uint32_t *>(s);
        if constexpr (MONO) {
            gray[i] = mono_gray4(src[i]);   // (rb_pipeline_push_mono_dev refuses sources that are not 4-byte aligned)
        } else if ((reinterpret_cast<uintptr_t>(s) & 3) == 0) {
            gray[i] = rgb_gray4(src[3 * i], src[3 * i + 1], src[3 * i + 2]);
        } else {
            // a caller's device buffer at any byte address (rb_pipeline_push_dev): the aligned words around the 12 bytes,
            // bounded by the batch's 12 * n4 bytes, as GRAY_ANYW reads them.  Decided here, per launch and warp-uniformly,
            // because one captured graph serves pushes whose sources differ in alignment.
            const uint8_t *p0 = reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(s) & ~(uintptr_t)3);
            const long long lo = (long long)(s - p0);
            gray[i] = gray4<false>(p0, lo + 12 * (long long)i, 4, lo, lo + 12 * (long long)n4);
        }
    } else {
        const int pv = pitch >> 2;
        const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // float4 of the pitched batch
        if (i >= (long long)nimg * h * pv) return;
        const int cb = MONO ? 1 : 3;   // bytes per pixel
        // (two bodies rather than one tail on (src, first byte, span): the shared form schedules the source load later and
        // compiles to other instructions)
        if constexpr (L == GRAY_ANYW) {
            const uint8_t *src = src_pp ? *src_pp : src_fixed;
            const uint8_t *p0 = reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(src) & ~(uintptr_t)3);
            const long long lo = (long long)(src - p0), hi = lo + (long long)nimg * cb * w * h;
            const long long row = i / pv;  // frame * h + y: frames are packed, so the pixel index of the row's start is row * w
            const int x = 4 * (int)(i - row * pv);
            const int nv = w - x < 4 ? w - x : 4;   // valid pixels of this float4 (1..4)
            gray[i] = gray4<MONO>(p0, lo + (long long)cb * (row * w + x), nv, lo, hi);
        } else {
            const long long row = i / pv;   // frame * h + y
            const int f = (int)(row / h), y = (int)(row - (long long)f * h);
            const int x = 4 * (int)(i - row * pv);
            const uint8_t *src = frames[f].data;
            const long long step = frames[f].step;
            const uint8_t *p0 = reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(src) & ~(uintptr_t)3);
            const long long lo = (long long)(src - p0), hi = lo + (long long)(h - 1) * step + (long long)cb * w;
            const int nv = w - x < 4 ? w - x : 4;
            gray[i] = gray4<MONO>(p0, lo + (long long)y * step + (long long)cb * x, nv, lo, hi);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Undistortion fused with the gray pass (rebvo_first_t.cpp:231 then sspace::build's first step): gray = float(r + g + b) of
// the undistorted pixel, whose channels are the integer bilinear sums >> 16 of biInterp (image_undistort.h:63-78).  The
// undistorted colour image itself is only consumed by the encoder / viewer (out of scope), so it is never materialised: per
// frame 3N (RGB) / N (mono) bytes in, 4N of gray out, the 32N-byte map stays L2-resident across the batch.
// The taps are gathered as aligned 32-bit words (a pixel's bytes start at any byte offset: two neighbouring words and a
// funnel shift; the two taps of a row are adjacent pixels almost everywhere, so three words (RGB) / one or two (mono) serve
// both) instead of a byte load per channel and tap, which bound the first version.
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
// GRAY_ALIGNED: the undistorted gray value of one pixel of the frame at src (N pixels).
// Mono: the RGB pass's three channel sums are all s = sum_k iw_k * m_k, so (u8)(r>>16) + (u8)(g>>16) + (u8)(b>>16) is
// 3 * (u8)(s>>16), with the same truncation.  One byte per tap; the two taps of a row in one aligned word, plus the next one
// only when the pair straddles a word boundary.  The source is 4-byte aligned (a frame is N bytes with N % 4 == 0, and
// rb_pipeline_push_mono_dev refuses unaligned buffers).
template <bool MONO>
__device__ __forceinline__ float ug_pixel(const uint8_t *__restrict__ src, const int4 ix, const int4 w, int N) {
    if constexpr (MONO) {
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
    } else {
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
            const int t[4] = {ix.x, ix.y, ix.z, ix.w}, ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const uint8_t *p = src + 3 * t[k];
                r += ww[k] * (int)p[0];
                g += ww[k] * (int)p[1];
                b += ww[k] * (int)p[2];
            }
        }
        const unsigned int s = (unsigned int)((uint8_t)(r >> 16)) + (unsigned int)((uint8_t)(g >> 16)) + (unsigned int)((uint8_t)(b >> 16));
        return (float)s;
    }
}
// GRAY_ANYW, GRAY_STRIDED: the four taps at bytes ofs[k] of the word array p0, of which the bytes [lo, hi) may be read (see
// frame_word); pairs: taps 0, 1 and taps 2, 3 are two runs of two adjacent pixels.  A mono pair's second byte is inside the
// frame, so when the pair straddles a word boundary its second word holds a byte of the frame.
template <bool MONO>
__device__ __forceinline__ float ug_taps(const uint8_t *__restrict__ p0, const long long ofs[4], bool pairs, long long lo,
                                         long long hi, const int4 w) {
    if constexpr (MONO) {
        int s;
        if (pairs) {
            s = 0;
#pragma unroll
            for (int row = 0; row < 2; row++) {
                const long long o = ofs[2 * row], wi = o >> 2;
                const unsigned int w0 = frame_word(p0, wi, lo, hi), w1 = (o & 3) == 3 ? frame_word(p0, wi + 1, lo, hi) : w0;
                const unsigned int v = __funnelshift_r(w0, w1, (int)(o & 3) * 8);   // bytes o, o + 1 in the low half
                s += (row ? w.z : w.x) * (int)(v & 0xffu) + (row ? w.w : w.y) * (int)((v >> 8) & 0xffu);
            }
        } else {
            s = w.x * (int)__ldg(p0 + ofs[0]) + w.y * (int)__ldg(p0 + ofs[1]) + w.z * (int)__ldg(p0 + ofs[2]) +
                w.w * (int)__ldg(p0 + ofs[3]);
        }
        return (float)(3u * (unsigned int)(uint8_t)(s >> 16));
    } else {
        int r = 0, g = 0, b = 0;
        if (pairs) {   // as ug_pixel
#pragma unroll
            for (int row = 0; row < 2; row++) {
                const long long o = ofs[2 * row], wi = o >> 2;
                const int sh = (int)(o & 3) * 8;
                const unsigned int w0 = frame_word(p0, wi, lo, hi), w1 = frame_word(p0, wi + 1, lo, hi),
                                   w2 = frame_word(p0, wi + 2, lo, hi);
                const unsigned int l = __funnelshift_r(w0, w1, sh), m = __funnelshift_r(w1, w2, sh);
                ug_acc(l, row ? w.z : w.x, r, g, b);
                ug_acc(__funnelshift_r(l, m, 24), row ? w.w : w.y, r, g, b);
            }
        } else {
            const int ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const long long wi = ofs[k] >> 2;
                ug_acc(__funnelshift_r(frame_word(p0, wi, lo, hi), frame_word(p0, wi + 1, lo, hi), (int)(ofs[k] & 3) * 8),
                       ww[k], r, g, b);
            }
        }
        const unsigned int s = (unsigned int)((uint8_t)(r >> 16)) + (unsigned int)((uint8_t)(g >> 16)) + (unsigned int)((uint8_t)(b >> 16));
        return (float)s;
    }
}
// GRAY_ANYW: the frame starts at byte t0 of the word array p0 (the batch's source rounded down to 4 bytes); cb bytes per pixel
template <bool MONO>
__device__ __forceinline__ float ug_pixel_any(const uint8_t *__restrict__ p0, long long t0, long long lo, long long hi,
                                              const int4 ix, const int4 w) {
    const int cb = MONO ? 1 : 3;
    const long long ofs[4] = {t0 + cb * ix.x, t0 + cb * ix.y, t0 + cb * ix.z, t0 + cb * ix.w};
    return ug_taps<MONO>(p0, ofs, ix.y == ix.x + 1 && ix.w == ix.z + 1, lo, hi, w);
}

// IMGS frames per thread: the 32-byte map entry of a pixel (L2-resident, but 739 MB of L2 reads per 64-frame launch when every
// frame fetches it again) is loaded once for IMGS frames.  taps: the map's inx, or for GRAY_STRIDED its ixy -- the packed
// indices split once into (x, y) when the map is built, so the kernel reads as many map bytes as the packed layouts and divides
// nothing; tap k of a frame is then at byte y*step + x*bpp of that frame, and the two-runs path needs the taps of a pair on one
// row.  GRAY_ANYW / GRAY_STRIDED write the pitched plane.
template <int IMGS, bool MONO, GrayLayout L>
__global__ void __launch_bounds__(256) k_undistort_gray(const uint8_t *const *__restrict__ src_pp,
                                                        const rb_frame *__restrict__ frames, float *__restrict__ gray,
                                                        const int4 *__restrict__ taps, const int4 *__restrict__ iw, int N,
                                                        int nimg, int wd, int pitch) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int img0 = blockIdx.y * IMGS;
    if (i >= N) return;
    const int cb = MONO ? 1 : 3;   // bytes per pixel
    float v[IMGS];
    if constexpr (L == GRAY_STRIDED) {
        const int4 xy = taps[i], w = iw[i];
        const int t[4] = {xy.x, xy.y, xy.z, xy.w};
        int tx[4], ty[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            tx[k] = t[k] & 0xffff;
            ty[k] = (int)((unsigned int)t[k] >> 16);
        }
        const bool pairs = ty[1] == ty[0] && tx[1] == tx[0] + 1 && ty[3] == ty[2] && tx[3] == tx[2] + 1;
        const int h = N / wd;
#pragma unroll
        for (int k = 0; k < IMGS; k++) {
            v[k] = 0.f;
            if (img0 + k >= nimg) continue;
            const uint8_t *src = frames[img0 + k].data;
            const long long step = frames[img0 + k].step;
            const uint8_t *p0 = reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(src) & ~(uintptr_t)3);
            const long long lo = (long long)(src - p0), hi = lo + (long long)(h - 1) * step + (long long)cb * wd;
            long long ofs[4];
#pragma unroll
            for (int j = 0; j < 4; j++) ofs[j] = lo + (long long)ty[j] * step + (long long)cb * tx[j];
            v[k] = ug_taps<MONO>(p0, ofs, pairs, lo, hi, w);
        }
    } else if constexpr (L == GRAY_ANYW) {
        // word indices count from the batch's source rounded down to 4 bytes; frame f starts at byte lo + f * cb * N
        const int4 ix = taps[i], w = iw[i];
        const uint8_t *src = *src_pp;
        const uint8_t *p0 = reinterpret_cast<const uint8_t *>(reinterpret_cast<uintptr_t>(src) & ~(uintptr_t)3);
        const long long lo = (long long)(src - p0), hi = lo + (long long)cb * N * nimg;
#pragma unroll
        for (int k = 0; k < IMGS; k++)
            v[k] = img0 + k < nimg ? ug_pixel_any<MONO>(p0, lo + (long long)cb * N * (img0 + k), lo, hi, ix, w) : 0.f;
    } else {
        const int4 ix = taps[i], w = iw[i];
        const uint8_t *src = *src_pp + (size_t)img0 * cb * N;
#pragma unroll
        for (int k = 0; k < IMGS; k++) v[k] = img0 + k < nimg ? ug_pixel<MONO>(src + (size_t)k * cb * N, ix, w, N) : 0.f;
    }
    const bool pitched = L != GRAY_ALIGNED;
    const int y = pitched ? i / wd : 0;
    const size_t o = pitched ? (size_t)y * pitch + (i - y * wd) : (size_t)i;   // gray[y * pitch + x]
    const size_t plane = pitched ? (size_t)pitch * (N / wd) : (size_t)N;
#pragma unroll
    for (int k = 0; k < IMGS; k++)
        if (img0 + k < nimg) gray[(size_t)(img0 + k) * plane + o] = v[k];
}

// ---------------------------------------------------------------------------------------------------
template <bool MONO, GrayLayout L>
static int gray_launch(rb_ctx *c, DogWS *ws, const rb_undistort *u, const uint8_t *const *src_pp, const rb_frame *frames,
                       int nimg) {
    if (!u) {
        const size_t n4 = (size_t)nimg * (L == GRAY_ALIGNED ? c->N : c->NP) / 4;
        k_gray<MONO, L><<<(unsigned)((n4 + 255) / 256), 256, 0, c->stream>>>(ws->rgb, src_pp, frames, (float4 *)ws->gray, n4,
                                                                             c->w, c->h, c->pitch, nimg);
    } else {
        const int4 *taps = L == GRAY_STRIDED ? u->ixy : u->inx;
        if (nimg >= 4)
            k_undistort_gray<4, MONO, L><<<dim3(rb_div_up(c->N, 256), rb_div_up(nimg, 4)), 256, 0, c->stream>>>(
                src_pp, frames, ws->gray, taps, u->iw, c->N, nimg, c->w, c->pitch);
        else
            k_undistort_gray<1, MONO, L><<<dim3(rb_div_up(c->N, 256), nimg), 256, 0, c->stream>>>(
                src_pp, frames, ws->gray, taps, u->iw, c->N, nimg, c->w, c->pitch);
    }
    RB_LAUNCH_CHECK();
    return RB_OK;
}

int rb_gray_enqueue(rb_ctx *c, DogWS *ws, const rb_undistort *und, bool mono, const void *const *src_pp,
                    const rb_frame *frames_dev, int nimg) {
    const uint8_t *const *pp = (const uint8_t *const *)src_pp;
    if (frames_dev)
        return (mono ? gray_launch<true, GRAY_STRIDED> : gray_launch<false, GRAY_STRIDED>)(c, ws, und, pp, frames_dev, nimg);
    if (und && !src_pp) return RB_ERR_ARG;   // (the undistorting kernels read the packed frames through src_pp only)
    if (c->pitch != c->w)
        return (mono ? gray_launch<true, GRAY_ANYW> : gray_launch<false, GRAY_ANYW>)(c, ws, und, pp, nullptr, nimg);
    return (mono ? gray_launch<true, GRAY_ALIGNED> : gray_launch<false, GRAY_ALIGNED>)(c, ws, und, pp, nullptr, nimg);
}

// detect.cu -- keyline extraction: edge_finder::detect (src/mtracklib/edge_finder.cpp:342-365) =
// UpdateThresh (:330-335) + build_mask (:67-214) + join_edges (:304-320), and reEstimateThresh (:373-405).
//
// The reference appends keylines in raster order and stops at kl_max.  Here:
//   k_update_thresh : the P-controller on the device-resident feedback state (no host round trip)
//   k_detect_a<R>   : all per-pixel tests in the (2R+1)^2 window of DetectorPlaneFitSize R = 1..4; candidates get
//                     mask=-2 and a float4 payload {m.x,m.y,xs,ys}; one warp owns a (row, 32-pixel) segment and writes
//                     its candidate count
//   k_seg_scan      : exclusive scan of the segment counts in raster order -> keyline ids, kn=min(total,kl_max)
//   k_detect_b      : ordered scatter of the keyline records (SoA) and of the id mask, cut at kl_max
//   k_join          : NextPoint/join_edges; "last writer wins" on p_id == atomicMax of the writer id
// Integer / float32 results are bit-identical to the reference; the plane fit is evaluated in
// float64 in the reference's summation order with contraction disabled.
#include "common.cuh"

// plane-fit pseudo inverses of every radius, packed at rb_pinv_offset(R) (capi.cu: plane_fit_tables)
__constant__ double c_pinv[RB_PINV_DOUBLES];

int rb_detect_upload_pinv(rb_ctx *c, const double *tab) {
    RB_CUDA(cudaMemcpyToSymbol(c_pinv, tab, sizeof(c_pinv)));
    return RB_OK;
}

// UpdateThresh (edge_finder.cpp:330-335) + the float casts build_mask receives (:349)
__global__ void k_update_thresh(DetChain *ch, MapState *st, double gain, int kl_ref, double tmax,
                                double tmin) {
    double t = ch->tresh;
    if (gain > 0) {
        t -= gain * (double)(kl_ref - ch->l_kl_num);
        t = t > tmax ? tmax : (t < tmin ? tmin : t);  // util::Constrain
        ch->tresh = t;
    }
    st->thresh_used = (float)t;
}

#define DET_BY 8
// grid: (ceil(w/32), ceil(h/DET_BY)), block (32, DET_BY).  R = DetectorPlaneFitSize (build_mask's win_s): a (2R+1)^2
// window, interior R <= x < w-R, R <= y < h-R (edge_finder.cpp:108-109)
template <int R>
__global__ void __launch_bounds__(32 * DET_BY) k_detect_a(const float *__restrict__ img0,
                                                          const float *__restrict__ dog,
                                                          int *__restrict__ mask,
                                                          float4 *__restrict__ cand,
                                                          int *__restrict__ seg_cnt,
                                                          const MapState *__restrict__ st, int w, int h,
                                                          int nchunk, float per_hist, float dog_thesh_f) {
    constexpr int NW = 2 * R + 1;                  // window width
    constexpr int TW = 32 + 2 * R, TH = DET_BY + 2 * R;
    constexpr int P0 = rb_pinv_offset(R), P1 = P0 + NW * NW, P2 = P1 + NW * NW;   // rows of PInv in c_pinv
    __shared__ float sd[TH][TW + 1];
    const int lane = threadIdx.x, ty = threadIdx.y;
    const int x0 = blockIdx.x * 32, y0 = blockIdx.y * DET_BY;
    // stage the DoG tile with an R-pixel halo
    for (int i = ty * 32 + lane; i < TH * TW; i += 32 * DET_BY) {
        const int r = i / TW, cc = i - r * TW;
        const int gx = x0 + cc - R, gy = y0 + r - R;
        sd[r][cc] = (gx >= 0 && gx < w && gy >= 0 && gy < h) ? dog[(size_t)gy * w + gx] : 0.f;
    }
    __syncthreads();
    const int x = x0 + lane, y = y0 + ty;
    if (y >= h) return;
    bool is_cand = false;
    float4 pay = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool interior = (x >= R && x < w - R && y >= R && y < h - R);
    if (interior) {
        const size_t idx = (size_t)y * w + x;
        const float grad_thesh = st->thresh_used;
        const float gx = img0[idx + 1] - img0[idx - 1];   // sspace::calc_gradient
        const float gy = img0[idx + w] - img0[idx - w];
        const float n2gI = gx * gx + gy * gy;             // util::norm2
        const float t1 = grad_thesh * (float)RB_MAX_IMG_VALUE;
        bool ok = !(n2gI < t1 * t1);                      // edge_finder.cpp:117-120
        if (ok) {
            int pn = 0;
#pragma unroll
            for (int i = 0; i < NW; i++)
#pragma unroll
                for (int j = 0; j < NW; j++) pn += (sd[ty + i][lane + j] > 0.f) ? 1 : -1;
            const float lim = (float)((2.0 * R + 1.0) * (2.0 * R + 1.0)) * per_hist;   // :137
            ok = !(fabs((double)pn) > (double)lim);       // :132
        }
        if (ok) {
            double th0 = 0.0, th1 = 0.0, th2 = 0.0;       // theta = PInv*Y, TooN dot: result=0; += a*b
#pragma unroll
            for (int i = 0; i < NW; i++)
#pragma unroll
                for (int j = 0; j < NW; j++) {
                    const double yv = (double)sd[ty + i][lane + j];
                    const int k = i * NW + j;
                    th0 = th0 + c_pinv[P0 + k] * yv;
                    th1 = th1 + c_pinv[P1 + k] * yv;
                    th2 = th2 + c_pinv[P2 + k] * yv;
                }
            const double den = th0 * th0 + th1 * th1;
            const float xs = (float)(-th0 * th2 / den);   // :146-147
            const float ys = (float)(-th1 * th2 / den);
            ok = !(fabsf(xs) > 0.5f || fabsf(ys) > 0.5f);  // :150
            if (ok) {
                const float mx = (float)th0, my = (float)th1;
                const float n2_m = mx * mx + my * my;
                const float t5 = t1 * dog_thesh_f;        // grad_thesh*max_img_value*dog_thesh
                ok = !(n2_m < t5 * t5);                   // :157-160
                if (ok) {
                    is_cand = true;
                    pay = make_float4(mx, my, xs, ys);
                }
            }
        }
        mask[idx] = is_cand ? -2 : -1;
        if (is_cand) cand[idx] = pay;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, is_cand);
    if (lane == 0) seg_cnt[y * nchunk + blockIdx.x] = __popc(bal);
}

// A detect with a wider window than the map's previous one: the pixels between the two margins leave the interior, and
// the narrower window may have left keyline ids there.  They become -1 like the rest of the border (edge_finder.cpp:39).
__global__ void k_mask_margin(int *__restrict__ mask, int w, int h, int r_old, int r_new) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * h) return;
    const int y = i / w, x = i - y * w;
    const int d = min(min(x, w - 1 - x), min(y, h - 1 - y));   // distance to the image border
    if (d >= r_old && d < r_new) mask[i] = -1;
}

// exclusive scan of nseg counts (raster order) by one block; kn = min(total, kl_max)
__global__ void __launch_bounds__(1024) k_seg_scan(int *__restrict__ seg, int nseg, MapState *st,
                                                   DetChain *ch, int kl_max) {
    __shared__ int warp_sum[32];
    __shared__ int base;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int per = (nseg + 1023) / 1024;
    const int b = tid * per, e = min(b + per, nseg);
    int s = 0;
    for (int i = b; i < e; i++) s += seg[i];
    int incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_sum[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int ws = warp_sum[lane];
        int wi = ws;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        warp_sum[lane] = wi - ws;  // exclusive over warps
        if (lane == 31) base = wi;
    }
    __syncthreads();
    int run = warp_sum[wid] + incl - s;
    for (int i = b; i < e; i++) {
        const int cnt = seg[i];
        seg[i] = run;
        run += cnt;
    }
    if (tid == 0) {
        const int total = base;
        int kn = total;
        if (kn > kl_max) kn = kl_max;   // build_mask stops when ++kn >= kl_max (:203)
        if (kn < 0) kn = 0;
        st->total_cand = total;
        st->kn = kn;
        st->nmatch = 0;
        if (ch) ch->l_kl_num = kn;      // detect(): l_kl_num = kn (:364)
    }
}

// warp per (row, chunk) segment: ordered scatter of keyline records
__global__ void __launch_bounds__(256) k_detect_b(int *__restrict__ mask, const float4 *__restrict__ cand,
                                                  const int *__restrict__ seg_off, KLSoA kl, int w, int h,
                                                  int nchunk, int kl_max, float ppx, float ppy, int border) {
    const int lane = threadIdx.x & 31;
    const int seg = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int y = seg / nchunk, ch = seg - y * nchunk;
    if (y < border || y >= h - border) return;
    const int x = ch * 32 + lane;
    const bool interior = (x >= border && x < w - border);
    const size_t idx = (size_t)y * w + x;
    const bool is_cand = interior && mask[idx] == -2;
    const unsigned bal = __ballot_sync(0xffffffffu, is_cand);
    if (!is_cand) return;
    const int id = seg_off[seg] + __popc(bal & ((1u << lane) - 1u));
    if (id >= kl_max) {   // past the cut: the reference never visits these pixels and clears the mask (:205-207)
        mask[idx] = -1;
        return;
    }
    const float4 p = cand[idx];
    const float mx = p.x, my = p.y;
    const float n2_m = mx * mx + my * my;
    const float n_m = sqrtf(n2_m);                       // :169
    const float ux = mx / n_m, uy = my / n_m;            // :170-171
    const float cx = (float)x + p.z, cy = (float)y + p.w;  // :173
    const float px = cx - ppx, py = cy - ppy;            // cam_model::Img2Hom
    mask[idx] = id;
    kl.p_inx[id] = (int)idx;
    kl.m_m[id] = make_float2(mx, my);
    kl.n_m[id] = n_m;
    kl.u_m[id] = make_float2(ux, uy);
    kl.c_p[id] = make_float2(cx, cy);
    kl.p_m[id] = make_float2(px, py);
    kl.p_m_0[id] = make_float2(px, py);
    kl.m_m0[id] = make_float2(0.f, 0.f);
    kl.n_m0[id] = 0.0;
    kl.rho[id] = RB_RHO_INIT;
    kl.s_rho[id] = RB_RHO_MAX;
    kl.rho0[id] = RB_RHO_INIT;
    kl.s_rho0[id] = RB_RHO_MAX;
    kl.m_num[id] = 0;
    kl.n_id[id] = -1;
    kl.p_id[id] = -1;
    kl.m_id[id] = -1;
    kl.m_id_f[id] = -1;
    kl.pack[2 * id] = make_float4(mx, my, cx, cy);
    kl.pack[2 * id + 1] = make_float4(ux, uy, n_m, 0.f);
}

// NextPoint (edge_finder.cpp:221-296) + join_edges (:304-320).
// A probe past the end of the mask counts as "no keyline".  With R = 1 a keyline on row h-2 (or column w-2) may sit
// exactly half a pixel further out: c_p rounds to row h-1 (column w-1), and a probe of the row below (of the next
// column on the last row) has index >= w*h.  The reference reads past its mask there (Image<int> is unchecked), so there
// is nothing defined to match; probes inside the image, including the row wrap at x = w-1, are the reference's.
// Probes never go below index 0: the rounded position is at least the keyline's own pixel, which is >= R >= 1.
__device__ __forceinline__ int probe(const int *__restrict__ mask, int i, int n) {
    return (unsigned)i < (unsigned)n ? mask[i] : -1;
}
__device__ __forceinline__ int next_point(int x, int y, float2 m, const int *__restrict__ mask, int w, int n) {
    const float tx = -m.y, ty = m.x;
    int k;
    const int sx = (ty > 0) ? (tx > 0 ? 1 : -1) : (tx < 0 ? -1 : 1);
    const int sy = (ty > 0) ? 1 : -1;
    if ((k = probe(mask, y * w + x + sx, n)) >= 0) return k;
    if ((k = probe(mask, (y + sy) * w + x, n)) >= 0) return k;
    if ((k = probe(mask, (y + sy) * w + x + sx, n)) >= 0) return k;
    return -1;
}

__global__ void __launch_bounds__(256) k_join(const int *__restrict__ mask, KLSoA kl,
                                              const MapState *__restrict__ st, int w, int h) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st->kn) return;
    const float2 cp = kl.c_p[i];
    const int x = (int)((double)cp.x + 0.5), y = (int)((double)cp.y + 0.5);  // util::round2int_positive: float+0.5 evaluates in double
    const int j = next_point(x, y, kl.m_m[i], mask, w, w * h);
    if (j < 0) return;
    atomicMax(&kl.p_id[j], i);   // sequential "kl[ikl2].p_id=ikl": the largest writer id survives
    kl.n_id[i] = j;
}

// ---- reEstimateThresh (edge_finder.cpp:373-405) ------------------------------------------------------
__global__ void k_reest_init(int *mm, int nh) {
    if (threadIdx.x == 0) {
        mm[0] = -1;          // max bits
        mm[1] = 0x7f7fffff;  // min bits (FLT_MAX)
    }
    for (int i = threadIdx.x; i < nh; i += blockDim.x) mm[2 + i] = 0;
}

__global__ void __launch_bounds__(256) k_nm_minmax(const float *__restrict__ n_m, MapState *st,
                                                   int *__restrict__ mm /* [2]: max bits, min bits */) {
    const int kn = st->kn;
    float mx = -1.f, mn = 3.4e38f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kn; i += gridDim.x * blockDim.x) {
        const float v = n_m[i];
        mx = fmaxf(mx, v);
        mn = fminf(mn, v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    }
    if ((threadIdx.x & 31) == 0 && mx >= 0.f) {  // n_m >= 0: the int order of the bit patterns is the float order
        atomicMax(&mm[0], __float_as_int(mx));
        atomicMin(&mm[1], __float_as_int(mn));
    }
}

__global__ void __launch_bounds__(256) k_nm_histo(const float *__restrict__ n_m, MapState *st,
                                                  const int *__restrict__ mm, int *__restrict__ histo,
                                                  unsigned int *ticket, int n, int knum) {
    extern __shared__ int sh[];
    const int kn = st->kn;
    for (int i = threadIdx.x; i < n; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const float max_dog = __int_as_float(mm[0]), min_dog = __int_as_float(mm[1]);
    const float range = max_dog - min_dog;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kn; i += gridDim.x * blockDim.x) {
        int b = (int)((float)n * (max_dog - n_m[i]) / range);   // :391
        b = b > n - 1 ? n - 1 : b;
        b = b < 0 ? 0 : b;
        atomicAdd(&sh[b], 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        if (sh[i]) atomicAdd(&histo[i], sh[i]);
    __threadfence();
    __shared__ bool last;
    if (threadIdx.x == 0) last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!last) return;
    __threadfence();
    for (int i = threadIdx.x; i < n; i += blockDim.x) sh[i] = __ldcg(&histo[i]);   // whole histogram in one go
    __syncthreads();
    if (threadIdx.x == 0) {
        float ret = 0.f;
        if (kn > 0) {
            int i = 0;
            // for(int a=0;i<n && a<knum;i++,a+=histo[i]);  -- skips bin 0, may index histo[n] (ignored: the
            // loop ends on i<n regardless)
            for (int a = 0; i < n && a < knum;) {
                i++;
                a += (i < n) ? sh[i] : 0;
            }
            ret = max_dog - (float)i * range / (float)n;   // :403
        }
        st->max_dog = max_dog;
        st->min_dog = min_dog;
        st->retuned = ret;
        *ticket = 0;
    }
    // leave the scratch ready for the next call (no separate init launch)
    for (int i = threadIdx.x; i < n + 1; i += blockDim.x) histo[i] = 0;
    if (threadIdx.x == 0) {
        const_cast<int *>(mm)[0] = -1;
        const_cast<int *>(mm)[1] = 0x7f7fffff;
    }
}

// ---------------------------------------------------------------------------------------------------
int rb_detect_enqueue(rb_ctx *c, rb_map *m, const float *img0, const float *dog,
                      const rb_detect_params *p, DetChain *chain_dev) {
    const int R = p->plane_fit_size;
    if (R < 1 || R > RB_PLANE_FIT_MAX) {   // (0: Phi^T Phi is singular)
        snprintf(c->err, sizeof(c->err), "DetectorPlaneFitSize must be 1..%d", RB_PLANE_FIT_MAX);
        return RB_ERR_ARG;
    }
    const int w = c->w, h = c->h;
    const int nchunk = rb_div_up(w, 32);
    int kl_max = p->kl_max > c->kcap ? c->kcap : p->kl_max;   // build_mask: kl_max>kl_size -> kl_size (:105)
    k_update_thresh<<<1, 1, 0, c->stream>>>(chain_dev, m->st, p->gain, p->kl_ref, p->thresh_max,
                                            p->thresh_min);
    RB_LAUNCH_CHECK();
    if (m->det_r > 0 && R > m->det_r) {
        k_mask_margin<<<rb_div_up(c->N, 256), 256, 0, c->stream>>>(m->mask, w, h, m->det_r, R);
        RB_LAUNCH_CHECK();
    }
    m->det_r = R;
    dim3 ga(nchunk, rb_div_up(h, DET_BY)), ba(32, DET_BY);
    // one instance per radius (k_detect_a<R> is only instantiated for R = 1..RB_PLANE_FIT_MAX)
    void (*const detect_a[RB_PLANE_FIT_MAX])(const float *, const float *, int *, float4 *, int *, const MapState *, int,
                                             int, int, float, float) = {k_detect_a<1>, k_detect_a<2>, k_detect_a<3>,
                                                                         k_detect_a<4>};
    detect_a[R - 1]<<<ga, ba, 0, c->stream>>>(img0, dog, m->mask, c->cand, c->seg_cnt, m->st, w, h, nchunk,
                                              (float)p->pos_neg_thresh, (float)p->dog_thresh);
    RB_LAUNCH_CHECK();
    const int nseg = h * nchunk;
    k_seg_scan<<<1, 1024, 0, c->stream>>>(c->seg_cnt, nseg, m->st, chain_dev, kl_max);
    RB_LAUNCH_CHECK();
    k_detect_b<<<rb_div_up(nseg, 8), 256, 0, c->stream>>>(m->mask, c->cand, c->seg_cnt, m->kl, w, h, nchunk,
                                                         kl_max, c->ppx, c->ppy, R);
    RB_LAUNCH_CHECK();
    k_join<<<rb_div_up(kl_max, 256), 256, 0, c->stream>>>(m->mask, m->kl, m->st, w, h);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

int rb_reestimate_enqueue(rb_ctx *c, rb_map *m, int knum, int nbins) {
    if (nbins < 1 || nbins > 4096) return RB_ERR_ARG;
    int *mm = (int *)c->dev_small;          // [0] max bits, [1] min bits, [2..] histogram
    int *histo = mm + 2;
    // mm / histogram are initialised at context creation and re-armed by k_nm_histo's last block
    const int blocks = 64;
    k_nm_minmax<<<blocks, 256, 0, c->stream>>>(m->kl.n_m, m->st, mm);
    RB_LAUNCH_CHECK();
    k_nm_histo<<<blocks, 256, sizeof(int) * nbins, c->stream>>>(m->kl.n_m, m->st, mm, histo, c->ticket, nbins,
                                                                knum);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

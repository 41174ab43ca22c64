// depth.cu -- the viewer's dense inverse-depth grid of one frame's net_keyline records, one CTA per fill:
//   d_filler.ResetData(); FillEdgeData(net_kl, kn, {0,0}, ThreshRelRho, ThreshMatchNum); InitCoarseFine();
//   Integrate(IterNum); computeDistance(Zeros)                  src/visualizer/visualizer.cpp:436-440
//   depth_filler(cam, {bw, bh}, BOUND_NONE)                      :303, src/visualizer/depth_filler.cpp
// Every product is the reference's double-precision expression sequence in the reference's order, so the grid is
// bit-identical (tests/test_gpu_depth_fill.py).  The one deviation: a record whose cell index is >= gw * gh (qy / bh >= gh)
// writes out of bounds in the reference (undefined behaviour); here it is dropped.
//
// Phases, separated by __syncthreads:
//   1. bucket the records by cell: warp-aggregated counts, a scan, a warp-aggregated scatter of (record index, rho, s_rho)
//      (global workspace), then each cell's short list sorted by record index -- FillEdgeData's order within a cell;
//   2. one thread per cell: the sequential information update of its records;
//   3. InitCoarseFine: under BOUND_NONE a tile mean reads only fixed cells and no level writes one, so every tile of every
//      level is independent: one thread per tile (the whole-grid tile, the longest serial chain, is tile 0 and starts
//      first), then each unfixed cell takes the mean of the finest level whose tile covers it and holds a fixed cell.
//      Integrate(init_cf = true) runs InitCoarseFine again, which is idempotent here;
//   4. Integrate1Step x iter_num, a skewed wavefront: cell (x, y) of sweep k runs at step x + 2y + 4k.  At that step
//      W/NW/N/NE hold their sweep-k values and E/SW/S/SE their sweep-(k-1) values, as in the raster-order Gauss-Seidel
//      loop, and no two cells of one step are neighbours: (gw-1) + 2(gh-1) + 4(iter_num-1) + 1 steps for all sweeps;
//   5. computeDistance(Zeros) / get3DPos, min_dist, and the cells written straight to their destination (mapped pinned
//      host memory in the pipeline).
// The grid (rho, s_rho, a fixed bit per cell, tile means) lives in shared memory when it fits (128x96 cells: ~221 KB),
// else in the global workspace with the same code: __syncthreads orders the CTA's global writes as well.
#include "depth.cuh"

#define NET_RHO_SCALING 10000.0   // include/CommLib/net_keypoint.h:32
#define DF_RHO_PRIOR 40.0         // RHO_MAX * 2 (depth_filler.cpp:47-49, RHO_MAX = 20 edge_finder.h:38)

__device__ __forceinline__ unsigned short rd16(const unsigned char *b) { return (unsigned short)(b[0] | (b[1] << 8)); }

// FillEdgeData's gates and cell index for record r (depth_filler.cpp:64-82); -1: skipped or dropped.  *rs = rho << 16 | s_rho
__device__ __forceinline__ int depth_key(const unsigned char *r, const DepthGeom &g, unsigned *rs) {
    const unsigned short qx = rd16(r), qy = rd16(r + 2), rh = rd16(r + 4), sr = rd16(r + 6);
    const unsigned char m_num = r[12];
    const double kl_rho = rh / NET_RHO_SCALING;
    const double kl_s_rho = sr / NET_RHO_SCALING;
    if (kl_s_rho / kl_rho > g.thresh_rel_rho) return -1;
    if (m_num < g.thresh_match_num) return -1;   // discart = true
    // data.GetIndex((qx + 0.f) / bl_size.w, (qy + 0.f) / bl_size.h): float quotients truncated to uint, y * w + x.  A record
    // in the remainder column lands in the first cell of the next row, as in the reference.
    const unsigned x = (unsigned)((float)qx / (float)(unsigned)g.bw);
    const unsigned y = (unsigned)((float)qy / (float)(unsigned)g.bh);
    const unsigned idx = y * (unsigned)g.gw + x;
    if (idx >= (unsigned)(g.gw * g.gh)) return -1;   // out of bounds in the reference: dropped
    *rs = ((unsigned)rh << 16) | sr;
    return (int)idx;
}

// One cell's list sorted by record index (the entries' high word; indices are distinct), by the cell's thread.  The scatter
// keeps lane order within a warp, so a list is made of a few sorted runs: insertion sort for the usual short list, heapsort
// (O(n log n) whatever the order) for a long one -- a cell holding most of a frame's records, when the block is about the
// frame's size.
#define DF_INSERTION_MAX 64
__device__ __forceinline__ void heap_sift(unsigned long long *a, int root, int n) {
    const unsigned long long v = a[root];
    for (;;) {
        int child = 2 * root + 1;
        if (child >= n) break;
        if (child + 1 < n && a[child + 1] > a[child]) child++;
        if (a[child] <= v) break;
        a[root] = a[child];
        root = child;
    }
    a[root] = v;
}
__device__ void sort_list(unsigned long long *a, int n) {
    if (n <= DF_INSERTION_MAX) {
        for (int i = 1; i < n; i++) {
            const unsigned long long v = a[i];
            int b = i - 1;
            while (b >= 0 && a[b] > v) {
                a[b + 1] = a[b];
                b--;
            }
            a[b + 1] = v;
        }
        return;
    }
    for (int r = n / 2 - 1; r >= 0; r--) heap_sift(a, r, n);
    for (int e = n - 1; e > 0; e--) {
        const unsigned long long t = a[0];
        a[0] = a[e];
        a[e] = t;
        heap_sift(a, 0, e);
    }
}

__global__ void __launch_bounds__(RB_DEPTH_THREADS, 1)
    k_depth_fill(const unsigned char *const *rec_pp, size_t rec_ofs, const unsigned char *rec_direct, const int *kn_p,
                 int kn_direct, int kcap, DepthGeom g, int *cnt, unsigned long long *list, unsigned char *gwork,
                 unsigned char *const *out_pp, size_t out_ofs, rb_depth_cell *out_direct, double2 *grid_out) {
    extern __shared__ __align__(16) unsigned char dsm[];
    __shared__ int s_part[32];
    __shared__ double s_min[32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nthr = blockDim.x;
    const int ncell = g.gw * g.gh, ncell32 = (ncell + 31) & ~31;
    int kn = kn_p ? *kn_p : kn_direct;
    kn = kn < 0 ? 0 : (kn > kcap ? kcap : kn);
    const unsigned char *rec = rec_pp ? rec_pp[0] + rec_ofs : rec_direct;
    unsigned char *wb = g.in_smem ? dsm : gwork;
    double *rho = reinterpret_cast<double *>(wb);
    double *srho = rho + ncell;
    double2 *tile = reinterpret_cast<double2 *>(srho + ncell);
    unsigned *fixbits = reinterpret_cast<unsigned *>(tile + g.ntiles);
    unsigned char *tile_ok = reinterpret_cast<unsigned char *>(fixbits + ncell32 / 32);
    const unsigned lt_mask = (1u << lane) - 1u;

    // ---- 1. bucket the records by cell, in record order within a cell
    for (int c = tid; c < ncell; c += nthr) cnt[c] = 0;
    __syncthreads();
    for (int j0 = 0; j0 < kn; j0 += nthr) {
        const int j = j0 + tid;
        unsigned rs = 0;
        const int key = j < kn ? depth_key(rec + (size_t)j * 15, g, &rs) : -1;
        const unsigned m = __match_any_sync(0xffffffffu, key);
        if (key >= 0 && lane == __ffs(m) - 1) atomicAdd(&cnt[key], __popc(m));
    }
    __syncthreads();
    {   // exclusive scan of cnt in place: thread t owns a contiguous chunk
        const int per = (ncell + nthr - 1) / nthr, a = tid * per, b = min(a + per, ncell);
        int s = 0;
        for (int c = a; c < b; c++) s += cnt[c];
        int incl = s;
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_part[wid] = incl;
        __syncthreads();
        if (wid == 0) {
            int v = lane < nthr / 32 ? s_part[lane] : 0;
            for (int o = 1; o < 32; o <<= 1) {
                const int u = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v += u;
            }
            s_part[lane] = v;
        }
        __syncthreads();
        int run = (wid ? s_part[wid - 1] : 0) + incl - s;
        for (int c = a; c < b; c++) {
            const int v = cnt[c];
            cnt[c] = run;
            run += v;
        }
    }
    __syncthreads();
    for (int j0 = 0; j0 < kn; j0 += nthr) {   // after this, cnt[c] is the end of cell c's list
        const int j = j0 + tid;
        unsigned rs = 0;
        const int key = j < kn ? depth_key(rec + (size_t)j * 15, g, &rs) : -1;
        const unsigned m = __match_any_sync(0xffffffffu, key);
        const int leader = __ffs(m) - 1;
        int base = 0;
        if (key >= 0 && lane == leader) base = atomicAdd(&cnt[key], __popc(m));
        base = __shfl_sync(m, base, leader);
        if (key >= 0) list[base + __popc(m & lt_mask)] = ((unsigned long long)j << 32) | rs;
    }
    __syncthreads();

    // ---- 2. ResetData + FillEdgeData: one thread per cell, its records in record order
    for (int c = tid; c < ncell32; c += nthr) {
        bool fixed = false;
        if (c < ncell) {
            const int lo = c ? cnt[c - 1] : 0, hi = cnt[c];
            sort_list(list + lo, hi - lo);
            double r = 1, I_rho = 1.0 / (DF_RHO_PRIOR * DF_RHO_PRIOR), s = DF_RHO_PRIOR;
            for (int a = lo; a < hi; a++) {
                const unsigned rs = (unsigned)list[a];
                const double kl_rho = (rs >> 16) / NET_RHO_SCALING;
                const double kl_s_rho = (rs & 0xffffu) / NET_RHO_SCALING;
                double i_rho = I_rho * r;
                const double kl_I_rho = 1 / (kl_s_rho * kl_s_rho);
                i_rho += kl_rho * kl_I_rho;
                I_rho += kl_I_rho;
                const double v_rho = I_rho > 0 ? 1.0 / I_rho : 1e20;
                r = i_rho * v_rho;
                s = sqrt(v_rho);
            }
            rho[c] = r;
            srho[c] = s;
            fixed = hi > lo;
        }
        const unsigned word = __ballot_sync(0xffffffffu, fixed);
        if (lane == 0) fixbits[c >> 5] = word;
    }
    __syncthreads();
#define DF_FIXED(c) ((fixbits[(c) >> 5] >> ((c) & 31)) & 1u)

    // ---- 3. InitCoarseFine (depth_filler.cpp:233-278): every tile of every level, sums dx outer, dy inner
    for (int t = tid; t < g.ntiles; t += nthr) {
        int l = 0;
        while (l + 1 < g.nlev && t >= g.loff[l + 1]) l++;
        const int sx = g.lsx[l], sy = g.lsy[l], k = t - g.loff[l];
        const int x0 = (k % g.lnx[l]) * sx, y0 = (k / g.lnx[l]) * sy;
        double mean_rho = 0, mean_srho = 0;
        int n = 0, nr = 0;
        for (int dx = 0; dx < sx; dx++)
            for (int dy = 0; dy < sy; dy++) {
                const int inx = (y0 + dy) * g.gw + x0 + dx;
                if (DF_FIXED(inx)) {
                    mean_rho += rho[inx];
                    mean_srho += srho[inx];
                    n++;
                    nr++;
                }
            }
        if (n > 0) {
            mean_rho /= n;
            mean_srho /= nr;
        }
        tile[t] = make_double2(mean_rho, mean_srho);
        tile_ok[t] = n > 0;
    }
    __syncthreads();
    for (int c = tid; c < ncell; c += nthr) {
        if (DF_FIXED(c)) continue;
        const int x = c % g.gw, y = c / g.gw;
        for (int l = g.nlev - 1; l >= 0; l--) {
            const int tx = x / g.lsx[l], ty = y / g.lsy[l];
            if (tx >= g.lnx[l] || ty >= g.lny[l]) continue;
            const int t = g.loff[l] + ty * g.lnx[l] + tx;
            if (!tile_ok[t]) continue;
            const double2 m = tile[t];
            rho[c] = m.x;
            srho[c] = m.y;   // !inboundary under BOUND_NONE
            break;
        }
    }
    __syncthreads();

    // ---- 4. Integrate1Step x iter_num (depth_filler.cpp:301-357) as one skewed wavefront
    if (g.iter_num > 0) {
        // one sweep spans steps 4k .. 4k + span; at step st only the sweeps with 0 <= st - 4k <= span have cells, so each
        // step visits at most (span / 4 + 1) * gh (sweep, row) pairs whatever iter_num is (64-bit step counter)
        const long long span = (long long)(g.gw - 1) + 2LL * (g.gh - 1);
        const long long steps = span + 4LL * (g.iter_num - 1) + 1;
        for (long long st = 0; st < steps; st++) {
            const long long k_lo = st > span ? (st - span + 3) / 4 : 0;
            const long long k_hi = min(st / 4, (long long)g.iter_num - 1);
            const int npairs = (int)(k_hi - k_lo + 1) * g.gh;   // (sweep, row) pairs; the step fixes the column
            for (int p = tid; p < npairs; p += nthr) {
                const int kk = p / g.gh, y = p - kk * g.gh;
                const long long xl = st - 2LL * y - 4 * (k_lo + kk);
                if (xl < 0 || xl >= g.gw) continue;
                const int x = (int)xl;
                const int inx = y * g.gw + x;
                if (DF_FIXED(inx)) continue;
                double r = 0, sr = 0;
                int n = 0;
                for (int dy = -1; dy <= 1; dy++)
                    for (int dx = -1; dx <= 1; dx++) {
                        if (dx == 0 && dy == 0) continue;
                        const int px = x + dx, py = y + dy;
                        if (px < 0 || px >= g.gw || py < 0 || py >= g.gh) continue;
                        r += rho[py * g.gw + px];
                        sr += srho[py * g.gw + px];
                        n++;
                    }
                const double w = 1;
                rho[inx] = (1 - w) * rho[inx] + w * r / n;
                srho[inx] = sr / n;
            }
            __syncthreads();
        }
    }

    // ---- 5. computeDistance(Zeros) (depth_filler.cpp:135-147) with get3DPos (depth_filler.h:115-122), min_dist
    rb_depth_cell *out = out_pp ? reinterpret_cast<rb_depth_cell *>(out_pp[1] + out_ofs) : out_direct;
    double dmin = 1e20;
    for (int c = tid; c < ncell; c += nthr) {
        const int x = c % g.gw, y = c / g.gw;
        // cam.Img2Hom<float>(x, y, ((float)i + 0.5) * bl_size.w, ...): a double product passed as float, minus pp in float
        const float ix = (float)(((float)x + 0.5) * (double)(unsigned)g.bw);
        const float iy = (float)(((float)y + 0.5) * (double)(unsigned)g.bh);
        const float hx = ix - g.ppx, hy = iy - g.ppy;
        const double r = rho[c];
        const double p0 = ((double)hx / g.zfm) / r, p1 = ((double)hy / g.zfm) / r, p2 = 1.0 / r;
        double nsq = 0;   // TooN::norm: sqrt of the dot product, summed from 0 in index order
        nsq += p0 * p0;
        nsq += p1 * p1;
        nsq += p2 * p2;
        const double d = sqrt(nsq);
        if (d < dmin) dmin = d;   // util::keep_min
        rb_depth_cell o;
        o.rho = r;
        o.s_rho = srho[c];
        o.dist = d;
        o.fixed = (int)DF_FIXED(c);
        o._pad = 0;
        out[c] = o;
        if (grid_out) grid_out[c] = make_double2(r, o.s_rho);   // for the image pass (k_depth_image) on the same stream
    }
#undef DF_FIXED
    for (int o = 16; o > 0; o >>= 1) {
        const double v = __shfl_down_sync(0xffffffffu, dmin, o);
        if (v < dmin) dmin = v;
    }
    if (lane == 0) s_min[wid] = dmin;
    __syncthreads();
    if (tid == 0) {
        double m = 1e20;
        for (int k = 0; k < nthr / 32; k++)
            if (s_min[k] < m) m = s_min[k];
        *reinterpret_cast<double *>(out + ncell) = m;
    }
}

int rb_depth_plan(rb_ctx *c, const rb_depth_params *p, DepthPlan *out) {
    if (!p || p->block_w < 1 || p->block_h < 1 || p->block_w > c->w || p->block_h > c->h || p->iter_num < 0) return RB_ERR_ARG;
    DepthGeom &g = out->g;
    memset(&g, 0, sizeof(g));
    g.bw = p->block_w;
    g.bh = p->block_h;
    g.gw = c->w / g.bw;
    g.gh = c->h / g.bh;
    g.thresh_rel_rho = p->thresh_rel_rho;
    g.thresh_match_num = p->thresh_match_num;
    g.iter_num = p->iter_num;
    g.ppx = c->ppx;
    g.ppy = c->ppy;
    g.zfm = c->zfm;
    // for (size_x = size.w, size_y = size.h; size_x > 1 && size_y > 1; size_x /= 2, size_y /= 2), tiles at x <= w - size_x
    for (int sx = g.gw, sy = g.gh; sx > 1 && sy > 1; sx /= 2, sy /= 2) {
        if (g.nlev == RB_DEPTH_MAX_LEVELS) return RB_ERR_ARG;
        g.lsx[g.nlev] = sx;
        g.lsy[g.nlev] = sy;
        g.lnx[g.nlev] = g.gw / sx;
        g.lny[g.nlev] = g.gh / sy;
        g.loff[g.nlev] = g.ntiles;
        g.ntiles += g.lnx[g.nlev] * g.lny[g.nlev];
        g.nlev++;
    }
    const size_t ncell = (size_t)g.gw * g.gh, ncell32 = (ncell + 31) & ~(size_t)31;
    out->grid_bytes = ncell * 16 + (size_t)g.ntiles * 16 + ncell32 / 8 + (((size_t)g.ntiles + 15) & ~(size_t)15);
    int optin = 0;
    RB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    cudaFuncAttributes fa;
    RB_CUDA(cudaFuncGetAttributes(&fa, k_depth_fill));
    const size_t max_dyn = (size_t)optin - fa.sharedSizeBytes;
    g.in_smem = out->grid_bytes <= max_dyn;
    out->dyn_smem = g.in_smem ? out->grid_bytes : 0;
    out->cells_bytes = ((ncell + 1) * sizeof(rb_depth_cell) + 255) & ~(size_t)255;
    // The attribute is one value per kernel and device, shared by every context and pipeline of the process: it is always set
    // to the device's whole opt-in budget, never to this plan's size, so no later plan can lower it under a pipeline whose
    // captured or eager launches need more.  (Concurrent calls write the same value.)
    if (g.in_smem)
        RB_CUDA(cudaFuncSetAttribute(k_depth_fill, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_dyn));
    return RB_OK;
}

// [cnt: ncell ints][list: kcap records][grid, when not in shared memory][final (rho, s_rho) per cell, for the image pass]
static size_t ws_cnt_bytes(const DepthPlan &pl) { return (((size_t)pl.g.gw * pl.g.gh) * sizeof(int) + 255) & ~(size_t)255; }
static size_t ws_list_bytes(int kcap) { return ((size_t)(kcap > 0 ? kcap : 1) * 8 + 255) & ~(size_t)255; }
static size_t ws_grid_bytes(const DepthPlan &pl) { return (pl.g.in_smem ? 0 : (pl.grid_bytes + 255) & ~(size_t)255); }
size_t rb_depth_ws_bytes(const DepthPlan &pl, int kcap) {
    return ws_cnt_bytes(pl) + ws_list_bytes(kcap) + ws_grid_bytes(pl) + (((size_t)pl.g.gw * pl.g.gh * 16 + 255) & ~(size_t)255);
}
double2 *rb_depth_ws_final(const DepthPlan &pl, int kcap, void *ws) {
    return (double2 *)((unsigned char *)ws + ws_cnt_bytes(pl) + ws_list_bytes(kcap) + ws_grid_bytes(pl));
}

int rb_depth_fill_enqueue(rb_ctx *c, const DepthPlan &pl, const unsigned char *const *rec_pp, size_t rec_ofs,
                          const unsigned char *rec, const int *kn_p, int kn, int kcap, void *ws,
                          unsigned char *const *out_pp, size_t out_ofs, rb_depth_cell *out, bool keep_final) {
    unsigned char *w = (unsigned char *)ws;
    int *cnt = (int *)w;
    unsigned long long *list = (unsigned long long *)(w + ws_cnt_bytes(pl));
    unsigned char *gwork = pl.g.in_smem ? nullptr : w + ws_cnt_bytes(pl) + ws_list_bytes(kcap);
    k_depth_fill<<<1, RB_DEPTH_THREADS, pl.dyn_smem, c->stream>>>(rec_pp, rec_ofs, rec, kn_p, kn, kcap, pl.g, cnt, list, gwork,
                                                                  out_pp, out_ofs, out,
                                                                  keep_final ? rb_depth_ws_final(pl, kcap, ws) : nullptr);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// ---- the dense inverse-depth image: depth_filler::getImgRho((float)x, (float)y, &s_rho) at every pixel (depth_filler.h:246-280)
// Each CTA stages the whole grid as float (rho, s_rho) pairs in shared memory (8 B per cell) when it fits, else reads the
// cells from global memory with the same code.  Thread t of the grid-stride loop computes 4 consecutive pixels of the
// row-major w x h plane (a quad may span two rows) and writes them as one 16-byte store per plane; the planes start on
// 16 bytes, so only a last partial quad (w * h not a multiple of 4) is written by scalar stores.
struct ImgAxis {   // the reference's expressions along one axis, for integer pixel coordinate v
    int f, c;
    float d;
};
__device__ __forceinline__ ImgAxis img_axis(int v, int b, int n) {
    // float x_histo = x / (float)bl_size.w - 0.5: a float quotient, the subtraction in double, stored as float
    const float hist = (float)((double)((float)v / (float)b) - 0.5);
    // int xf = std::min(std::max(floor(x_histo), 0.0), size.w - 1.0), xc likewise with ceil
    ImgAxis a;
    a.f = (int)fmin(fmax(floor((double)hist), 0.0), n - 1.0);
    a.c = (int)fmin(fmax(ceil((double)hist), 0.0), n - 1.0);
    a.d = hist - (float)a.f;   // float dx = x_histo - xf
    return a;
}
__device__ __forceinline__ float img_bilin(float v00, float v10, float v01, float v11, float dx, float dy) {
    // rho00*(1-dx)*(1-dy)+rho10*dx*(1-dy)+rho01*(1-dx)*dy+rho11*dx*dy, left to right in float (no contraction: -fmad=false)
    return v00 * (1 - dx) * (1 - dy) + v10 * dx * (1 - dy) + v01 * (1 - dx) * dy + v11 * dx * dy;
}

__global__ void __launch_bounds__(RB_DEPTH_IMG_THREADS)
    k_depth_image(const double *src, int stride, DepthImgGeom g, float *const *out_pp, size_t out_ofs, float *out_direct,
                  size_t plane_floats) {
    extern __shared__ __align__(16) float2 gsm[];
    const int ncell = g.gw * g.gh;
    if (g.in_smem) {
        for (int c = threadIdx.x; c < ncell; c += blockDim.x)
            gsm[c] = make_float2((float)src[(size_t)c * stride], (float)src[(size_t)c * stride + 1]);
        __syncthreads();
    }
    float *rho = out_pp ? reinterpret_cast<float *>(reinterpret_cast<unsigned char *>(out_pp[0]) + out_ofs) : out_direct;
    float *srho = g.planes == 2 ? rho + plane_floats : nullptr;
    const long long npx = (long long)g.w * g.h, nq = (npx + 3) >> 2;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += (long long)gridDim.x * blockDim.x) {
        const long long p0 = q << 2;
        int y = (int)(p0 / g.w), x = (int)(p0 - (long long)y * g.w);
        float r[4], s[4];
        ImgAxis ay = img_axis(y, g.bh, g.gh);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            r[k] = s[k] = 0.f;
            if (p0 + k < npx) {
                const ImgAxis ax = img_axis(x, g.bw, g.gw);
                const int i00 = ay.f * g.gw + ax.f, i10 = ay.f * g.gw + ax.c, i01 = ay.c * g.gw + ax.f, i11 = ay.c * g.gw + ax.c;
                float2 c00, c10, c01, c11;
                if (g.in_smem) {
                    c00 = gsm[i00], c10 = gsm[i10], c01 = gsm[i01], c11 = gsm[i11];
                } else {
                    c00 = make_float2((float)src[(size_t)i00 * stride], (float)src[(size_t)i00 * stride + 1]);
                    c10 = make_float2((float)src[(size_t)i10 * stride], (float)src[(size_t)i10 * stride + 1]);
                    c01 = make_float2((float)src[(size_t)i01 * stride], (float)src[(size_t)i01 * stride + 1]);
                    c11 = make_float2((float)src[(size_t)i11 * stride], (float)src[(size_t)i11 * stride + 1]);
                }
                r[k] = img_bilin(c00.x, c10.x, c01.x, c11.x, ax.d, ay.d);
                if (srho) s[k] = img_bilin(c00.y, c10.y, c01.y, c11.y, ax.d, ay.d);
            }
            if (++x == g.w) {
                x = 0;
                ay = img_axis(++y, g.bh, g.gh);
            }
        }
        if (p0 + 4 <= npx) {
            *reinterpret_cast<float4 *>(rho + p0) = make_float4(r[0], r[1], r[2], r[3]);
            if (srho) *reinterpret_cast<float4 *>(srho + p0) = make_float4(s[0], s[1], s[2], s[3]);
        } else {
#pragma unroll
            for (int k = 0; k < 4; k++) {
                if (p0 + k >= npx) break;
                rho[p0 + k] = r[k];
                if (srho) srho[p0 + k] = s[k];
            }
        }
    }
}

int rb_depth_image_plan(rb_ctx *c, const DepthGeom &fg, int planes, DepthImgPlan *out) {
    DepthImgGeom &g = out->g;
    g.w = c->w;
    g.h = c->h;
    g.gw = fg.gw;
    g.gh = fg.gh;
    g.bw = fg.bw;
    g.bh = fg.bh;
    g.planes = planes;
    const size_t need = (size_t)g.gw * g.gh * sizeof(float2);
    int optin = 0;
    RB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device));
    cudaFuncAttributes fa;
    RB_CUDA(cudaFuncGetAttributes(&fa, k_depth_image));
    const size_t max_dyn = (size_t)optin - fa.sharedSizeBytes;
    g.in_smem = need <= max_dyn;
    out->dyn_smem = g.in_smem ? need : 0;
    // one value per kernel and device for the whole process: always the device's whole opt-in budget (as k_depth_fill's)
    if (g.in_smem)
        RB_CUDA(cudaFuncSetAttribute(k_depth_image, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_dyn));
    // one CTA per SM at most: each CTA stages the whole grid, and the pass is bound by its stores, not by its arithmetic
    const long long nq = ((long long)g.w * g.h + 3) / 4;
    const long long ctas = (nq + RB_DEPTH_IMG_THREADS - 1) / RB_DEPTH_IMG_THREADS;
    out->ctas = (int)(ctas < c->sm_count ? ctas : c->sm_count);
    return RB_OK;
}

int rb_depth_image_enqueue(rb_ctx *c, const DepthImgPlan &ip, const double *src, int stride, float *const *out_pp,
                           size_t out_ofs, float *out, size_t plane_floats) {
    k_depth_image<<<ip.ctas, RB_DEPTH_IMG_THREADS, ip.dyn_smem, c->stream>>>(src, stride, ip.g, out_pp, out_ofs, out,
                                                                             plane_floats);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// the stage call: records from host memory, the grid back to host memory; the context's scratch grows to the largest call
extern "C" int rb_depth_fill_net(rb_ctx *c, const void *records, int n, const rb_depth_params *p, rb_depth_cell *out,
                                 int *gw, int *gh, double *min_dist) {
    if (!c || n < 0 || (n > 0 && !records) || !p || !out) return RB_ERR_ARG;
    RB_ENTER(c);
    DepthPlan pl;
    int r = rb_depth_plan(c, p, &pl);
    if (r) return r;
    const size_t ncell = (size_t)pl.g.gw * pl.g.gh;
    const size_t rec_bytes = ((size_t)n * 15 + 255) & ~(size_t)255;
    const size_t need = rec_bytes + pl.cells_bytes + rb_depth_ws_bytes(pl, n);
    if (need > c->depth_ws_bytes) {
        cudaFree(c->depth_ws);
        c->depth_ws = nullptr;
        c->depth_ws_bytes = 0;
        RB_CUDA(cudaMalloc(&c->depth_ws, need));
        c->depth_ws_bytes = need;
    }
    unsigned char *recd = (unsigned char *)c->depth_ws;
    rb_depth_cell *cells = (rb_depth_cell *)(recd + rec_bytes);
    if (n > 0) RB_CUDA(cudaMemcpyAsync(recd, records, (size_t)n * 15, cudaMemcpyHostToDevice, c->stream));
    if ((r = rb_depth_fill_enqueue(c, pl, nullptr, 0, recd, nullptr, n, n, (unsigned char *)cells + pl.cells_bytes, nullptr, 0,
                                   cells, false)))
        return r;
    RB_CUDA(cudaMemcpyAsync(out, cells, ncell * sizeof(rb_depth_cell), cudaMemcpyDeviceToHost, c->stream));
    double md = 0;
    RB_CUDA(cudaMemcpyAsync(&md, cells + ncell, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    if (gw) *gw = pl.g.gw;
    if (gh) *gh = pl.g.gh;
    if (min_dist) *min_dist = md;
    return RB_OK;
}

// the stage call: cells from host memory (those rb_depth_fill_net / rb_pipeline_depth return), the planes back to host memory.
// The kernel reads the uploaded cells in place: rho and s_rho are the first two of each cell's four doubles.
static_assert(offsetof(rb_depth_cell, s_rho) == sizeof(double) && sizeof(rb_depth_cell) == 4 * sizeof(double),
              "rb_depth_cell: rho, s_rho, then two more doubles' worth");
extern "C" int rb_depth_image(rb_ctx *c, const rb_depth_cell *cells, int gw, int gh, const rb_depth_params *p, float *rho,
                              float *s_rho) {
    if (!c || !cells || !p || !rho) return RB_ERR_ARG;
    RB_ENTER(c);
    DepthPlan pl;
    int r = rb_depth_plan(c, p, &pl);
    if (r) return r;
    if (gw != pl.g.gw || gh != pl.g.gh) return RB_ERR_ARG;
    DepthImgPlan ip;
    if ((r = rb_depth_image_plan(c, pl.g, s_rho ? 2 : 1, &ip))) return r;
    const size_t ncell = (size_t)gw * gh, plane = ((size_t)c->N + 63) & ~(size_t)63;
    const size_t cells_bytes = (ncell * sizeof(rb_depth_cell) + 255) & ~(size_t)255;
    const size_t need = cells_bytes + 2 * plane * sizeof(float);
    if (need > c->depth_ws_bytes) {
        cudaFree(c->depth_ws);
        c->depth_ws = nullptr;
        c->depth_ws_bytes = 0;
        RB_CUDA(cudaMalloc(&c->depth_ws, need));
        c->depth_ws_bytes = need;
    }
    unsigned char *celld = (unsigned char *)c->depth_ws;
    float *img = (float *)(celld + cells_bytes);
    RB_CUDA(cudaMemcpyAsync(celld, cells, ncell * sizeof(rb_depth_cell), cudaMemcpyHostToDevice, c->stream));
    if ((r = rb_depth_image_enqueue(c, ip, (const double *)celld, (int)(sizeof(rb_depth_cell) / sizeof(double)), nullptr, 0,
                                    img, plane)))
        return r;
    RB_CUDA(cudaMemcpyAsync(rho, img, (size_t)c->N * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    if (s_rho) RB_CUDA(cudaMemcpyAsync(s_rho, img + plane, (size_t)c->N * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    return RB_OK;
}

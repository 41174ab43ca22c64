// tracker.cu -- edge-map tracker and mapper kernels:
//   global_tracker::build_field / TryVelRot / Minimizer_RV   (src/mtracklib/global_tracker.cpp)
//   edge_tracker::EstimateQuantile / FordwardMatch / rotate_keylines / directed_matching+search_match /
//   Regularize_1_iter / UpdateInverseDepthKalman(ARLU) / EstimateReScalingOpt (src/mtracklib/edge_tracker.cpp)
//
// Per-keyline arithmetic follows the reference expression by expression in float64 (float32 where the
// reference's operands are float) with contraction disabled (-fmad=false).  Sums over keylines (JtJ, JtF,
// score, rescaling) use a fixed-order warp-shuffle / block / grid reduction: deterministic, but not the
// reference's pairwise tree, so they agree to rounding (tests use rel 1e-11), not bitwise.
#include "tracker.cuh"
#include "lm.cuh"
#include "frame.cuh"

#define TVR_T 256
#define RES_SENTINEL 0x7FF8DEADBEEF0001ull

// Cycle stamps of one evaluation kernel (build with -DRB_TVR_PROF, see scratch tooling); compiled out of the product.
#ifdef RB_TVR_PROF
__device__ long long g_tvr_prof[256 * 16];
#define TVR_STAMP(k) do { if (threadIdx.x == 0) g_tvr_prof[blockIdx.x * 16 + (k)] = clock64(); } while (0)
__device__ __forceinline__ long long tvr_gtime() {
    long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
#define TVR_GSTAMP(k) do { if (threadIdx.x == 0) g_tvr_prof[blockIdx.x * 16 + (k)] = tvr_gtime(); } while (0)
extern "C" int rb_debug_fetch(long long *out) {
    return (int)cudaMemcpyFromSymbol(out, g_tvr_prof, sizeof(long long) * 256 * 16);
}
#else
#define TVR_STAMP(k) do { } while (0)
#define TVR_GSTAMP(k) do { } while (0)
#endif

struct CamC {
    double zfm, inv_zf;
    float ppx, ppy;
    int w, h;
};

static CamC make_cam(const rb_ctx *c) {
    CamC k;
    k.zfm = c->zfm;
    k.inv_zf = 1 / c->zfm;
    k.ppx = c->ppx;
    k.ppy = c->ppy;
    k.w = c->w;
    k.h = c->h;
    return k;
}

int rb_track_state_alloc(rb_ctx *c, rb_map *m) {
    TrackState host;
    memset(&host, 0, sizeof(host));
    const int nblk = rb_div_up(c->kcap, TVR_T);
    const size_t K = c->kcap + 32;
    host.nblk = nblk;
    RB_CUDA(cudaMalloc(&host.blk_has, sizeof(int) * nblk));
    RB_CUDA(cudaMalloc(&host.blk_last_fi, sizeof(double) * nblk));
    RB_CUDA(cudaMalloc(&host.partials, sizeof(double) * 28 * TVR_T));
    RB_CUDA(cudaMalloc(&host.carry, sizeof(double) * 3 * TVR_T));
    RB_CUDA(cudaMemsetAsync(host.carry, 0, sizeof(double) * 3 * TVR_T, c->stream));
    RB_CUDA(cudaMalloc(&host.ctl, sizeof(MinCtl)));
    RB_CUDA(cudaMemsetAsync(host.ctl, 0, sizeof(MinCtl), c->stream));
    // slots of the multi-cluster minimiser: [2][MC_GMAX][16][2][64]
    RB_CUDA(cudaMalloc(&host.ll, sizeof(unsigned long long) * 2 * 8 * 16 * 2 * 64));
    RB_CUDA(cudaMemsetAsync(host.ll, 0, sizeof(unsigned long long) * 2 * 8 * 16 * 2 * 64, c->stream));
    RB_CUDA(cudaMalloc(&host.fm_best, sizeof(FmBest) * K));
    RB_CUDA(cudaMalloc(&host.reg_r, sizeof(double) * K));
    RB_CUDA(cudaMalloc(&host.reg_s, sizeof(double) * K));
    RB_CUDA(cudaMalloc(&host.reg_set, K));
    RB_CUDA(cudaMalloc(&m->ts, sizeof(TrackState)));
    RB_CUDA(cudaMemcpyAsync(m->ts, &host, sizeof(host), cudaMemcpyHostToDevice, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    m->ts_host = host;
    return RB_OK;
}

void rb_track_state_free(rb_map *m) {
    TrackState &h = m->ts_host;
    cudaFree(h.blk_has);
    cudaFree(h.blk_last_fi);
    cudaFree(h.partials);
    cudaFree(h.carry);
    cudaFree(h.ctl);
    cudaFree(h.ll);
    cudaFree(h.fm_best);
    cudaFree(h.reg_r);
    cudaFree(h.reg_s);
    cudaFree(h.reg_set);
    cudaFree(m->ts);
}

// =====================================================================================================
// EstimateQuantile (edge_tracker.cpp:1148-1186)
// =====================================================================================================
__global__ void __launch_bounds__(256) k_quantile(const double *__restrict__ s_rho, MapState *st,
                                                  int *__restrict__ histo, unsigned int *ticket, double smin,
                                                  double smax, double perc, int n, FrameState *fs,
                                                  const unsigned int *frame_count, MapState *nst) {
    pdl_wait();
    pdl_launch();
    extern __shared__ int sh[];
    if (fs && blockIdx.x == 0 && threadIdx.x == 0) d_frame_pre(fs, *frame_count, nst);   // folded one-thread stage
    const int kn = st->kn;
    for (int i = threadIdx.x; i < n; i += blockDim.x) sh[i] = 0;
    __syncthreads();
    const double range = smax - smin;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kn; i += gridDim.x * blockDim.x) {
        int b = (int)((double)n * (s_rho[i] - smin) / range);
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
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        sh[i] = __ldcg(&histo[i]);
        histo[i] = 0;   // leave the scratch histogram zeroed for the next call
    }
    __syncthreads();
    // "for i: if (a > perc * kn) {q = bin i; break;} a += histo[i]" = the first bin whose exclusive prefix sum exceeds the
    // threshold: one warp, 4 bins per lane, shuffle scan (instead of a serial loop at the end of every frame's first kernel)
    if (threadIdx.x < 32 && n <= 128) {
        const int lane = threadIdx.x;
        int b[4], tot = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            b[k] = 4 * lane + k < n ? sh[4 * lane + k] : 0;
            tot += b[k];
        }
        int incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        int a = incl - tot, hit = -1;   // exclusive prefix of this lane's first bin
        const double thr = perc * (double)kn;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (hit < 0 && 4 * lane + k < n && (double)a > thr) hit = 4 * lane + k;
            a += b[k];
        }
        const unsigned int m = __ballot_sync(0xffffffffu, hit >= 0);
        const int first = m ? __shfl_sync(0xffffffffu, hit, __ffs(m) - 1) : -1;
        if (lane == 0) {
            st->s_rho_q = first >= 0 ? (double)first * range / (double)n + smin : 1e3;
            *ticket = 0;
        }
    } else if (threadIdx.x == 0 && n > 128) {
        double q = 1e3;
        for (int i = 0, a = 0; i < n; i++) {
            if ((double)a > perc * (double)kn) {
                q = (double)i * range / (double)n + smin;
                break;
            }
            a += sh[i];
        }
        st->s_rho_q = q;
        *ticket = 0;
    }
}

int rb_quantile_enqueue(rb_ctx *c, rb_map *m, double smin, double smax, double perc, int nbins, FrameState *fs,
                        const unsigned int *frame_count_dev, MapState *nst) {
    if (nbins < 1 || nbins > 4096) return RB_ERR_ARG;
    int *histo = (int *)((char *)c->dev_small + RB_DS_QHISTO);  // zeroed at creation and by the kernel's tail
    RB_KLAUNCH(k_quantile, 64, 256, sizeof(int) * nbins, m->kl.s_rho, m->st, histo, c->ticket + 2, smin, smax, perc,
               nbins, fs, frame_count_dev, nst);
    return RB_OK;
}

// =====================================================================================================
// build_field (global_tracker.cpp:61-105): winner per pixel = smallest |t|, ties -> larger keyline id,
// i.e. atomicMin of (|t| << 32 | ~ikl).  ~0 = no entry.
// =====================================================================================================
__global__ void __launch_bounds__(256) k_build_field(unsigned long long *__restrict__ field, KLSoA kl,
                                                     const MapState *__restrict__ st, int radius, float min_mod_v,
                                                     int min_mod_from_state, int w, int h) {
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int span = 2 * radius;
    const int ikl = (int)(gid / span);
    if (ikl >= st->kn) return;
    const int t = (int)(gid - (long long)ikl * span) - radius;   // t in [-radius, radius)
    const float min_mod = min_mod_from_state ? st->retuned : min_mod_v;
    if (min_mod > 0 && kl.n_m[ikl] < min_mod) return;
    const float2 u = kl.u_m[ikl], cp = kl.c_p[ikl];
    const float fx = u.x * (float)t + cp.x, fy = u.y * (float)t + cp.y;
    const int xi = (int)roundf(fx), yi = (int)roundf(fy);       // Image::GetIndexRC (image.h:121-126)
    if (xi >= w || yi >= h || xi < 0 || yi < 0) return;
    const unsigned int at = (unsigned int)(t < 0 ? -t : t);
    const unsigned long long key = ((unsigned long long)at << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned int)ikl);
    atomicMin(&field[(size_t)yi * w + xi], key);
}

int rb_build_field_enqueue(rb_ctx *c, rb_map *m, int radius, float min_mod, bool from_state) {
    if (radius < 1) return RB_ERR_ARG;
    RB_CUDA(cudaMemsetAsync(m->field, 0xff, sizeof(unsigned long long) * (size_t)c->N, c->stream));
    const long long threads = (long long)c->kcap * 2 * radius;
    k_build_field<<<(unsigned)((threads + 255) / 256), 256, 0, c->stream>>>(m->field, m->kl, m->st, radius, min_mod,
                                                                          from_state ? 1 : 0, c->w, c->h);
    RB_LAUNCH_CHECK();
    m->field_radius = radius;
    return RB_OK;
}

// =====================================================================================================
// Minimizer_RV: LM driver executed by the last block of every evaluation kernel
// =====================================================================================================
__device__ __forceinline__ double max_element36(const double *M) {
    double m = M[0];
    for (int i = 1; i < 36; i++)
        if (M[i] > m) m = M[i];
    return m;
}
__device__ void lm_build_api(const LMState &s, double *A, double *rhs) {
    for (int i = 0; i < 36; i++) A[i] = s.JtJ[i];
    for (int i = 0; i < 6; i++) {
        A[i * 6 + i] = s.JtJ[i * 6 + i] + s.u;  // ApI = JtJ + Identity*u
        rhs[i] = -s.JtF[i];
    }
}
// Cholesky<6>(ApI).backsub(rhs) with every index known at compile time, so that the factor lives in registers (the
// generic chol6_* of lm.cuh share their arrays with the Jacobi fallback and end up in local memory, which made this
// serial step the longest part of an evaluation).  Same operations in the same order as TooN's do_compute/backsub;
// returns the smallest / largest pivot for the conditioning test of the SVD-replacement path.
template <bool RECIP_SCALE = false>   // true: y *= 1/diag (TooN's matrix backsub, used by get_inverse); false: y /= diag
__device__ __forceinline__ void chol6_solve_reg(const double (&M)[36], const double (&v)[6], double (&x)[6],
                                                double &dmin, double &dmax) {
    double a[36];
#pragma unroll
    for (int i = 0; i < 36; i++) a[i] = M[i];
#pragma unroll
    for (int col = 0; col < 6; col++) {
        double inv_diag = 1;
#pragma unroll
        for (int row = col; row < 6; row++) {
            double val = a[row * 6 + col];
#pragma unroll
            for (int col2 = 0; col2 < col; col2++) val -= a[col2 * 6 + col] * a[row * 6 + col2];
            if (row == col) {
                a[row * 6 + col] = val;
                inv_diag = 1 / val;
            } else {
                a[col * 6 + row] = val;
                a[row * 6 + col] = val * inv_diag;
            }
        }
    }
    dmin = a[0];
    dmax = a[0];
#pragma unroll
    for (int i = 1; i < 6; i++) {
        dmin = fmin(dmin, a[i * 6 + i]);
        dmax = fmax(dmax, a[i * 6 + i]);
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        double val = v[i];
#pragma unroll
        for (int j = 0; j < i; j++) val -= a[i * 6 + j] * y[j];
        y[i] = val;
    }
#pragma unroll
    for (int i = 0; i < 6; i++) {
        if (RECIP_SCALE) y[i] *= 1 / a[i * 6 + i];
        else y[i] /= a[i * 6 + i];
    }
#pragma unroll
    for (int i = 5; i >= 0; i--) {
        double val = y[i];
#pragma unroll
        for (int j = i + 1; j < 6; j++) val -= a[j * 6 + i] * x[j];
        x[i] = val;
    }
}
__device__ __noinline__ void lm_solve_fallback(LMState &s) {   // rank-deficient ApI: SVD<> pseudo-inverse semantics
    double A[36], rhs[6], h[6];
    lm_build_api(s, A, rhs);
    sym_svd_backsub(A, 6, rhs, h);
    for (int i = 0; i < 6; i++) s.h[i] = h[i];
}
__device__ void lm_solve(LMState &s, bool use_svd) {
    double A[36], rhs[6], h[6], dmin, dmax;
#pragma unroll
    for (int i = 0; i < 36; i++) A[i] = s.JtJ[i];
#pragma unroll
    for (int i = 0; i < 6; i++) {
        A[i * 6 + i] = s.JtJ[i * 6 + i] + s.u;  // ApI = JtJ + Identity*u
        rhs[i] = -s.JtF[i];
    }
    // Cholesky<6> svdApI(ApI); h = svdApI.backsub(-JtF)   (main loop, global_tracker.cpp:766-767)
    // SVD<> svdApI(ApI); h = svdApI.backsub(-JtF)          (init iterations, :659-661): ApI is SPD with a condition
    // number far below SVD.h's 1e9 cut, so the pseudo-inverse is the inverse and the LDL^T solve returns the same
    // vector up to rounding; the Jacobi pseudo-inverse is kept for rank-deficient input.
    chol6_solve_reg(A, rhs, h, dmin, dmax);
#pragma unroll
    for (int i = 0; i < 6; i++) s.h[i] = h[i];
    if (use_svd && !(dmin > 0 && dmin * 1e7 > dmax)) lm_solve_fallback(s);
#pragma unroll
    for (int i = 0; i < 6; i++) s.Xnew[i] = s.X[i] + s.h[i];
}
__device__ void lm_request(LMState &s, const double *X, int res_in, int res_out) {
    for (int i = 0; i < 6; i++) s.Xeval[i] = X[i];
    s.res_in = res_in;
    s.res_out = res_out;
}
__device__ void lm_take_first(LMState &s) {   // F = TryVelRot(JtJ, JtF, X ...); F0 = F; u = tau*max(JtJ)
    s.F = s.last_score;
    for (int i = 0; i < 36; i++) s.JtJ[i] = s.JtJn[i];
    for (int i = 0; i < 6; i++) s.JtF[i] = s.JtFn[i];
    s.F0 = s.F;
    s.u = 1e-3 * max_element36(s.JtJ);
}
// returns true when the step was accepted
__device__ bool lm_update(LMState &s, bool gain_with_den) {
    s.Fnew = s.last_score;
    if (gain_with_den) {
        double den = 0;  // 0.5*h*(u*h-JtF): TooN dot of (0.5*h) and (u*h-JtF)
        for (int i = 0; i < 6; i++) den += (0.5 * s.h[i]) * (s.u * s.h[i] - s.JtF[i]);
        s.gain = (s.F - s.Fnew) / den;
    } else {
        s.gain = s.F - s.Fnew;
    }
    if (s.gain > 0) {
        s.F = s.Fnew;
        for (int i = 0; i < 6; i++) s.X[i] = s.Xnew[i];
        for (int i = 0; i < 36; i++) s.JtJ[i] = s.JtJn[i];
        for (int i = 0; i < 6; i++) s.JtF[i] = s.JtFn[i];
        const double g = 2 * s.gain - 1;
        const double f = 1 - (g * g * g);
        s.u *= (0.33 > f ? 0.33 : f);  // std::max(0.33, ...)
        s.v = 2;
        s.eff_steps++;
        return true;
    }
    s.u *= s.v;
    s.v *= 2;
    return false;
}
__device__ void lm_after_zero_pass(LMState &s) {   // global_tracker.cpp:686-700
    for (int i = 0; i < 6; i++) s.Xt[i] = s.X[i];
    s.Ft = s.F;
    s.F0t = s.F0;
    s.ut = s.u;
    s.vt = s.v;
    s.eff_steps_t = s.eff_steps;
    s.eff_steps = 0;
    for (int i = 0; i < 3; i++) {
        s.X[i] = s.Vel_in[i];
        s.X[3 + i] = s.W0_in[i];
    }
    lm_request(s, s.X, -1, s.iRN);
}
__device__ void lm_after_prior_pass(LMState &s) {  // :734-747
    if (s.F > s.Ft) {
        for (int i = 0; i < 6; i++) s.X[i] = s.Xt[i];
        s.F = s.Ft;
        s.F0 = s.F0t;
        s.u = s.ut;
        s.v = s.vt;
        s.eff_steps = s.eff_steps_t;
        s.iRN = s.iRt;
    }
    const int t = s.iRN;
    s.iRN = s.iR;
    s.iR = t;
    lm_request(s, s.X, s.iR, s.iRN);
}
// RRV = Cholesky<6>(JtJ).get_inverse() (:795-801): column c = backsub(e_c) with the matrix overload's y *= 1/diag.
// Threads 0..5 of the calling block each factorise (registers) and solve one column.
__device__ __forceinline__ void lm_finalize_cov(LMState &s, int tid) {
    if (tid < 6) {
        double A[36], ec[6], x[6], dmin, dmax;
#pragma unroll
        for (int i = 0; i < 36; i++) A[i] = s.JtJ[i];
#pragma unroll
        for (int i = 0; i < 6; i++) ec[i] = (i == tid) ? 1.0 : 0.0;
        chol6_solve_reg<true>(A, ec, x, dmin, dmax);
        if (tid < 3) {
#pragma unroll
            for (int i = 0; i < 3; i++) s.RVel[i * 3 + tid] = x[i];
        } else {
#pragma unroll
            for (int i = 0; i < 3; i++) s.RW0[i * 3 + (tid - 3)] = x[3 + i];
        }
    }
}
__device__ void lm_finalize(LMState &s, MapState *fst) {   // :793-816; RVel / RW0 come from lm_finalize_cov
    for (int i = 0; i < 3; i++) {
        s.Vel[i] = s.X[i];
        s.W0[i] = s.X[3 + i];
    }
    for (int i = 0; i < 36; i++) s.W_X[i] = s.JtJ[i];
    if (s.eff_steps > 0) {
        double nh = 0, nx = 0;
        for (int i = 0; i < 6; i++) nh += s.h[i] * s.h[i];
        for (int i = 0; i < 6; i++) nx += s.X[i] * s.X[i];
        s.rel_error = sqrt(nh) / (sqrt(nx) + 1e-30);
        s.rel_error_score = s.F / s.F0;
    } else {
        s.rel_error = 1e20;
        s.rel_error_score = 1e20;
    }
    s.score = s.F;
    if (fst) fst->frame_count = fst->frame_count + 1;   // FrameCount++ (one CTA of the cluster kernel does it)
}

__device__ __forceinline__ void lm_step(LMState &s, int step, MapState *fst) {
    switch (step) {
        case STEP_INIT_FIRST_ZERO:
            lm_take_first(s);   // v = 2 from the declaration (:620)
            if (s.init_iter <= 0) {
                lm_after_zero_pass(s);
            } else {
                lm_solve(s, true);
                lm_request(s, s.Xnew, -1, s.iRt);
            }
            break;
        case STEP_INIT_ITER_ZERO:
            lm_update(s, true);
            lm_solve(s, true);
            lm_request(s, s.Xnew, -1, s.iRt);
            break;
        case STEP_INIT_LAST_ZERO:
            lm_update(s, false);
            lm_after_zero_pass(s);
            break;
        case STEP_INIT_FIRST_PRIOR:
            lm_take_first(s);
            s.v = 2;
            if (s.init_iter <= 0) {
                lm_after_prior_pass(s);
            } else {
                lm_solve(s, true);
                lm_request(s, s.Xnew, -1, s.iRN);
            }
            break;
        case STEP_INIT_ITER_PRIOR:
            lm_update(s, true);
            lm_solve(s, true);
            lm_request(s, s.Xnew, -1, s.iRN);
            break;
        case STEP_INIT_LAST_PRIOR:
            lm_update(s, false);
            lm_after_prior_pass(s);
            break;
        case STEP_MAIN_FIRST:
            lm_take_first(s);
            s.v = 2;
            if (s.iter_max <= 0) {
                lm_finalize(s, fst);
            } else {
                lm_solve(s, false);
                lm_request(s, s.Xnew, s.iR, s.iRN);
            }
            break;
        case STEP_MAIN_ITER:
        case STEP_MAIN_LAST:
            if (lm_update(s, true)) {   // std::swap(ResidualNew,Residual)
                const int t = s.iRN;
                s.iRN = s.iR;
                s.iR = t;
            }
            if (step == STEP_MAIN_LAST) {
                lm_finalize(s, fst);
            } else {
                lm_solve(s, false);
                lm_request(s, s.Xnew, s.iR, s.iRN);
            }
            break;
        default:
            break;
    }
}

struct ResPtrs {
    double *r[3];
};

// Sum 28 per-thread values over the block in a fixed order.  Inside a warp: a transposing butterfly -- at distance
// 16, 8, .. 1 every lane keeps one half of its values and trades the other half with its partner, so after 5 steps
// (16+8+4+2+1 = 31 exchanges instead of 28 x 5) lane l holds the warp's sum of value l.  Across warps: one
// shared-memory hop, thread k < 28 adds the warps' sums of value k in warp order.  dst[k * dst_stride] = sum k.
struct Red28Smem {
    double part[TVR_T / 32][32];
};
__device__ __forceinline__ double warp_transpose_sum28(const double (&acc)[28], int lane) {
    double v[16];
    {
        const bool up = (lane & 16) != 0;
#pragma unroll
        for (int k = 0; k < 16; k++) {
            const double hi = (k + 16 < 28) ? acc[k + 16] : 0.0;
            const double keep = up ? hi : acc[k], send = up ? acc[k] : hi;
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
        const bool up = (lane & o) != 0;
#pragma unroll
        for (int k = 0; k < o; k++) {
            const double keep = up ? v[k + o] : v[k], send = up ? v[k] : v[k + o];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
    }
    return v[0];
}
template <bool PJ>
__device__ __forceinline__ void reduce28(const double (&acc)[28], Red28Smem &rs, int tid, int lane, int wid,
                                         double *dst, int dst_stride) {
    if (PJ) {
        const double w = warp_transpose_sum28(acc, lane);
        __syncthreads();   // the previous user of rs is done
        rs.part[wid][lane] = w;
        __syncthreads();
        if (tid < 28) {
            double t = rs.part[0][tid];
#pragma unroll
            for (int ww = 1; ww < TVR_T / 32; ww++) t += rs.part[ww][tid];
            dst[tid * dst_stride] = t;
        }
    } else {
        double v = acc[27];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        __syncthreads();
        if (lane == 0) rs.part[0][wid] = v;
        __syncthreads();
        if (tid == 0) {
            double t = 0;
#pragma unroll
            for (int ww = 0; ww < TVR_T / 32; ww++) t += rs.part[0][ww];
            dst[27 * dst_stride] = t;
        }
    }
}

// Minimizer_RV preamble (global_tracker.cpp:596-650): configuration, LM variables, request of the first evaluation
__device__ void lm_begin(LMState &s, const MapState *old_st, const MapState *f_st, const double *VW,
                         const rb_minimizer_args &a, double max_r, double max_s_rho, int s_rho_from_state,
                         unsigned int frame_count, int fc_from_state) {
    s.max_r = max_r;
    s.match_thresh = a.match_thresh;
    s.k_huber = a.reweight_distance;
    s.match_num_thresh = a.match_num_thresh;
    s.iter_max = a.iter_max;
    s.init_type = a.init_type;
    s.init_iter = a.init_iter;
    s.s_rho_min = s_rho_from_state ? old_st->s_rho_q : max_s_rho;
    s.frame_count = fc_from_state ? f_st->frame_count : frame_count;
    for (int i = 0; i < 3; i++) {
        s.Vel_in[i] = VW[i];
        s.W0_in[i] = VW[3 + i];
    }
    s.iR = 0;
    s.iRN = 1;
    s.iRt = 2;
    s.v = 2;
    s.u = 0;
    s.eff_steps = 0;
    s.n_eval = 0;
    s.no_keylines = 0;
    s.pad_ = 0;
    s.F = s.F0 = s.Fnew = 0;
    for (int i = 0; i < 6; i++) s.h[i] = 0;
    if (a.init_type == 1) {
        for (int i = 0; i < 3; i++) {
            s.X[i] = VW[i];
            s.X[3 + i] = VW[3 + i];
        }
        lm_request(s, s.X, s.iR, s.iRN);
    } else if (a.init_type == 0) {
        for (int i = 0; i < 6; i++) s.X[i] = 0;
        lm_request(s, s.X, s.iR, s.iRN);
    } else {
        for (int i = 0; i < 6; i++) s.X[i] = 0;
        lm_request(s, s.X, -1, s.iRt);
    }
}
__global__ void k_lm_begin(TrackState *ts, const MapState *old_st, const MapState *f_st, const double *VW,
                           rb_minimizer_args a, double max_r, double max_s_rho, int s_rho_from_state,
                           unsigned int frame_count, int fc_from_state) {
    lm_begin(ts->lm, old_st, f_st, VW, a, max_r, max_s_rho, s_rho_from_state, frame_count, fc_from_state);
}

// ---- pieces of one TryVelRot evaluation (global_tracker.cpp:285-543), shared by the one-launch-per-evaluation
// kernel and by the persistent whole-minimisation kernel -------------------------------------------------------
struct TvrConst {          // constants of one minimisation
    double max_r, match_thresh, s_rho_min, k_huber;
    unsigned int mnt;      // min(match_num_thresh, FrameCount)
};
struct KlOp {              // operands of one old keyline; x0/y0/z0 do not depend on the evaluated pose
    float2 m;
    double x0, y0, z0, s_rho;
    int m_num;
    float n_m;
};
__device__ __forceinline__ KlOp load_klop(const KLSoA &old, int i, const CamC &cam) {
    KlOp o;
    const float2 pm = old.p_m[i];
    const double rho = old.rho[i];
    o.s_rho = old.s_rho[i];
    o.m_num = old.m_num[i];
    o.m = old.m_m[i];
    o.n_m = old.n_m[i];
    // KltoI3PMatrix + ProyI3Pto3PMatrix (global_tracker.cpp:552-570, ne10wrapper.h:413-424)
    o.z0 = 1 / rho;
    const double pz_zf0 = cam.inv_zf * o.z0;
    o.x0 = pz_zf0 * (double)pm.x;
    o.y0 = pz_zf0 * (double)pm.y;
    return o;
}
// a / b given y = RN(1/b): q = RN(a*y), one exact remainder, one correction -> RN(a/b) (Markstein); the seven
// divisions by q_rho of a keyline share one reciprocal.  Checked against IEEE division on 4e8 random and adversarial
// operand pairs (no mismatch); the only difference is the sign of a zero quotient of a negative zero.
__device__ __forceinline__ double div_with_rcp(double a, double b, double y) {
    const double q = a * y;
    const double r = fma(-b, q, a);
    return fma(r, y, q);
}
struct TvrSmem {
    Red28Smem red;
    double wlast[TVR_T / 32];
    int whas[TVR_T / 32];
};
struct TrackPtrs {         // the pointers inside TrackState, passed by value (no dependent load to reach them)
    LMState *lm;
    int *blk_has;
    double *blk_last_fi, *partials, *carry;
    struct MinCtl *ctl;
    unsigned long long *ll;
};

// per-keyline part: projection, field lookup, residual, Jacobian products
template <bool RW, bool PJ>
__device__ __forceinline__ void tvr_body(const KlOp &o, bool has_rin, double r_prev, const double *sR,
                                         const double *sV, const double *sRM, const TvrConst &tc, const CamC &cam,
                                         const unsigned long long *__restrict__ field,
                                         const float4 *__restrict__ fpack, double *__restrict__ rout,
                                         int *__restrict__ m_id_f, int i, double (&acc)[28], bool &matched,
                                         bool &need, double &fi_own, bool &wrote, double &r_w) {
    const double max_r = tc.max_r;
    const double x0 = o.x0, y0 = o.y0, z0 = o.z0;
    // SE3on3PMatrix (ne10wrapper.h:375-405): MulC, MlAc, MlAc, then Vel + .
    double px = sR[0] * x0;
    px = px + sR[1] * y0;
    px = px + sR[2] * z0;
    px = sV[0] + px;
    double py = sR[3] * x0;
    py = py + sR[4] * y0;
    py = py + sR[5] * z0;
    py = sV[1] + py;
    double pz = sR[6] * x0;
    pz = pz + sR[7] * y0;
    pz = pz + sR[8] * z0;
    pz = sV[2] + pz;
    // ProyP3toI3PMatrix (ne10wrapper.h:429-445)
    const double rho_p = 1 / pz;
    const double pz_zf = cam.zfm * rho_p;
    const double qx = pz_zf * px, qy = pz_zf * py;
    double f = 0, dfx = 0, dfy = 0;
    int mid_f = -1;
    const bool skip = (o.s_rho > tc.s_rho_min) || ((unsigned int)o.m_num < tc.mnt);   // :356
    if (!skip) {
        const double pix = qx + (double)cam.ppx, piy = qy + (double)cam.ppy;   // cam_mod.Hom2Img
        const int x = (int)(pix + 0.5), y = (int)(piy + 0.5);                   // util::round2int_positive
        double weight = 1;
        if (RW && has_rin) {
            const double r = fabs(r_prev);
            if (r > tc.k_huber) weight = tc.k_huber / r;                       // :370-372
        }
        if (x < 1 || y < 1 || x >= cam.w - 1 || y >= cam.h - 1) {               // :376
            f = max_r;
            if (RW) f *= weight;
            if (rout) rout[i] = max_r;   // (the cluster kernel keeps the residual buffers in shared memory: rout == nullptr)
            wrote = true;
            r_w = max_r;
        } else {
            const float mrx = (float)(sRM[0] * (double)o.m.x + sRM[1] * (double)o.m.y);   // :386-388
            const float mry = (float)(sRM[2] * (double)o.m.x + sRM[3] * (double)o.m.y);
            const unsigned long long key = field[(size_t)y * cam.w + x];
            bool hit = false;
            if (key != ~0ull) {
                const int ikl = (int)(0xFFFFFFFFu - (unsigned int)(key & 0xFFFFFFFFull));
                const float4 a = fpack[2 * ikl], b = fpack[2 * ikl + 1];
                const double p_n2 = (double)(o.n_m * o.n_m);                   // Test_f_k (global_tracker.h:89-104)
                const double p_esc = (double)(mrx * a.x + mry * a.y);
                if (!(fabs(p_esc - p_n2) > tc.match_thresh * p_n2)) {
                    const double dx = pix - (double)a.z, dy = piy - (double)a.w;   // Calc_f_J2 :254-262
                    const double fi = dx * (double)b.x + dy * (double)b.y;
                    dfx = (double)b.x;
                    dfy = (double)b.y;
                    f = fi;
                    matched = true;
                    fi_own = fi;
                    mid_f = ikl;
                    hit = true;
                }
            }
            if (!hit) {
                f = max_r;
                need = true;
            }
            if (RW) {
                f *= weight;
                dfx *= weight;
                dfy *= weight;
            }
        }
    }
    if (m_id_f) m_id_f[i] = mid_f;   // only the last evaluation of a minimisation is visible afterwards
    // Jacobians (:419-449) and the 1/q_rho scaling (:452-463)
    const double qvel = (cam.zfm * dfx * sV[0] + cam.zfm * dfy * sV[1]) + (qx * dfx + qy * dfy) * sV[2];
    double q_rho = sqrt(o.s_rho * qvel * o.s_rho * qvel + 1);
    if (!RW) q_rho = o.s_rho;
    if (PJ) {
        double t0 = cam.zfm * rho_p;
        double J0 = t0 * dfx, J1 = t0 * dfy;
        t0 = rho_p * qx;
        double J2 = t0 * dfx;
        t0 = rho_p * qy;
        J2 = J2 + t0 * dfy;
        double J3 = J1 * pz;
        J3 = J3 + J2 * py;
        double J4 = J0 * pz;
        J4 = J4 + J2 * px;
        t0 = J0 * py;
        double J5 = -1.0 * t0;
        J5 = J5 + J1 * px;
        const double iq = 1 / q_rho;
        double J[6] = {div_with_rcp(J0, q_rho, iq), div_with_rcp(J1, q_rho, iq), div_with_rcp(J2, q_rho, iq),
                       div_with_rcp(J3, q_rho, iq), div_with_rcp(J4, q_rho, iq), div_with_rcp(J5, q_rho, iq)};
        f = div_with_rcp(f, q_rho, iq);
        int k = 0;
#pragma unroll
        for (int a = 0; a < 6; a++)
#pragma unroll
            for (int b = a; b < 6; b++) acc[k++] = J[a] * J[b];
#pragma unroll
        for (int a = 0; a < 6; a++) acc[21 + a] = J[a] * f;
    } else {
        f = f / q_rho;
    }
    acc[27] = f * f;
}

// "DResidualNew[ikl]=fi" keeps the fi of the last matched keyline before ikl (fi is a function-level variable,
// :341,399-408): in-block scan here; misses that precede the block's first match get RES_SENTINEL and are resolved
// lazily by whoever reads the buffer, from the per-(buffer, block) carry table.  Then the block's 28 sums go to
// partials[k][vb] in a fixed order, and its "has a match / last matched fi" summary to blk_has / blk_last_fi.
template <bool PJ>
__device__ __forceinline__ void tvr_block_tail(bool active, bool matched, bool need, double fi_own,
                                               double *__restrict__ rout, int i, const double (&acc)[28],
                                               TvrSmem &sm, double *dst, int dst_stride, int *has_out,
                                               double *last_out, int tid, int lane, int wid, bool &wrote,
                                               double &r_w) {
    const unsigned int bal = __ballot_sync(0xffffffffu, matched);
    const unsigned int lower = bal & ((1u << lane) - 1u);
    const int src = lower ? 31 - __clz(lower) : 0;
    const double prev_fi = __shfl_sync(0xffffffffu, fi_own, src);
    const int hi = bal ? 31 - __clz(bal) : 0;
    const double wl = __shfl_sync(0xffffffffu, fi_own, hi);
    __syncthreads();   // the previous user of sm is done
    if (lane == 0) {
        sm.whas[wid] = bal != 0;
        sm.wlast[wid] = wl;
    }
    __syncthreads();
    if (active) {
        if (matched) {
            rout[i] = fi_own;
            wrote = true;
            r_w = fi_own;
        } else if (need) {
            double v = prev_fi;
            bool found = lower != 0;
            if (!found) {
                for (int ww = wid - 1; ww >= 0; ww--)
                    if (sm.whas[ww]) {
                        v = sm.wlast[ww];
                        found = true;
                        break;
                    }
            }
            if (!found) v = __longlong_as_double((long long)RES_SENTINEL);
            reinterpret_cast<unsigned long long *>(rout)[i] = (unsigned long long)__double_as_longlong(v);
            wrote = true;
            r_w = v;
        }
    }
    if (tid == 0) {
        int has = 0;
        double lastv = 0;
        for (int ww = 0; ww < TVR_T / 32; ww++)
            if (sm.whas[ww]) {
                has = 1;
                lastv = sm.wlast[ww];
            }
        *has_out = has;
        *last_out = lastv;
    }
    reduce28<PJ>(acc, sm.red, tid, lane, wid, dst, dst_stride);
}

// grid reduction of the per-block partials (layout [28][TVR_T], nb <= TVR_T blocks) in a fixed order: warp w owns sums
// w, w+8, ...; its lanes add the lane-strided entries (every load in flight at once), then one xor tree per sum.
// The caller synchronises before reading s_tot.
template <bool PJ>
__device__ __forceinline__ void tvr_grid_reduce(const double *partials, int nb, double *s_tot, int lane, int wid) {
    constexpr int NW = TVR_T / 32;
    if (PJ) {
        double v[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int k = wid + NW * q;
            double x[NW];
#pragma unroll
            for (int j = 0; j < NW; j++) {
                const int b = lane + 32 * j;
                x[j] = (k < 28 && b < nb) ? __ldcg(partials + k * TVR_T + b) : 0.0;
            }
            double t = x[0];
#pragma unroll
            for (int j = 1; j < NW; j++) t += x[j];
            v[q] = t;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int q = 0; q < 4; q++) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
        if (lane == 0)
#pragma unroll
            for (int q = 0; q < 4; q++)
                if (wid + NW * q < 28) s_tot[wid + NW * q] = v[q];
    } else if (wid == 0) {
        double t = 0;
#pragma unroll
        for (int j = 0; j < NW; j++) {
            const int b = lane + 32 * j;
            t += (b < nb) ? __ldcg(partials + 27 * TVR_T + b) : 0.0;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (lane == 0) s_tot[27] = t;
    }
}

// stale-fi carries: block b inherits the last matched fi of the nearest earlier block that has one (0 at the start);
// one ballot per warp finds it.  blockDim.x == TVR_T >= nb; thread b brings block b's summary (0 beyond nb).
__device__ __forceinline__ double tvr_carries(int has, double lastv, double *carry_out, int nb, double *s_blast,
                                            unsigned int *s_wmask, int tid, int lane, int wid) {
    const unsigned int mask = __ballot_sync(0xffffffffu, has != 0);
    s_blast[tid] = lastv;
    if (lane == 0) s_wmask[wid] = mask;
    __syncthreads();
    double cy = 0;
    if (tid < nb) {
        const unsigned int lower = mask & ((1u << lane) - 1u);
        if (lower) {
            cy = s_blast[wid * 32 + 31 - __clz(lower)];
        } else {
            for (int ww = wid - 1; ww >= 0; ww--) {
                const unsigned int mm = s_wmask[ww];
                if (mm) {
                    cy = s_blast[ww * 32 + 31 - __clz(mm)];
                    break;
                }
            }
        }
        carry_out[tid] = cy;
    }
    return cy;
}

// totals -> JtJn / JtFn / score of the evaluation (sign fix-ups :484-490)
template <bool PJ>
__device__ __forceinline__ void lm_ingest(LMState &L, const double *s_tot) {
    if (PJ) {
        int k = 0;
        for (int a = 0; a < 6; a++)
            for (int b = a; b < 6; b++) L.JtJn[a * 6 + b] = s_tot[k++];
        for (int a = 0; a < 6; a++) L.JtFn[a] = s_tot[21 + a];
        for (int a = 0; a < 2; a++) {
            L.JtFn[a + 2] = -L.JtFn[a + 2];
            for (int b = 0; b < 2; b++) {
                L.JtJn[(a + 0) * 6 + (b + 2)] = -L.JtJn[(a + 0) * 6 + (b + 2)];
                L.JtJn[(a + 2) * 6 + (b + 4)] = -L.JtJn[(a + 2) * 6 + (b + 4)];
            }
        }
        for (int a = 0; a < 6; a++)
            for (int b = a + 1; b < 6; b++) L.JtJn[b * 6 + a] = L.JtJn[a * 6 + b];
    }
    L.last_score = s_tot[27];
    L.n_eval++;
}

// One TryVelRot evaluation + the LM step that follows it, one launch per evaluation (stage-level API rb_try_vel_rot,
// and minimisations whose keyline capacity exceeds what the persistent kernel below can keep co-resident).
template <bool RW, bool PJ>
__global__ void __launch_bounds__(TVR_T) k_tvr_eval(KLSoA old, const MapState *__restrict__ old_st,
                                                    const unsigned long long *__restrict__ field,
                                                    const float4 *__restrict__ fpack, MapState *f_st, TrackPtrs tp,
                                                    ResPtrs res, unsigned int *ticket, CamC cam, int step) {
    __shared__ double sR[9], sV[3], sRM[4];
    __shared__ TvrSmem sm;
    __shared__ double s_tot[28];
    __shared__ bool s_last;
    LMState &lm = *tp.lm;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) {   // the two exponentials run on two warps side by side (each is a serial sin/cos chain)
        double X[6];
        for (int i = 0; i < 6; i++) X[i] = lm.Xeval[i];
        so3_exp(X + 3, sR);                        // SO3<> RotW0(VelRot.slice<3,3>())
        for (int i = 0; i < 3; i++) sV[i] = X[i];
    } else if (tid == 32) {
        double wz[3] = {0, 0, lm.Xeval[5]}, RMf[9];
        so3_exp(wz, RMf);                          // SO3<> RotM(makeVector(0,0,VelRot[5]))
        sRM[0] = RMf[0];
        sRM[1] = RMf[1];
        sRM[2] = RMf[3];
        sRM[3] = RMf[4];
    }
    __syncthreads();
    const int res_in = lm.res_in, res_out = lm.res_out;
    TvrConst tc;
    tc.max_r = lm.max_r;
    tc.match_thresh = lm.match_thresh;
    tc.s_rho_min = lm.s_rho_min;
    tc.k_huber = lm.k_huber;
    tc.mnt = lm.match_num_thresh < lm.frame_count ? lm.match_num_thresh : lm.frame_count;
    const double *__restrict__ rin = (RW && res_in >= 0) ? res.r[res_in] : nullptr;
    double *__restrict__ rout = res.r[res_out];

    const int K0 = old_st->kn;
    const int i = blockIdx.x * TVR_T + tid;
    const bool active = i < K0;
    double acc[28];
#pragma unroll
    for (int k = 0; k < 28; k++) acc[k] = 0;
    bool matched = false, need = false, wrote = false;
    double fi_own = 0, r_w = 0;
    if (active) {
        const KlOp o = load_klop(old, i, cam);
        double r_prev = (RW && rin) ? rin[i] : 0.0;
        if (RW && rin && (unsigned long long)__double_as_longlong(r_prev) == RES_SENTINEL)
            r_prev = tp.carry[res_in * TVR_T + blockIdx.x];   // stale-fi carry of the evaluation that wrote rin
        tvr_body<RW, PJ>(o, rin != nullptr, r_prev, sR, sV, sRM, tc, cam, field, fpack, rout, old.m_id_f, i, acc,
                         matched, need, fi_own, wrote, r_w);
    }
    tvr_block_tail<PJ>(active, matched, need, fi_own, rout, i, acc, sm, tp.partials + blockIdx.x, TVR_T,
                       tp.blk_has + blockIdx.x, tp.blk_last_fi + blockIdx.x, tid, lane, wid, wrote, r_w);
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    // ================= last block: grid reduction, stale-fi carries, LM step ==========================
    __threadfence();
    const int nb = gridDim.x;   // <= TVR_T (checked by the host)
    tvr_grid_reduce<PJ>(tp.partials, nb, s_tot, lane, wid);
    __shared__ double s_blast[TVR_T];
    __shared__ unsigned int s_wmask[TVR_T / 32];
    {
        int has = 0;
        double lastv = 0;
        if (tid < nb) {
            has = __ldcg(tp.blk_has + tid);
            lastv = __ldcg(tp.blk_last_fi + tid);
        }
        tvr_carries(has, lastv, tp.carry + res_out * TVR_T, nb, s_blast, s_wmask, tid, lane, wid);
    }
    // the serial LM step works on a shared-memory copy of the state (global round trips would dominate it)
    __shared__ LMState s_lm;
    {
        const double *src = reinterpret_cast<const double *>(&lm);
        double *dst = reinterpret_cast<double *>(&s_lm);
        for (int k = tid; k < (int)(sizeof(LMState) / sizeof(double)); k += TVR_T) dst[k] = __ldcg(src + k);
    }
    __syncthreads();
    if (tid == 0) {
        lm_ingest<PJ>(s_lm, s_tot);
        lm_step(s_lm, step, f_st);
        *ticket = 0;
    }
    __syncthreads();
    if (step == STEP_MAIN_LAST || (step == STEP_MAIN_FIRST && s_lm.iter_max <= 0)) {
        lm_finalize_cov(s_lm, tid);
        __syncthreads();
    }
    {
        const double *src = reinterpret_cast<const double *>(&s_lm);
        double *dst = reinterpret_cast<double *>(&lm);
        for (int k = tid; k < (int)(sizeof(LMState) / sizeof(double)); k += TVR_T) dst[k] = src[k];
    }
}

// =====================================================================================================
// Whole Minimizer_RV in ONE launch (min_cluster.cuh).  The ~12 evaluations of a frame are strictly dependent (each pose
// comes out of the LM step on the previous sums), so with one launch per evaluation a frame pays 12x (launch + operand
// re-load + last-block hand-over through L2).  Shared declarations of the persistent forms:
// =====================================================================================================
#define MIN_MAX_EVALS 32
struct MinSetup {
    rb_minimizer_args a;
    double max_r, max_s_rho;
    const double *VW;
    unsigned int frame_count;
    int s_rho_from_state, fc_from_state;
    int debug_abort;
    int early_operands;   // the kernel before this one on the stream writes no keyline array of the old map (see k_minimizer_cluster)
};

__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long *p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long *p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_volatile_u32(const unsigned int *p) {
    unsigned int v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// =====================================================================================================
// FordwardMatch (edge_tracker.cpp:380-436), first part.  Sequential rule: a later old keyline replaces the holder of
// its target unless the holder's rho is strictly larger => winner = arg max rho, ties -> largest index, i.e. the
// lexicographic maximum of (dbl_key(rho), i) over the old keylines i with m_id_f[i] == f.  One 128-bit CAS per offer
// (k_fm_argmax, or the cluster minimiser right after its last evaluation has written m_id_f).
// =====================================================================================================
__device__ __forceinline__ unsigned long long dbl_key(double v) {   // monotonic map double -> uint64
    unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
// one 128-bit CAS of *rec from (ck, ci) to (key, i); (ok, oi) = what the record held
__device__ __forceinline__ void fm_cas(FmBest *rec, unsigned long long ck, long long ci, unsigned long long key, long long i,
                                       unsigned long long &ok, long long &oi) {
    asm volatile(
        "{\n\t.reg .b128 cmp, swp, old;\n\t"
        "mov.b128 cmp, {%2, %3};\n\tmov.b128 swp, {%4, %5};\n\t"
        "atom.relaxed.gpu.global.cas.b128 old, [%6], cmp, swp;\n\t"
        "mov.b128 {%0, %1}, old;\n\t}"
        : "=l"(ok), "=l"(oi)
        : "l"(ck), "l"(ci), "l"(key), "l"(i), "l"(rec)
        : "memory");
}
// one step of an offer: false once *rec holds (key, i) or a lexicographically larger pair; (ck, ci) = the expected value
__device__ __forceinline__ bool fm_retry(unsigned long long key, long long i, unsigned long long &ck, long long &ci,
                                         unsigned long long ok, long long oi) {
    if (ok == ck && oi == ci) return false;
    ck = ok;
    ci = oi;
    return key > ck || (key == ck && i > ci);
}
// raises *rec to (key, i) unless it already holds a lexicographically larger pair.  The first CAS expects the cleared
// record {0, -1} instead of reading it (a plain 16-byte read may tear); every later one compares the value a CAS returned.
__device__ __forceinline__ void d_fm_offer(FmBest *rec, unsigned long long key, long long i) {
    unsigned long long ck = 0ull, ok;
    long long ci = -1, oi;
    do fm_cas(rec, ck, ci, key, i, ok, oi);
    while (fm_retry(key, i, ck, ci, ok, oi));
}
__device__ __forceinline__ void d_fm_argmax_one(const KLSoA &old, int i, int nkn, FmBest *best) {
    const int f = old.m_id_f[i];
    if (f < 0 || f >= nkn) return;
    d_fm_offer(&best[f], dbl_key(old.rho[i]), i);
}
// the offers of old keylines i0 and i1 (i1 < 0: none) with their loads and their CAS round trips in flight together
__device__ __forceinline__ void d_fm_argmax_two(const KLSoA &old, int i0, int i1, int nkn, FmBest *best) {
    const int f0 = old.m_id_f[i0], f1 = i1 >= 0 ? old.m_id_f[i1] : -1;
    const unsigned long long k0 = dbl_key(old.rho[i0]), k1 = i1 >= 0 ? dbl_key(old.rho[i1]) : 0ull;
    bool a0 = f0 >= 0 && f0 < nkn, a1 = f1 >= 0 && f1 < nkn;
    unsigned long long c0 = 0ull, c1 = 0ull, o0 = 0ull, o1 = 0ull;
    long long d0 = -1, d1 = -1, p0 = -1, p1 = -1;
    while (a0 || a1) {
        if (a0) fm_cas(&best[f0], c0, d0, k0, i0, o0, p0);
        if (a1) fm_cas(&best[f1], c1, d1, k1, i1, o1, p1);
        a0 = a0 && fm_retry(k0, i0, c0, d0, o0, p0);
        a1 = a1 && fm_retry(k1, i1, c1, d1, o1, p1);
    }
}

// one-cluster form (16 CTAs x 512 threads: co-residency guaranteed, 16 SMs) and multi-cluster form (G x 16 CTAs x 256 threads)
#define MC_T 512
#define MC_NS mc_one
#include "min_cluster.cuh"
#undef MC_T
#undef MC_NS
#define MC_T 256
#define MC_NS mc_multi
#include "min_cluster.cuh"
#undef MC_T
#undef MC_NS

static TrackPtrs track_ptrs(const rb_map *fmap) {
    TrackPtrs tp;
    tp.lm = &fmap->ts->lm;
    tp.blk_has = fmap->ts_host.blk_has;
    tp.blk_last_fi = fmap->ts_host.blk_last_fi;
    tp.partials = fmap->ts_host.partials;
    tp.carry = fmap->ts_host.carry;
    tp.ctl = fmap->ts_host.ctl;
    tp.ll = fmap->ts_host.ll;
    return tp;
}

template <bool RW, bool PJ>
static int launch_eval(rb_ctx *c, rb_map *fmap, rb_map *old, int step) {
    ResPtrs rp;
    for (int i = 0; i < 3; i++) rp.r[i] = fmap->res[i];
    const int nblk = fmap->ts_host.nblk;
    k_tvr_eval<RW, PJ><<<nblk, TVR_T, 0, c->stream>>>(old->kl, old->st, fmap->field, fmap->kl.pack, fmap->st,
                                                     track_ptrs(fmap), rp, c->ticket + 1, make_cam(c), step);
    RB_LAUNCH_CHECK();
    return RB_OK;
}
static int launch_eval_step(rb_ctx *c, rb_map *fmap, rb_map *old, int step) {
    if (step >= STEP_MAIN_FIRST) return launch_eval<true, true>(c, fmap, old, step);
    if (step == STEP_INIT_LAST_ZERO || step == STEP_INIT_LAST_PRIOR) return launch_eval<false, false>(c, fmap, old, step);
    return launch_eval<false, true>(c, fmap, old, step);
}

// per-device set-up of the cluster minimiser (rb_ctx_create, after cudaSetDevice): opt-ins + how many keylines per CTA
// fit.  Leaves c->min_cluster_kpc = 0 when the device cannot run it (the one-launch-per-evaluation path serves then).
void rb_mapper_cluster_setup();   // (defined after the mapper's cluster kernels)
template <typename K>
static bool mc_prepare(K kern, int threads, int clusters, size_t dyn, int dev_max) {
    cudaFuncAttributes fa;
    if (cudaFuncGetAttributes(&fa, kern) != cudaSuccess) return false;
    if (dyn + fa.sharedSizeBytes > (size_t)dev_max) return false;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) return false;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn) != cudaSuccess) return false;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(MC_C * clusters);
    cfg.blockDim = dim3(threads);
    cfg.dynamicSmemBytes = dyn;
    int ncl = 0;
    return cudaOccupancyMaxActiveClusters(&ncl, kern, &cfg) == cudaSuccess && ncl >= clusters;
}
int rb_minimizer_cluster_setup(rb_ctx *c) {
    rb_mapper_cluster_setup();
    c->min_cluster_kpc = 0;
    c->min_cluster_g = 1;
    const char *fa_ = getenv("REBVO_B200_MIN_FORCE_ABORT");
    c->min_debug_abort = fa_ ? atoi(fa_) : 0;
    const char *xe = getenv("REBVO_B200_MIN_XCHG");
    c->min_cluster_xchg = xe ? atoi(xe) : 1;
    int dev_max = 0;
    if (cudaDeviceGetAttribute(&dev_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, c->device) != cudaSuccess) return RB_OK;
    int kfast = MC_KPC_FAST;                   // keylines per cluster rank kept in shared memory (the rest works from global memory)
    const char *kf = getenv("REBVO_B200_MIN_KPC");
    if (kf && atoi(kf) >= 32) kfast = atoi(kf) & ~31;
    // one cluster: always possible when the capacity fits its virtual-warp tables
    {
        int kpc = (c->kcap + MC_C - 1) / MC_C;
        kpc = (kpc + 31) & ~31;
        if (kpc <= 512 * (3584 / 512)) {
            if (kpc > kfast) kpc = kfast;
            const size_t dyn = (size_t)kpc * MC_BYTES_PER_KL + 64;
            if (mc_prepare(mc_one::k_minimizer_cluster<1>, 512, 1, dyn, dev_max) &&
                mc_prepare(mc_one::k_minimizer_cluster<0>, 512, 1, dyn, dev_max)) {
                c->min_cluster_kpc = kpc;
                c->min_cluster_dyn = dyn;
            }
        }
    }
    cudaGetLastError();
    // several clusters (default 4 = 64 SMs): the per-evaluation keyline pass is the longest part of a round and scales with
    // the SMs; the clusters exchange their sums through L2.  Needs all clusters co-resident: checked here for an idle
    // device (spins are bounded and abort otherwise), so contexts that share a GPU should ask for REBVO_B200_MIN_G=1.
    int G = 4;
    const char *ge = getenv("REBVO_B200_MIN_G");
    if (ge) G = atoi(ge);
    if (G > MC_GMAX) G = MC_GMAX;
    if (c->min_cluster_kpc > 0 && G > 1) {
        int kpc = (c->kcap + MC_C * G - 1) / (MC_C * G);
        kpc = (kpc + 31) & ~31;
        if (kpc <= 256 * (3584 / 256)) {
            int kf2 = (kfast / G + 31) & ~31;
            if (kpc > kf2) kpc = kf2;
            const size_t dyn = (size_t)kpc * MC_BYTES_PER_KL + 64;
            if (mc_prepare(mc_multi::k_minimizer_cluster<1>, 256, G, dyn, dev_max) &&
                mc_prepare(mc_multi::k_minimizer_cluster<0>, 256, G, dyn, dev_max)) {
                c->min_cluster_g = G;
                c->min_cluster_kpc_multi = kpc;
                c->min_cluster_dyn_multi = dyn;
            }
        }
    }
    cudaGetLastError();
    return RB_OK;
}

static int launch_minimizer_cluster(rb_ctx *c, rb_map *fmap, rb_map *old, const McPlan &plan, const MinSetup &su,
                                    FrameState *post_fs) {
    const int G = c->min_cluster_g;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(MC_C * G);
    cfg.blockDim = dim3(G > 1 ? 256 : 512);
    cfg.dynamicSmemBytes = G > 1 ? c->min_cluster_dyn_multi : c->min_cluster_dyn;
    cfg.stream = c->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = c->pdl ? 1 : 0;
    c->launches++;
    ResPtrs rp;
    for (int i = 0; i < 3; i++) rp.r[i] = fmap->res[i];
    auto kern = G > 1 ? (c->min_cluster_xchg ? mc_multi::k_minimizer_cluster<1> : mc_multi::k_minimizer_cluster<0>)
                      : (c->min_cluster_xchg ? mc_one::k_minimizer_cluster<1> : mc_one::k_minimizer_cluster<0>);
    const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, old->kl, (const MapState *)old->st,
                                             (const unsigned long long *)fmap->field, (const float4 *)fmap->kl.pack,
                                             fmap->st, &fmap->ts->lm, &fmap->ts_host.ctl->abort, make_cam(c), plan, su,
                                             post_fs, post_fs ? fmap->ts_host.fm_best : nullptr,
                                             G > 1 ? c->min_cluster_kpc_multi : c->min_cluster_kpc, rp,
                                             fmap->ts_host.ll, fmap->ts_host.ctl);
    if (e != cudaSuccess) {
        snprintf(c->err, sizeof(c->err), "Minimizer_RV cluster launch: %s", cudaGetErrorString(e));
        return RB_ERR_CUDA;
    }
    return RB_OK;
}

int rb_minimizer_enqueue(rb_ctx *c, rb_map *fmap, rb_map *old, const double *VW_dev, const rb_minimizer_args *a,
                         double max_s_rho, bool s_rho_from_state, unsigned int frame_count, bool fc_from_state,
                         FrameState *post_fs, bool *post_folded) {
    if (post_folded) *post_folded = false;
    if (fmap->field_radius <= 0) {
        snprintf(c->err, sizeof(c->err), "Minimizer_RV before build_field");
        return RB_ERR_STATE;
    }
    const int nblk = fmap->ts_host.nblk;
    if (nblk > TVR_T) return RB_ERR_ARG;
    // the evaluation sequence of Minimizer_RV (global_tracker.cpp:640-791) is fixed by the configuration
    const int n = a->init_iter, m = a->iter_max;
    int steps[2 * MIN_MAX_EVALS], ns = 0;
    if (n < 0 || m < 0 || 2 * (n + 1) + m + 1 > 2 * MIN_MAX_EVALS) return RB_ERR_ARG;
    if (a->init_type != 0 && a->init_type != 1) {
        steps[ns++] = STEP_INIT_FIRST_ZERO;
        for (int i = 0; i < n; i++) steps[ns++] = i == n - 1 ? STEP_INIT_LAST_ZERO : STEP_INIT_ITER_ZERO;
        steps[ns++] = STEP_INIT_FIRST_PRIOR;
        for (int i = 0; i < n; i++) steps[ns++] = i == n - 1 ? STEP_INIT_LAST_PRIOR : STEP_INIT_ITER_PRIOR;
    }
    steps[ns++] = STEP_MAIN_FIRST;
    for (int j = 0; j < m; j++) steps[ns++] = j == m - 1 ? STEP_MAIN_LAST : STEP_MAIN_ITER;
    int r;
    if (c->min_persist && c->min_cluster && c->min_cluster_kpc > 0 && ns <= MIN_MAX_EVALS) {
        // rounds of the cluster kernel: the two init tries of type 2 share their rounds
        McPlan plan;
        memset(&plan, 0, sizeof(plan));
        plan.merge_round = -1;
        int k = 0;
        if (a->init_type != 0 && a->init_type != 1) {
            for (int i = 0; i <= n; i++, k++) {
                plan.sa[k] = i == 0 ? STEP_INIT_FIRST_ZERO : i == n ? STEP_INIT_LAST_ZERO : STEP_INIT_ITER_ZERO;
                plan.sb[k] = i == 0 ? STEP_INIT_FIRST_PRIOR : i == n ? STEP_INIT_LAST_PRIOR : STEP_INIT_ITER_PRIOR;
            }
            plan.merge_round = k - 1;
        }
        plan.sb[k++] = STEP_MAIN_FIRST;
        for (int j = 0; j < m; j++) plan.sb[k++] = j == m - 1 ? STEP_MAIN_LAST : STEP_MAIN_ITER;
        plan.n = k;
        MinSetup su;
        su.a = *a;
        su.max_r = (double)fmap->field_radius;
        su.max_s_rho = max_s_rho;
        su.VW = VW_dev;
        su.frame_count = frame_count;
        su.s_rho_from_state = s_rho_from_state ? 1 : 0;
        su.fc_from_state = fc_from_state ? 1 : 0;
        su.debug_abort = c->min_debug_abort;
        su.early_operands = c->min_early ? 1 : 0;
        if ((r = launch_minimizer_cluster(c, fmap, old, plan, su, post_fs))) return r;
        if (post_folded) *post_folded = post_fs != nullptr;
        return RB_OK;
    }
    RB_CUDA(cudaMemsetAsync(fmap->res[0], 0, sizeof(double) * (size_t)c->kcap, c->stream));   // Residual[i]=0 (:625)
    k_lm_begin<<<1, 1, 0, c->stream>>>(fmap->ts, old->st, fmap->st, VW_dev, *a, (double)fmap->field_radius,
                                       max_s_rho, s_rho_from_state ? 1 : 0, frame_count, fc_from_state ? 1 : 0);
    RB_LAUNCH_CHECK();
    for (int i = 0; i < ns; i++)
        if ((r = launch_eval_step(c, fmap, old, steps[i]))) return r;
    return RB_OK;
}

int rb_minimizer_check_abort(rb_ctx *c, rb_map *fmap) {
    int ab = 0;
    RB_CUDA(cudaMemcpyAsync(&ab, &fmap->ts_host.ctl->abort, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    if (!ab) return RB_OK;
    RB_CUDA(cudaMemsetAsync(&fmap->ts_host.ctl->abort, 0, sizeof(int), c->stream));
    RB_CUDA(cudaStreamSynchronize(c->stream));
    snprintf(c->err, sizeof(c->err), "Minimizer_RV: an exchange between the kernel's CTAs timed out (results are NaN)");
    return RB_ERR_CUDA;
}

// materialise the lazily resolved entries of a residual buffer (host export of DResidualNew in rb_try_vel_rot)
__global__ void __launch_bounds__(TVR_T) k_resolve_res(double *res, const double *carry, const MapState *old_st) {
    const int i = blockIdx.x * TVR_T + threadIdx.x;
    if (i >= old_st->kn) return;
    if (reinterpret_cast<unsigned long long *>(res)[i] == RES_SENTINEL) res[i] = carry[blockIdx.x];
}
int rb_resolve_res_enqueue(rb_ctx *c, rb_map *fmap, rb_map *old, int buf) {
    k_resolve_res<<<fmap->ts_host.nblk, TVR_T, 0, c->stream>>>(fmap->res[buf], fmap->ts_host.carry + buf * TVR_T, old->st);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// single evaluation for the parity tests (rb_try_vel_rot)
__global__ void k_lm_single(TrackState *ts, const double *X, int res_in, int res_out, double max_r, double mt,
                            double s_rho_min, unsigned int mnt, unsigned int fc, double k_huber) {
    LMState &s = ts->lm;
    for (int i = 0; i < 6; i++) s.Xeval[i] = X[i];
    s.res_in = res_in;
    s.res_out = res_out;
    s.max_r = max_r;
    s.match_thresh = mt;
    s.s_rho_min = s_rho_min;
    s.match_num_thresh = mnt;
    s.frame_count = fc;
    s.k_huber = k_huber;
}

int rb_try_vel_rot_enqueue(rb_ctx *c, rb_map *fmap, rb_map *old, const double *X_dev, int reweight, int procjf,
                           double match_thresh, double s_rho_min, unsigned int mnt, unsigned int fc,
                           double k_huber) {
    if (fmap->field_radius <= 0) return RB_ERR_STATE;
    k_lm_single<<<1, 1, 0, c->stream>>>(fmap->ts, X_dev, 0, 1, (double)fmap->field_radius, match_thresh, s_rho_min,
                                        mnt, fc, k_huber);
    RB_LAUNCH_CHECK();
    if (reweight && procjf) return launch_eval<true, true>(c, fmap, old, STEP_NONE);
    if (reweight) return launch_eval<true, false>(c, fmap, old, STEP_NONE);
    if (procjf) return launch_eval<false, true>(c, fmap, old, STEP_NONE);
    return launch_eval<false, false>(c, fmap, old, STEP_NONE);
}

// =====================================================================================================
// rotate_keylines (edge_tracker.cpp:42-76)
// =====================================================================================================
// The rotation of one keyline as values: the in-place rotation below and the matching kernel, which rotates the old
// keylines it probes on the fly, share these two helpers, so both see the same bits.
struct RotPt {
    float2 pm;
    double rho, s_rho;
};
// (p_m, rho, s_rho) rotated by R; unchanged when the rotated point has no finite depth
__device__ __forceinline__ RotPt d_rot_pt(const double (&R)[9], double zf, float2 pm, double rho, double s_rho) {
    const double v0 = (double)pm.x / zf, v1 = (double)pm.y / zf, v2 = 1;
    double q0 = 0, q1 = 0, q2 = 0;   // TooN Matrix*Vector: dot accumulates from 0
    q0 = q0 + R[0] * v0; q0 = q0 + R[1] * v1; q0 = q0 + R[2] * v2;
    q1 = q1 + R[3] * v0; q1 = q1 + R[4] * v1; q1 = q1 + R[5] * v2;
    q2 = q2 + R[6] * v0; q2 = q2 + R[7] * v1; q2 = q2 + R[8] * v2;
    RotPt o = {pm, rho, s_rho};
    if (fabs(q2) > 0) {
        o.pm = make_float2((float)(q0 / q2 * zf), (float)(q1 / q2 * zf));
        o.rho = rho / q2;
        o.s_rho = s_rho / q2;
    }
    return o;
}
// m_m rotated by R
__device__ __forceinline__ float2 d_rot_m(const double (&R)[9], float2 m) {
    const double m0 = (double)m.x, m1 = (double)m.y;
    double r0 = 0, r1 = 0;
    r0 = r0 + R[0] * m0; r0 = r0 + R[1] * m1; r0 = r0 + R[2] * 0.0;
    r1 = r1 + R[3] * m0; r1 = r1 + R[4] * m1; r1 = r1 + R[5] * 0.0;
    return make_float2((float)r0, (float)r1);
}
// keyline i of kl rotated by R, from its p_m, rho, s_rho and m_m as loaded by the caller
__device__ __forceinline__ void d_rotate_vals(const KLSoA &kl, int i, const double (&R)[9], double zf, float2 pm, double rho,
                                              double s_rho, float2 m) {
    const RotPt pt = d_rot_pt(R, zf, pm, rho, s_rho);
    kl.p_m[i] = pt.pm;
    kl.rho[i] = pt.rho;
    kl.s_rho[i] = pt.s_rho;
    const float2 mr = d_rot_m(R, m);
    kl.m_m[i] = mr;
    float4 p = kl.pack[2 * i];
    p.x = mr.x;
    p.y = mr.y;
    kl.pack[2 * i] = p;
}
__device__ __forceinline__ void d_rotate(const KLSoA &kl, int i, const double *__restrict__ Rp, double zf) {
    double R[9];
#pragma unroll
    for (int k = 0; k < 9; k++) R[k] = Rp[k];
    d_rotate_vals(kl, i, R, zf, kl.p_m[i], kl.rho[i], kl.s_rho[i], kl.m_m[i]);
}
__global__ void __launch_bounds__(256) k_rotate(KLSoA kl, const MapState *st, const double *__restrict__ Rp,
                                                double zf) {
    pdl_wait();
    pdl_launch();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st->kn) return;
    d_rotate(kl, i, Rp, zf);
}

// =====================================================================================================
// FordwardMatch (edge_tracker.cpp:380-436), second part: the arg-max (d_fm_offer, above the minimiser) is complete.
// Indexed by OLD keyline: the winner of new keyline f copies its own record into neu[f], then (ROT) rotates itself in
// place -- no thread reads another thread's old keyline, so the two need no barrier between them.
// =====================================================================================================
__global__ void __launch_bounds__(256) k_fm_init(FmBest *best, const MapState *nst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nst->kn) return;
    best[i] = FmBest{0ull, -1ll};
}
__global__ void __launch_bounds__(256) k_fm_argmax(KLSoA old, const MapState *ost, const MapState *nst, FmBest *best) {
    pdl_wait();
    pdl_launch();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ost->kn) return;
    d_fm_argmax_one(old, i, nst->kn, best);
}
template <bool ROT>
__global__ void __launch_bounds__(256) k_fm_apply_rotate(KLSoA old, KLSoA neu, const MapState *ost, MapState *nst,
                                                         const FmBest *best, const double *__restrict__ Rp, double zf) {
    pdl_wait();
    pdl_launch();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < ost->kn;
    bool hit = false;
    double R[9], rho = 0, s_rho = 0;
#pragma unroll
    for (int k = 0; k < 9; k++) R[k] = ROT ? Rp[k] : 0.0;
    float2 pm = make_float2(0.f, 0.f), m = pm;
    if (in) {   // keyline i's record is loaded once, before any store, for the copy and for the rotation
        const int f = old.m_id_f[i];
        rho = old.rho[i];
        s_rho = old.s_rho[i];
        pm = old.p_m[i];
        m = old.m_m[i];
        if (f >= 0 && f < nst->kn && __ldcg(&best[f].idx) == i) {
            neu.rho[f] = rho;
            neu.s_rho[f] = s_rho;
            neu.m_num[f] = old.m_num[i] + 1;
            neu.m_id[f] = i;
            neu.p_m_0[f] = pm;
            neu.m_m0[f] = m;
            neu.n_m0[f] = (double)old.n_m[i];
            hit = true;
        }
    }
    const unsigned int bal = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&nst->fwd_match, __popc(bal));
    if (ROT && in) d_rotate_vals(old, i, R, zf, pm, rho, s_rho, m);
}
__global__ void k_set_int(int *p, int v) { *p = v; }

// the arg-max scratch of a map only depends on its keyline count: the pipeline clears it before the minimiser
int rb_forward_match_init_enqueue(rb_ctx *c, rb_map *neu) {
    k_fm_init<<<rb_div_up(c->kcap, 256), 256, 0, c->stream>>>(neu->ts_host.fm_best, neu->st);
    RB_LAUNCH_CHECK();
    return RB_OK;
}
int rb_forward_match_argmax_enqueue(rb_ctx *c, rb_map *old, rb_map *neu) {
    RB_KLAUNCH(k_fm_argmax, rb_div_up(c->kcap, 256), 256, 0, old->kl, (const MapState *)old->st,
               (const MapState *)neu->st, neu->ts_host.fm_best);
    return RB_OK;
}
int rb_forward_match_apply_enqueue(rb_ctx *c, rb_map *old, rb_map *neu, const double *R_dev) {
    const int nb = rb_div_up(c->kcap, 256);
    const FmBest *best = neu->ts_host.fm_best;
    if (R_dev)
        RB_KLAUNCH(k_fm_apply_rotate<true>, nb, 256, 0, old->kl, neu->kl, (const MapState *)old->st, neu->st, best, R_dev,
                   c->zfm);
    else
        RB_KLAUNCH(k_fm_apply_rotate<false>, nb, 256, 0, old->kl, neu->kl, (const MapState *)old->st, neu->st, best, R_dev,
                   c->zfm);
    return RB_OK;
}
int rb_forward_match_enqueue(rb_ctx *c, rb_map *old, rb_map *neu) {
    if (!c->counters_preset) {   // the per-frame pipeline zeroes the counters in k_frame_pre
        k_set_int<<<1, 1, 0, c->stream>>>(&neu->st->fwd_match, 0);
        RB_LAUNCH_CHECK();
    }
    int r;
    if ((r = rb_forward_match_init_enqueue(c, neu))) return r;
    if ((r = rb_forward_match_argmax_enqueue(c, old, neu))) return r;
    return rb_forward_match_apply_enqueue(c, old, neu, nullptr);
}

int rb_rotate_enqueue(rb_ctx *c, rb_map *m, const double *R_dev) {
    RB_KLAUNCH(k_rotate, rb_div_up(c->kcap, 256), 256, 0, m->kl, (const MapState *)m->st, R_dev, c->zfm);
    return RB_OK;
}

// =====================================================================================================
// directed_matching + search_match (edge_tracker.cpp:158-374)
// =====================================================================================================
#define DM_G 4   // lanes per keyline of the directed search (must divide 32, even)
// The search of new keyline (kpm, krho, ks_rho, km, kn_m) among the old keylines of omask; every lane of the warp calls
// it.  Returns the matched old keyline (or -1) in every lane of the keyline's group.  ROT: the old map is not rotated yet,
// so each candidate is rotated by R here, with the arithmetic of rotate_keylines.
//
// DM_G lanes per keyline: the search along the epipolar segment probes up to 2 * t_steps pixels in a fixed order
// (t_i = 0, 1, ...; for each the near side, then the far side) and stops at the first accepted candidate.  Unmatched
// keylines walk the whole segment, a chain of ~80 dependent lookups; here probe number s = 2 t_i + dir belongs to lane
// s mod DM_G of the keyline's group, the lanes advance in lock step (DM_G probes per iteration) and the lowest lane with
// a hit in an iteration is the first hit of the sequential order.  tp / tn are still built by repeated +-1 (each lane
// takes DM_G / 2 steps per iteration), so every probe sees the same bits as the reference's.
template <bool ROT>
__device__ __forceinline__ int d_dm_search(const KLSoA &old, const int *__restrict__ omask,
                                           const DMatchArgs *__restrict__ ap, const CamC &cam, double min_thr_mod,
                                           double cang_min_edge, double max_radius, double loc_unc, bool valid, int g,
                                           float2 kpm, double krho, double ks_rho, float2 km, float kn_m,
                                           const double (&R)[9]) {
    const int lane = threadIdx.x & 31;
    int jm = -1;
    {
        const double zf = cam.zfm;
        const double *BR = ap->BackRot, *Vel = ap->Vel, *RV = ap->RVel;
        // p_m3 = BackRot*(p_m.x, p_m.y, zfm)
        const double a0 = (double)kpm.x, a1 = (double)kpm.y, a2 = zf;
        double p30 = 0, p31 = 0, p32 = 0;
        p30 = p30 + BR[0] * a0; p30 = p30 + BR[1] * a1; p30 = p30 + BR[2] * a2;
        p31 = p31 + BR[3] * a0; p31 = p31 + BR[4] * a1; p31 = p31 + BR[5] * a2;
        p32 = p32 + BR[6] * a0; p32 = p32 + BR[7] * a1; p32 = p32 + BR[8] * a2;
        const float pmx = (float)(p30 * zf / p32), pmy = (float)(p31 * zf / p32);
        const double k_rho = krho * zf / p32;
        const float pi0x = pmx + cam.ppx, pi0y = pmy + cam.ppy;             // Hom2Img on Point2DF
        double t_x = -(Vel[0] * zf - Vel[2] * (double)pmx);
        double t_y = -(Vel[1] * zf - Vel[2] * (double)pmy);
        double norm_t = sqrt(t_x * t_x + t_y * t_y);
        const double D0 = zf, D1 = zf, D2 = (double)(-pmx - pmy);           // DrDv
        double r0 = 0, r1 = 0, r2 = 0;                                      // DrDv.as_row()*RVel
        r0 = r0 + D0 * RV[0]; r0 = r0 + D1 * RV[3]; r0 = r0 + D2 * RV[6];
        r1 = r1 + D0 * RV[1]; r1 = r1 + D1 * RV[4]; r1 = r1 + D2 * RV[7];
        r2 = r2 + D0 * RV[2]; r2 = r2 + D1 * RV[5]; r2 = r2 + D2 * RV[8];
        double sigma2_t = 0;
        sigma2_t = sigma2_t + r0 * D0; sigma2_t = sigma2_t + r1 * D1; sigma2_t = sigma2_t + r2 * D2;
        double dq_min, dq_max, dq_rho;
        int t_steps;
        if (norm_t > 1e-6) {
            t_x /= norm_t;
            t_y /= norm_t;
            dq_rho = norm_t * k_rho;
            dq_min = fmax(0.0, norm_t * (k_rho - ks_rho)) - loc_unc;
            dq_max = fmin(max_radius, norm_t * (k_rho + ks_rho)) + loc_unc;
            if (dq_rho > dq_max) {
                dq_rho = (dq_max + dq_min) / 2;
                t_steps = (int)(dq_rho + 0.5);
            } else {
                t_steps = (int)(fmax(dq_max - dq_rho, dq_rho - dq_min) + 0.5);
            }
        } else {
            t_x = (double)km.x;
            t_y = (double)km.y;
            norm_t = (double)kn_m;
            t_x /= norm_t;
            t_y /= norm_t;
            norm_t = 1;
            dq_min = -max_radius - loc_unc;
            dq_max = max_radius + loc_unc;
            dq_rho = 0;
            t_steps = (int)dq_max;
        }
        const double norm_m = (double)kn_m;
        double tn = dq_rho, tp = dq_rho + 1;
        int t_i = g >> 1;
        const int dir = g & 1;
        for (int k = 0; k < (g >> 1); k++) {   // this lane's first probe
            tp += 1;
            tn -= 1;
        }
        bool active = valid;
        while (true) {
            int j_hit = -1;
            if (active && t_i < t_steps) {
                const double t = dir ? tp : tn;
                const bool inside = dir ? !(t > dq_max) : !(t < dq_min);
                if (inside) {
                    const float fx = (float)(t_x * t + (double)pi0x), fy = (float)(t_y * t + (double)pi0y);
                    const int xi = (int)roundf(fx), yi = (int)roundf(fy);       // GetIndexRC
                    if (!(xi >= cam.w || yi >= cam.h || xi < 0 || yi < 0)) {
                        const int j = omask[(size_t)yi * cam.w + xi];
                        if (j >= 0) {
                            const double norm_m0 = (double)old.n_m[j];
                            const float2 om = ROT ? d_rot_m(R, old.m_m[j]) : old.m_m[j];
                            const double cang = (double)(om.x * km.x + om.y * km.y) / (norm_m0 * norm_m);
                            if (!(cang < cang_min_edge || fabs(norm_m0 / norm_m - 1) > min_thr_mod)) {
                                double s_rho = old.s_rho[j], rho = old.rho[j];
                                if (ROT) {
                                    const RotPt pt = d_rot_pt(R, zf, old.p_m[j], rho, s_rho);
                                    rho = pt.rho;
                                    s_rho = pt.s_rho;
                                }
                                const double v_rho_dr = (loc_unc * loc_unc + s_rho * s_rho * norm_t * norm_t + sigma2_t * rho * rho);
                                const double e = t - norm_t * rho;
                                if (!(e * e > v_rho_dr)) j_hit = j;
                            }
                        }
                    }
                }
            }
            const unsigned int bal = __ballot_sync(0xffffffffu, j_hit >= 0);
            const unsigned int grp = (bal >> (lane & ~(DM_G - 1))) & ((1u << DM_G) - 1u);
            const int src = grp ? (lane & ~(DM_G - 1)) + __ffs(grp) - 1 : lane;
            const int jw = __shfl_sync(0xffffffffu, j_hit, src);
            if (grp) {   // the lowest lane with a hit = the first accepted probe of the sequential order
                jm = jw;
                active = false;
            }
#pragma unroll
            for (int k = 0; k < DM_G / 2; k++) {
                tp += 1;
                tn -= 1;
            }
            t_i += DM_G / 2;
            if (!__any_sync(0xffffffffu, active && t_i < t_steps)) break;
        }
    }
    return jm;
}
__global__ void __launch_bounds__(128) k_directed_match(KLSoA neu, MapState *nst, KLSoA old,
                                                        const int *__restrict__ omask, const DMatchArgs *__restrict__ ap,
                                                        CamC cam, double min_thr_mod, double cang_min_edge,
                                                        double max_radius, double loc_unc, const int *enable) {
    pdl_wait();
    pdl_launch();
    if (enable && !*enable) return;
    const int gi = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = gi / DM_G, g = gi % DM_G;
    const bool valid = i < nst->kn;
    const int ic = valid ? i : 0;   // (lanes without a keyline run on keyline 0 and never probe)
    const double R[9] = {};
    int jm = d_dm_search<false>(old, omask, ap, cam, min_thr_mod, cang_min_edge, max_radius, loc_unc, valid, g,
                                neu.p_m[ic], neu.rho[ic], neu.s_rho[ic], neu.m_m[ic], neu.n_m[ic], R);
    bool got = false;
    if (g != 0) jm = -1;   // one lane of the group writes
    if (jm >= 0) {                                                     // :343-366
        neu.rho[i] = old.rho[jm];
        neu.s_rho[i] = old.s_rho[jm];
        neu.m_id[i] = jm;
        neu.m_num[i] = old.m_num[jm] + 1;
        neu.p_m_0[i] = old.p_m[jm];
        neu.m_m0[i] = old.m_m[jm];
        neu.n_m0[i] = (double)old.n_m[jm];
        got = true;
    }
    const unsigned int bal = __ballot_sync(0xffffffffu, got);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&nst->nmatch, __popc(bal));
}

// FordwardMatch's apply and directed_matching in one kernel, indexed by new keyline, with the old map still unrotated
// (rb_match_enqueue): the forward winner of keyline i is final in best[i] once the minimiser has run, and the search
// rotates the few old keylines it probes by R0 itself.  The result is the directed hit (rotated) if there is one, else
// the forward winner (unrotated), else nothing.  The keyline's (rho, s_rho) after matching go to reg_r / reg_s for every
// keyline, not to the map: the regularisation that follows reads its neighbours from there (k_reg_ekf).
__global__ void __launch_bounds__(128) k_match(KLSoA neu, MapState *nst, KLSoA old, const int *__restrict__ omask,
                                               const FmBest *best, const DMatchArgs *__restrict__ ap,
                                               const double *__restrict__ Rp, double *__restrict__ reg_r,
                                               double *__restrict__ reg_s, CamC cam, double min_thr_mod,
                                               double cang_min_edge, double max_radius, double loc_unc,
                                               const int *__restrict__ do_match) {
    pdl_wait();
    pdl_launch();
    // (the grid covers the capacity: a block past the map's keylines has nothing to do, not even the search set-up)
    if ((int)(blockIdx.x * (blockDim.x / DM_G)) >= nst->kn) return;
    const int gi = blockIdx.x * blockDim.x + threadIdx.x;
    const int i = gi / DM_G, g = gi % DM_G;
    const bool valid = i < nst->kn;
    const int ic = valid ? i : 0;   // (lanes without a keyline run on keyline 0 and never probe)
    const longlong2 b = __ldcg(reinterpret_cast<const longlong2 *>(best + ic));   // FmBest {key, idx}, 16 bytes
    const float2 kpm = neu.p_m[ic], km = neu.m_m[ic];
    const float kn_m = neu.n_m[ic];
    double R[9];
#pragma unroll
    for (int k = 0; k < 9; k++) R[k] = Rp[k];
    const int fw = valid ? (int)b.y : -1;
    double krho, ks_rho;   // what FordwardMatch leaves in the keyline: the search range depends on it
    if (fw >= 0) {
        krho = old.rho[fw];
        ks_rho = old.s_rho[fw];
    } else {
        krho = neu.rho[ic];
        ks_rho = neu.s_rho[ic];
    }
    int jm = -1;
    if (*do_match)   // (uniform over the grid)
        jm = d_dm_search<true>(old, omask, ap, cam, min_thr_mod, cang_min_edge, max_radius, loc_unc, valid, g, kpm, krho,
                               ks_rho, km, kn_m, R);
    bool got = false;
    if (valid && g == 0) {   // one lane of the group writes
        double rho = krho, s_rho = ks_rho;
        if (jm >= 0) {                                                     // directed_matching :343-366
            const RotPt pt = d_rot_pt(R, cam.zfm, old.p_m[jm], old.rho[jm], old.s_rho[jm]);
            rho = pt.rho;
            s_rho = pt.s_rho;
            neu.m_id[i] = jm;
            neu.m_num[i] = old.m_num[jm] + 1;
            neu.p_m_0[i] = pt.pm;
            neu.m_m0[i] = d_rot_m(R, old.m_m[jm]);
            neu.n_m0[i] = (double)old.n_m[jm];
            got = true;
        } else if (fw >= 0) {                                              // FordwardMatch
            neu.m_id[i] = fw;
            neu.m_num[i] = old.m_num[fw] + 1;
            neu.p_m_0[i] = old.p_m[fw];
            neu.m_m0[i] = old.m_m[fw];
            neu.n_m0[i] = (double)old.n_m[fw];
        }
        reg_r[i] = rho;
        reg_s[i] = s_rho;
    }
    const unsigned int bal = __ballot_sync(0xffffffffu, got);
    const unsigned int fbal = __ballot_sync(0xffffffffu, valid && g == 0 && fw >= 0);
    if ((threadIdx.x & 31) == 0) {
        if (bal) atomicAdd(&nst->nmatch, __popc(bal));
        if (fbal) atomicAdd(&nst->fwd_match, __popc(fbal));
    }
}

int rb_directed_matching_enqueue(rb_ctx *c, rb_map *neu, rb_map *old, const DMatchArgs *args_dev, double min_thr_mod,
                                 double min_thr_ang, double max_radius, double loc_uncertainty, const int *enable_dev) {
    const double cang_min_edge = cos(min_thr_ang * M_PI / 180.0);
    if (!c->counters_preset) {   // the per-frame pipeline zeroes the counters in k_frame_pre
        k_set_int<<<1, 1, 0, c->stream>>>(&neu->st->nmatch, 0);
        RB_LAUNCH_CHECK();
    }
    RB_KLAUNCH(k_directed_match, rb_div_up(c->kcap * DM_G, 128), 128, 0, neu->kl, neu->st, old->kl, old->mask, args_dev,
               make_cam(c), min_thr_mod, cang_min_edge, max_radius, loc_uncertainty, enable_dev);
    return RB_OK;
}
int rb_match_enqueue(rb_ctx *c, rb_map *neu, rb_map *old, const DMatchArgs *args_dev, const double *R_dev,
                     double min_thr_mod, double min_thr_ang, double max_radius, double loc_uncertainty,
                     const int *do_match_dev) {
    const double cang_min_edge = cos(min_thr_ang * M_PI / 180.0);
    const TrackState &t = neu->ts_host;
    RB_KLAUNCH(k_match, rb_div_up(c->kcap * DM_G, 128), 128, 0, neu->kl, neu->st, old->kl, (const int *)old->mask,
               (const FmBest *)t.fm_best, args_dev, R_dev, t.reg_r, t.reg_s, make_cam(c), min_thr_mod, cang_min_edge,
               max_radius, loc_uncertainty, do_match_dev);
    return RB_OK;
}

// =====================================================================================================
// Regularize_1_iter (edge_tracker.cpp:87-148), double buffered like the reference
// =====================================================================================================
// first half of Regularize_1_iter for keyline i, with the (rho, s_rho) of i and its neighbours read from rho / s_rho:
// whether it applies, and if so the smoothed pair in r_out / s_out
__device__ __forceinline__ bool d_reg_vals(const KLSoA &kl, int i, const double *rho, const double *s_rho, double thresh,
                                           double &r_out, double &s_out) {
    bool did = false;
    const int ni = kl.n_id[i], pi = kl.p_id[i];
    if (ni >= 0 && pi >= 0) {
        const double krho = rho[i], ks = s_rho[i];
        const double nrho = rho[ni], ns = s_rho[ni];
        const double prho = rho[pi], ps = s_rho[pi];
        const double d = nrho - prho;
        if (!(d * d > ns * ns + ps * ps)) {
            const float2 nm = kl.m_m[ni], pmv = kl.m_m[pi];
            const float nnm = kl.n_m[ni], pnm = kl.n_m[pi];
            // floats: (kn.m_m.x*kp.m_m.x+kn.m_m.y*kp.m_m.y)/(kn.n_m*kp.n_m) evaluates in float
            double alpha = (double)((nm.x * pmv.x + nm.y * pmv.y) / (nnm * pnm));
            if (!(alpha - thresh < 0)) {
                alpha = (alpha - thresh) / (1 - thresh);
                alpha /= fabs(nrho - prho) / (ns + ps) + 1;
                const double wr = 1 / (ks * ks);
                const double wrn = alpha / (ns * ns);
                const double wrp = alpha / (ps * ps);
                r_out = (krho * wr + nrho * wrn + prho * wrp) / (wr + wrn + wrp);
                s_out = (ks * wr + ns * wrn + ps * wrp) / (wr + wrn + wrp);
                did = true;
            }
        }
    }
    return did;
}
// ... in place: smoothed (rho, s_rho) into r / s, set[i] says whether it applies
__device__ __forceinline__ bool d_reg_a(const KLSoA &kl, int i, double *__restrict__ r, double *__restrict__ s,
                                        unsigned char *__restrict__ set, double thresh) {
    const bool did = d_reg_vals(kl, i, kl.rho, kl.s_rho, thresh, r[i], s[i]);
    set[i] = did ? 1 : 0;
    return did;
}
__global__ void __launch_bounds__(256) k_regularize_a(KLSoA kl, MapState *st, double *__restrict__ r,
                                                      double *__restrict__ s, unsigned char *__restrict__ set,
                                                      double thresh, const int *enable) {
    if (enable && !*enable) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool did = i < st->kn ? d_reg_a(kl, i, r, s, set, thresh) : false;
    const unsigned int bal = __ballot_sync(0xffffffffu, did);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&st->reg_num, __popc(bal));
}
__global__ void __launch_bounds__(256) k_regularize_b(KLSoA kl, const MapState *st, const double *__restrict__ r,
                                                      const double *__restrict__ s,
                                                      const unsigned char *__restrict__ set, const int *enable) {
    if (enable && !*enable) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st->kn || !set[i]) return;
    kl.rho[i] = r[i];
    kl.s_rho[i] = s[i];
}

int rb_regularize_enqueue(rb_ctx *c, rb_map *m, double thresh, const int *enable_dev) {
    TrackState &t = m->ts_host;
    const int nb = rb_div_up(c->kcap, 256);
    if (!c->counters_preset) {   // the per-frame pipeline zeroes the counters in k_frame_pre
        k_set_int<<<1, 1, 0, c->stream>>>(&m->st->reg_num, 0);
        RB_LAUNCH_CHECK();
    }
    k_regularize_a<<<nb, 256, 0, c->stream>>>(m->kl, m->st, t.reg_r, t.reg_s, t.reg_set, thresh, enable_dev);
    RB_LAUNCH_CHECK();
    k_regularize_b<<<nb, 256, 0, c->stream>>>(m->kl, m->st, t.reg_r, t.reg_s, t.reg_set, enable_dev);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// =====================================================================================================
// UpdateInverseDepthKalman -> UpdateInverseDepthKalmanARLU (edge_tracker.cpp:695-724, 954-1055)
// =====================================================================================================
__device__ __forceinline__ void d_ekf(const KLSoA &kl, int i, double rho, double s_rho,
                                      const double *__restrict__ velp, double zf, double q_abs, double loc_unc) {
    const double vel0 = velp[0], vel1 = velp[1], vel2 = velp[2];
    kl.s_rho0[i] = s_rho;
    const float2 pm = kl.p_m[i], pm0 = kl.p_m_0[i], mm0 = kl.m_m0[i];
    const double n_m0 = kl.n_m0[i];
    const double qx = (double)pm.x, qy = (double)pm.y, q0x = (double)pm0.x, q0y = (double)pm0.y;
    double v_rho = s_rho * s_rho;
    const double u_x = (double)mm0.x / n_m0, u_y = (double)mm0.y / n_m0;
    const double Y = u_x * (qx - q0x) + u_y * (qy - q0y);
    const double H = u_x * (vel0 * zf - vel2 * q0x) + u_y * (vel1 * zf - vel2 * q0y);
    const double rho_p = 1 / (1.0 / rho + vel2);
    kl.rho0[i] = rho_p;
    double F = 1 / (1 + rho * vel2);
    F = F * F;
    const double p_p = F * v_rho * F + q_abs * q_abs;
    const double e = Y - H * rho_p;
    const double S = H * p_p * H + loc_unc * loc_unc;
    const double K = p_p * H * (1 / S);
    rho = rho_p + (K * e);
    v_rho = (1 - K * H) * p_p;
    s_rho = sqrt(v_rho);
    if (rho < RB_RHO_MIN) {
        s_rho += RB_RHO_MIN - rho;
        rho = RB_RHO_MIN;
    } else if (rho > RB_RHO_MAX) {
        rho = RB_RHO_MAX;
    } else if (isnan(rho) || isnan(s_rho) || isinf(rho) || isinf(s_rho)) {
        rho = RB_RHO_INIT;
        s_rho = RB_RHO_MAX;
    } else if (s_rho < 0) {
        rho = RB_RHO_INIT;
        s_rho = RB_RHO_MAX;
    }
    kl.rho[i] = rho;
    kl.s_rho[i] = s_rho;
}
__global__ void __launch_bounds__(256) k_ekf(KLSoA kl, const MapState *st, const double *__restrict__ velp, double zf,
                                             double q_abs, double loc_unc, const int *enable) {
    if (enable && !*enable) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st->kn) return;
    if (kl.m_id[i] < 0) return;
    d_ekf(kl, i, kl.rho[i], kl.s_rho[i], velp, zf, q_abs, loc_unc);
}
int rb_ekf_enqueue(rb_ctx *c, rb_map *m, const double *vel_dev, double q_abs, double loc_unc, const int *enable_dev) {
    k_ekf<<<rb_div_up(c->kcap, 256), 256, 0, c->stream>>>(m->kl, m->st, vel_dev, c->zfm, q_abs, loc_unc, enable_dev);
    RB_LAUNCH_CHECK();
    return RB_OK;
}

// pipeline variants (wide grids: these two stages are FP64-heavy per keyline and want every SM):
// first half of Regularize_1_iter with the "after directed_matching" gate folded in (block 0 publishes it) ...
__global__ void __launch_bounds__(256) k_regularize_a_gate(KLSoA kl, MapState *st, double *__restrict__ r,
                                                           double *__restrict__ s, unsigned char *__restrict__ set,
                                                           double thresh, FrameState *fs, int match_threshold) {
    pdl_wait();
    pdl_launch();
    const bool en = fs->do_match && st->nmatch >= match_threshold;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        d_frame_post_match(fs, st, match_threshold);
        st->do_map = fs->do_map;   // for this map's rescaling on the side stream: the next frame rewrites FrameState
    }
    if (!en) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool did = i < st->kn ? d_reg_a(kl, i, r, s, set, thresh) : false;
    const unsigned int bal = __ballot_sync(0xffffffffu, did);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&st->reg_num, __popc(bal));
}
// ... and its write-back half + UpdateInverseDepthKalman in one pass: both only touch the thread's own keyline, so
// the EKF takes the regularised (rho, s_rho) straight from registers
__global__ void __launch_bounds__(256) k_regb_ekf(KLSoA kl, const MapState *st, const double *__restrict__ r,
                                                  const double *__restrict__ s,
                                                  const unsigned char *__restrict__ set,
                                                  const double *__restrict__ velp, double zf, double q_abs,
                                                  double loc_unc, const int *enable, FrameState *pose_fs,
                                                  const MapState *ost, const LMState *lm, rb_nav *nav,
                                                  const FrameArgs *fa) {
    pdl_wait();
    pdl_launch();
    // the frame's pose integration + matrix logarithms (one thread) beside the EKF instead of in the map-update
    // kernel's tail: V and R are final since the gate of the previous kernel.  The last block of the grid has no keylines.
    // With nav, the whole nav record too (the rescaling runs on a side stream and only fills in its Kp / RKp).
    if (pose_fs && blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
        if (nav) d_frame_finish(pose_fs, st, ost, lm->score, nav, fa, false);
        else d_frame_pose(pose_fs);
    }
    if (enable && !*enable) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= st->kn) return;
    double rho, s_rho;
    if (set[i]) {
        rho = r[i];
        s_rho = s[i];
        kl.rho[i] = rho;
        kl.s_rho[i] = s_rho;
    } else {
        rho = kl.rho[i];
        s_rho = kl.s_rho[i];
    }
    if (kl.m_id[i] < 0) return;
    d_ekf(kl, i, rho, s_rho, velp, zf, q_abs, loc_unc);
}
int rb_regularize_ekf_enqueue(rb_ctx *c, rb_map *m, double thresh, FrameState *fs, int match_threshold,
                              const double *vel_dev, double q_abs, double loc_unc, const int *do_map_dev,
                              const MapState *ost, rb_nav *nav, const FrameArgs *fa) {
    TrackState &t = m->ts_host;
    const int nb = rb_div_up(c->kcap, 256);
    RB_KLAUNCH(k_regularize_a_gate, nb, 256, 0, m->kl, m->st, t.reg_r, t.reg_s, t.reg_set, thresh, fs, match_threshold);
    RB_KLAUNCH(k_regb_ekf, nb, 256, 0, m->kl, (const MapState *)m->st, (const double *)t.reg_r, (const double *)t.reg_s,
               (const unsigned char *)t.reg_set, vel_dev, c->zfm, q_abs, loc_unc, do_map_dev, fs, ost,
               (const LMState *)&m->ts->lm, nav, fa);
    return RB_OK;
}

// The map update after k_match, in one pass: every thread evaluates the match-count gate itself (its inputs are final),
// the regularisation reads (rho, s_rho) of a keyline and its neighbours from the scratch pair r / s that k_match filled,
// and the EKF takes the smoothed pair from registers; every keyline's rho / s_rho is written back (the scratch values
// when the gate is closed).  Thread i also runs rotate_keylines(R0) on old keyline i: nothing reads the old map after
// k_match, and the map stays what a caller of the pipeline sees.  One spare thread runs the gate's frame part, then the
// pose integration / nav record, as k_regularize_a_gate and k_regb_ekf do.
__global__ void __launch_bounds__(256) k_reg_ekf(KLSoA kl, MapState *st, const double *__restrict__ r,
                                                 const double *__restrict__ s, double thresh, FrameState *fs,
                                                 int match_threshold, double zf, double q_abs, double loc_unc, KLSoA old,
                                                 const MapState *ost, const double *__restrict__ Rp, const LMState *lm,
                                                 rb_nav *nav, const FrameArgs *fa) {
    pdl_wait();
    pdl_launch();
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
        d_frame_post_match(fs, st, match_threshold);
        st->do_map = fs->do_map;   // for this map's rescaling on the side stream: the next frame rewrites FrameState
        if (nav) d_frame_finish(fs, st, ost, lm->score, nav, fa, false);
        else d_frame_pose(fs);
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < ost->kn) d_rotate(old, i, Rp, zf);
    // (the gate thread above only changes fs->V when the gate is closed, and then no thread reads it)
    const bool en = fs->do_match && st->nmatch >= match_threshold;
    bool did = false;
    if (i < st->kn) {
        double rho = r[i], s_rho = s[i];
        if (en) did = d_reg_vals(kl, i, r, s, thresh, rho, s_rho);
        if (en && kl.m_id[i] >= 0) {
            d_ekf(kl, i, rho, s_rho, fs->V, zf, q_abs, loc_unc);
        } else {
            kl.rho[i] = rho;
            kl.s_rho[i] = s_rho;
        }
    }
    const unsigned int bal = __ballot_sync(0xffffffffu, did);
    if ((threadIdx.x & 31) == 0 && bal) atomicAdd(&st->reg_num, __popc(bal));
}
int rb_reg_ekf_enqueue(rb_ctx *c, rb_map *m, rb_map *old, double thresh, FrameState *fs, int match_threshold,
                       double q_abs, double loc_unc, const double *R_dev, rb_nav *nav, const FrameArgs *fa) {
    const TrackState &t = m->ts_host;
    RB_KLAUNCH(k_reg_ekf, rb_div_up(c->kcap, 256), 256, 0, m->kl, m->st, (const double *)t.reg_r,
               (const double *)t.reg_s, thresh, fs, match_threshold, c->zfm, q_abs, loc_unc, old->kl,
               (const MapState *)old->st, R_dev, (const LMState *)&m->ts->lm, nav, fa);
    return RB_OK;
}



// =====================================================================================================
// Map update of a frame in ONE thread-block cluster: Regularize_1_iter (edge_tracker.cpp:87-148),
// UpdateInverseDepthKalman (:695-724, 954-1055), EstimateReScalingOpt (:1104-1140) and the rescaling itself.
//
// These stages are light per keyline but separated by grid-wide dependencies (the smoothing reads neighbours, each
// of the five rescaling iterations needs sums over all keylines): as separate kernels, or as one kernel exchanging
// through L2, a frame paid far more launch / hand-over latency than arithmetic.  A cluster of 16 CTAs holds
// the whole edge map (thread t of CTA r owns keylines (j*16 + r)*MU_T + t), synchronises with barrier.cluster and
// all-reduces the two sums of an iteration through distributed shared memory: every CTA stores its pair into every
// CTA's slot table, one cluster barrier, every CTA adds the 16 pairs in rank order.  One launch, ~6 cluster barriers.
// Sums: per thread in keyline order, warp xor-tree, warps in order, ranks in order -- fixed, not the reference's
// sequential order (parity to rounding, as for every other reduction here).
// The optional head / tail are the per-frame pipeline's scalar glue (frame.cuh), folded in to save their launches.
// =====================================================================================================
#include <cooperative_groups.h>
namespace cg = cooperative_groups;
#define MU_T 512
#define MU_C 16   // (non-portable cluster size, like the minimiser's)
#define MU_QBINS 128   // largest QCutOffNumBins the folded EstimateQuantile takes
#define MU_KJ 2   // keylines per thread whose rescaling operands stay in registers (kn <= MU_KJ*MU_C*MU_T = 16384)

struct MapUpdArgs {
    int do_reg, do_ekf, do_rescale, re_escale, gate_post_match;
    double reg_thresh;
    const double *vel;       // EKF: translation of the frame (device)
    double zf, q_abs, loc_unc;
    double s_rho_min;        // rescaling
    unsigned int mnm;
    const int *enable;       // stage-level API: run only if *enable (nullptr = run)
    FrameState *fs;          // pipeline: gate = match count (post-match glue folded in), tail = pose integration
    int match_threshold;
    const MapState *ost;
    const LMState *lm;
    rb_nav *nav;
    const FrameArgs *fa;
    // EstimateQuantile of THIS map (what the next frame's loop body starts with, rebvo_second_t.cpp:172) and that loop-body
    // start, folded into the tail: q_bins > 0 enables it
    int q_bins;
    double q_min, q_max, q_perc;
    MapState *nst_next;
    int xchg;                // 1: st.async + mbarrier all-reduce inside the rescaling iterations, 0: barrier.cluster
    rb_nav *kp_nav;          // pipeline, rescaling on the side stream: the record whose Kp / RKp it fills in (no fs)
};

__device__ __forceinline__ void mu_block_sum2(double &a, double &b, double (*sw)[2], int tid) {
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
        sw[wid][0] = a;
        sw[wid][1] = b;
    }
    __syncthreads();
    double x = 0, y = 0;
#pragma unroll
    for (int k = 0; k < MU_T / 32; k++) {
        x += sw[k][0];
        y += sw[k][1];
    }
    a = x;
    b = y;
    __syncthreads();   // sw may be reused
}

__global__ void __cluster_dims__(MU_C, 1, 1) __launch_bounds__(MU_T) k_map_update(KLSoA kl, MapState *st,
                                                                                  double *__restrict__ reg_r,
                                                                                  double *__restrict__ reg_s,
                                                                                  unsigned char *__restrict__ reg_set,
                                                                                  MapUpdArgs a) {
    pdl_wait();
    pdl_launch();
    cg::cluster_group cluster = cg::this_cluster();
    __shared__ double sw[MU_T / 32][2];
    __shared__ __align__(16) double slots[2][MU_C][2];   // [iteration parity][rank][sum]
    __shared__ __align__(8) unsigned long long xbar[2];  // one mbarrier per iteration parity (st.async exchange)
    __shared__ int xfail;
    __shared__ int qh[MU_QBINS];           // EstimateQuantile histogram of this CTA's keylines (rank 0, later: the cluster's)
    __shared__ int qtab[MU_C][MU_QBINS];   // rank 0: every CTA's histogram (plain DSMEM stores: no initialisation to order)
    const int tid = threadIdx.x, rank = (int)cluster.block_rank();
    const int kn = st->kn;
    if (a.q_bins > 0)
        for (int b = tid; b < a.q_bins; b += MU_T) qh[b] = 0;   // (complete before anybody adds: cluster barriers below)
    bool en;
    if (a.fs && a.gate_post_match) {   // "after directed_matching" gate (rebvo_second_t.cpp:410-423) folded in
        en = a.fs->do_match && st->nmatch >= a.match_threshold;
        cluster.sync();   // every CTA has read the gate inputs before CTA 0 rewrites FrameState
        if (rank == 0 && tid == 0) d_frame_post_match(a.fs, st, a.match_threshold);
    } else {
        en = !a.enable || *a.enable;
    }
    const int i0 = rank * MU_T + tid, stride = MU_C * MU_T;
    if (en) {
        // ---- Regularize_1_iter, first half: needs every neighbour's (rho, s_rho) before anybody writes --------
        if (a.do_reg) {
            int cnt = 0;
            for (int i = i0; i < kn; i += stride) cnt += d_reg_a(kl, i, reg_r, reg_s, reg_set, a.reg_thresh) ? 1 : 0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
            if ((tid & 31) == 0 && cnt) atomicAdd(&st->reg_num, cnt);
            cluster.sync();
        }
        // ---- write-back half + EKF: both only touch the thread's own keyline ------------------------------
        if (a.do_reg || a.do_ekf) {
            for (int i = i0; i < kn; i += stride) {
                double rho, s_rho;
                if (a.do_reg && reg_set[i]) {
                    rho = reg_r[i];
                    s_rho = reg_s[i];
                    kl.rho[i] = rho;
                    kl.s_rho[i] = s_rho;
                } else {
                    rho = kl.rho[i];
                    s_rho = kl.s_rho[i];
                }
                if (a.do_ekf && kl.m_id[i] >= 0) d_ekf(kl, i, rho, s_rho, a.vel, a.zf, a.q_abs, a.loc_unc);
            }
        }
        // ---- EstimateReScalingOpt: 5 fixed-point iterations on Kp -----------------------------------------
        if (a.do_rescale) {
            bool valid[MU_KJ];
            double r2[MU_KJ], r02[MU_KJ], s2[MU_KJ], s0v[MU_KJ];
#pragma unroll
            for (int j = 0; j < MU_KJ; j++) {
                const int i = i0 + j * stride;
                valid[j] = false;
                r2[j] = r02[j] = s2[j] = s0v[j] = 0;
                if (i < kn) {
                    const double s0 = kl.s_rho0[i], s = kl.s_rho[i];
                    if (!((unsigned int)kl.m_num[i] < a.mnm || s0 <= 0 || s > a.s_rho_min)) {
                        const double r = kl.rho[i], r0 = kl.rho0[i];
                        valid[j] = true;
                        r2[j] = r * r;
                        r02[j] = r0 * r0;
                        s2[j] = s * s;
                        s0v[j] = s0;
                    }
                }
            }
            // all-reduce of an iteration's two sums: every CTA sends its pair to every CTA with st.async, completion counted on the
            // receiver's mbarrier (as in k_minimizer_cluster): no cluster barrier, no fence inside the five dependent iterations
            // REBVO_B200_MU_XCHG=0: the barrier version (a barrier.cluster per iteration).
            const bool xchg = a.xchg != 0;
            if (xchg) {
                if (tid == 0) {
                    mc_mbar_init(&xbar[0], 1);
                    mc_mbar_init(&xbar[1], 1);
                    xfail = 0;
                    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
                }
                cluster.sync();   // every CTA's barriers exist before anybody sends
            }
            double Kp = 1.0, RKp = 0;
            for (int iter = 0; iter < 5; iter++) {
                if (xchg && tid == 0) mc_mbar_expect_tx(&xbar[iter & 1], MU_C * 16u);
                double sa = 0, sb = 0;
#pragma unroll
                for (int j = 0; j < MU_KJ; j++)
                    if (valid[j]) {   // r*r/den and r0*r0/den through one reciprocal (div_with_rcp == IEEE division)
                        const double den = s2[j] + Kp * Kp * s0v[j] * s0v[j];
                        const double iden = 1 / den;
                        sa += div_with_rcp(r2[j], den, iden);
                        sb += div_with_rcp(r02[j], den, iden);
                    }
                for (int i = i0 + MU_KJ * stride; i < kn; i += stride) {   // maps beyond the register window
                    const double s0 = kl.s_rho0[i], s = kl.s_rho[i];
                    if (!((unsigned int)kl.m_num[i] < a.mnm || s0 <= 0 || s > a.s_rho_min)) {
                        const double r = kl.rho[i], r0 = kl.rho0[i];
                        const double den = s * s + Kp * Kp * s0 * s0;
                        sa += r * r / den;
                        sb += r0 * r0 / den;
                    }
                }
                mu_block_sum2(sa, sb, sw, tid);
                if (xchg) {
                    if (tid < MU_C)
                        mc_st_async_v2(mc_mapa(mc_smem_u32(&slots[iter & 1][rank][0]), (unsigned int)tid), sa, sb,
                                       mc_mapa(mc_smem_u32(&xbar[iter & 1]), (unsigned int)tid));
                    if (tid < 32) {   // one warp waits for the 16 pairs, the block follows through the barrier below
                        const long long t0 = clock64();
                        while (!mc_mbar_try_wait(&xbar[iter & 1], (unsigned int)(iter >> 1) & 1u))
                            if (clock64() - t0 > (1ll << 28)) {
                                xfail = 1;
                                break;
                            }
                    }
                    __syncthreads();
                } else {
                    if (tid < MU_C) {   // this CTA's pair into every CTA's table
                        double *dst = cluster.map_shared_rank(&slots[iter & 1][rank][0], tid);
                        dst[0] = sa;
                        dst[1] = sb;
                    }
                    cluster.sync();
                }
                double rTr = 0, rTr0 = 0;
#pragma unroll
                for (int k = 0; k < MU_C; k++) {
                    rTr += slots[iter & 1][k][0];
                    rTr0 += slots[iter & 1][k][1];
                }
                if (kn > 0) {   // "if(kn<=0) return 1;"
                    Kp = rTr0 > 0 ? sqrt(rTr / rTr0) : 1;
                    RKp = 1 / rTr0;
                }
            }
            if (xchg && xfail) Kp = RKp = __longlong_as_double(0x7FF8000000000000ll);   // (an exchange timed out: poison, do not hang)
            if (a.re_escale)
                for (int i = i0; i < kn; i += stride) {
                    kl.rho[i] = kl.rho[i] / Kp;
                    kl.s_rho[i] = kl.s_rho[i] / Kp;
                }
            if (rank == 0 && tid == 0) {
                st->Kp = Kp;
                if (kn > 0) st->RKp = RKp;
                if (a.kp_nav) {   // what d_frame_finish takes into the record after a rescaling
                    a.kp_nav->Kp = st->Kp;
                    a.kp_nav->RKp = st->RKp;
                }
            }
        }
    }
    if (a.q_bins > 0) {   // EstimateQuantile (edge_finder.cpp: histogram of s_rho over all keylines) on the final s_rho of this map
        __syncthreads();   // (qh zeroed; this thread's own s_rho writes are visible to it)
        const double range = a.q_max - a.q_min;
        for (int i = i0; i < kn; i += stride) {
            int b = (int)((double)a.q_bins * (kl.s_rho[i] - a.q_min) / range);
            b = b > a.q_bins - 1 ? a.q_bins - 1 : b;
            b = b < 0 ? 0 : b;
            atomicAdd(&qh[b], 1);
        }
        __syncthreads();
        int *t0 = cluster.map_shared_rank(&qtab[rank][0], 0);
        for (int b = tid; b < a.q_bins; b += MU_T) t0[b] = qh[b];
    }
    cluster.sync();   // no CTA may exit while a peer can still store into its shared memory
    if (rank == 0 && a.q_bins > 0) {
        for (int b = tid; b < a.q_bins; b += MU_T) {
            int t = 0;
#pragma unroll
            for (int r = 0; r < MU_C; r++) t += qtab[r][b];
            qh[b] = t;
        }
        __syncthreads();
    }
    if (rank == 0 && tid == 0) {
        if (a.fs && a.nav) d_frame_finish(a.fs, st, a.ost, a.lm->score, a.nav, a.fa, true);
        if (a.q_bins > 0) {
            const double range = a.q_max - a.q_min;
            double q = 1e3;
            for (int i = 0, acc = 0; i < a.q_bins; i++) {
                if ((double)acc > a.q_perc * (double)kn) {
                    q = (double)i * range / (double)a.q_bins + a.q_min;
                    break;
                }
                acc += qh[i];
            }
            st->s_rho_q = q;
            if (a.fs && a.nst_next) d_frame_pre(a.fs, a.fa->next_frame_count, a.nst_next);   // loop-body start of the next frame
        }
    }
}

static int launch_map_update(rb_ctx *c, rb_map *m, const MapUpdArgs &a_in, bool pdl) {
    MapUpdArgs a = a_in;
    a.xchg = c->mu_xchg ? 1 : 0;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(MU_C);
    cfg.blockDim = dim3(MU_T);
    cfg.stream = c->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    TrackState &t = m->ts_host;
    c->launches++;
    RB_CUDA(cudaLaunchKernelEx(&cfg, k_map_update, m->kl, m->st, t.reg_r, t.reg_s, t.reg_set, a));
    return RB_OK;
}

// the pipeline's whole map update (gate, smoothing, EKF, rescaling, pose integration / nav record)
int rb_map_update_enqueue(rb_ctx *c, rb_map *m, double reg_thresh, const double *vel_dev, double q_abs, double loc_unc,
                          double s_rho_min, unsigned int match_num_min, int re_escale, FrameState *fs,
                          int match_threshold, const MapState *ost, rb_nav *nav, const FrameArgs *fa, bool fused,
                          const rb_quantile_fold *qf) {
    MapUpdArgs a;
    memset(&a, 0, sizeof(a));
    // fused: the match-count gate, Regularize_1_iter and the EKF run inside this cluster kernel too (one launch instead of
    // three); otherwise the pipeline has run them on wide grids (rb_regularize_ekf_enqueue) and published fs->do_map
    a.do_reg = a.do_ekf = fused ? 1 : 0;
    a.do_rescale = 1;
    a.re_escale = re_escale;
    a.reg_thresh = reg_thresh;
    a.vel = vel_dev;
    a.zf = c->zfm;
    a.q_abs = q_abs;
    a.loc_unc = loc_unc;
    a.s_rho_min = s_rho_min;
    a.mnm = match_num_min;
    a.fs = fs;
    a.enable = &fs->do_map;   // published by k_regularize_a_gate
    a.gate_post_match = fused ? 1 : 0;
    a.match_threshold = match_threshold;
    a.ost = ost;
    a.lm = &m->ts->lm;
    a.nav = nav;
    a.fa = fa;
    if (qf && qf->nbins > 0 && qf->nbins <= MU_QBINS) {
        a.q_bins = qf->nbins;
        a.q_min = qf->smin;
        a.q_max = qf->smax;
        a.q_perc = qf->perc;
        a.nst_next = qf->nst_next;
    }
    return launch_map_update(c, m, a, c->pdl);
}

// EstimateReScalingOpt alone (stage-level API, and the per-frame pipeline's side stream with kp_nav): the same kernel with
// only its last phase, hence the same bits.  Launched without programmatic serialization: on the side stream it must not
// become resident (16 SMs spinning in griddepcontrol.wait) while the tracker stream's kernels still run.
int rb_rescale_enqueue(rb_ctx *c, rb_map *m, double s_rho_min, unsigned int match_num_min, int re_escale,
                       const int *enable_dev, rb_nav *kp_nav) {
    MapUpdArgs a;
    memset(&a, 0, sizeof(a));
    a.do_rescale = 1;
    a.re_escale = re_escale;
    a.s_rho_min = s_rho_min;
    a.mnm = match_num_min;
    a.enable = enable_dev;
    a.kp_nav = kp_nav;
    return launch_map_update(c, m, a, false);
}

// per-device opt-in of the mapper's 16-CTA cluster kernel (called from rb_minimizer_cluster_setup at context creation)
void rb_mapper_cluster_setup() {
    cudaFuncSetAttribute(k_map_update, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    cudaGetLastError();
}

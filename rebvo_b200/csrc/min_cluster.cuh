// min_cluster.cuh -- global_tracker::Minimizer_RV (src/mtracklib/global_tracker.cpp:578-819) in ONE thread-block
// cluster.  Included by tracker.cu after the per-keyline body (tvr_keyline) and the LM pieces (lm_*).
//
// A minimisation is ~12 TryVelRot evaluations, each a sum over all old keylines followed by a 6x6 LM step whose result
// is the next evaluation's pose: a chain of grid-wide reductions.  Exchanging through L2 between ~65 independent
// blocks cost two L2 round trips + a 65 x 59-slot gather per evaluation (2/3 of the kernel).  Here the whole edge map
// lives in one cluster of MC_C CTAs (guaranteed co-resident by the cluster launch, so nothing can dead-lock when
// several pipelines share a GPU):
//   * CTA r owns the contiguous keylines [r*kpc, (r+1)*kpc); their pose-independent operands (back-projected point,
//     s_rho) and the three residual buffers Res0/Res1/Rest stay in shared memory for the whole minimisation;
//   * per evaluation every CTA reduces its 28 sums + stale-fi summary and sends them to EVERY CTA of the cluster with
//     st.async (distributed shared memory, completion counted on the receiver's mbarrier: no cluster-wide barrier,
//     no fence, L1 stays valid); every CTA adds the MC_C contributions in rank order and runs the LM step itself --
//     all CTAs compute bit-identical poses, so there is no request broadcast at all;
//   * the zero-initialised and the prior-initialised tries of init type 2 (:644-751) are independent of each other
//     (no re-weighting, different output buffers Rest / ResidualNew): both poses are evaluated in the same round and
//     their LM steps run on two warps side by side, so 2*(init_iter+1) dependent rounds become init_iter+1.
// Sums: per thread in keyline order, transposing warp butterfly, warps in order, ranks in order -- fixed, deterministic,
// not the reference's pairwise tree (tests: rel 1e-10 on JtJ/JtF, V/W abs 1e-9).
// The kernel is a template over the CTA size T: 512 threads for the one-cluster form, 256 for the multi-cluster form.
#pragma once

#define MC_C 16                      // CTAs per cluster (non-portable size, one CTA per SM)
#define MC_GMAX 8                    // clusters of one minimisation
#define MC_PW 30                     // doubles per pose and CTA in the exchange: 28 sums, has-a-match, last matched fi
#define MC_XW 60
#ifndef MC_KPC_FAST
#define MC_KPC_FAST 1280               // keylines per CTA kept in shared memory (16 x 1280 = 20480 per edge map); see McView
#endif
#define MC_SPIN_LIMIT (1ll << 29)    // ~0.27 s: a broken exchange aborts with NaN results instead of hanging the device
#define MC_BYTES_PER_KL 57           // x0,y0,z0,s_rho, 3 residual buffers (double) + 1 flag byte
#define MC_KPC_MAX 3584              // keylines per CTA at most: MC_C * MC_KPC_MAX = 57344 >= KEYLINE_MAX
#define MC_NV (MC_KPC_MAX / 32)      // "virtual warps" of a CTA (32 consecutive keylines each)

#ifdef RB_TVR_PROF   // stamps: [CTA][round (15 = kernel level)][16]
#define MC_STAMP(e, k) do { if (threadIdx.x == 0 && blockIdx.x < 16) g_tvr_prof[(blockIdx.x * 16 + (e)) * 16 + (k)] = clock64(); } while (0)
#else
#define MC_STAMP(e, k) do { } while (0)
#endif
#ifdef RB_TVR_PROF   // %globaltimer of "sums published" / "column gathered" per CTA and round (inter-cluster skew vs mechanism)
__device__ long long g_mc_gt[128 * 16 * 2];
extern "C" int rb_debug_fetch_gt(long long *out) { return (int)cudaMemcpyFromSymbol(out, g_mc_gt, sizeof(g_mc_gt)); }
#define MC_GT(e, k) do { if (threadIdx.x == 0 && blockIdx.x < 128) g_mc_gt[(blockIdx.x * 16 + (e)) * 2 + (k)] = tvr_gtime(); } while (0)
#else
#define MC_GT(e, k) do { } while (0)
#endif

struct McPlan {
    int n, merge_round;              // merge_round: the round after which the better init try is picked (-1: none)
    unsigned char sa[MIN_MAX_ROUNDS];   // zero-init try's step of the round (STEP_NONE when the round has one pose)
    unsigned char sb[MIN_MAX_ROUNDS];   // prior-init try / main loop step
};

__device__ __forceinline__ unsigned int mc_smem_u32(const void *p) { return (unsigned int)__cvta_generic_to_shared(p); }
__device__ __forceinline__ unsigned int mc_mapa(unsigned int addr, unsigned int rank) {
    unsigned int r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ unsigned int mc_cluster_rank() {
    unsigned int r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void mc_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void mc_st_async_v2(unsigned int raddr, double a, double b, unsigned int rmbar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v2.f64 [%0], {%1, %2}, [%3];" ::"r"(raddr),
                 "d"(a), "d"(b), "r"(rmbar)
                 : "memory");
}
__device__ __forceinline__ void mc_mbar_init(unsigned long long *bar, unsigned int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mc_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mc_mbar_expect_tx(unsigned long long *bar, unsigned int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mc_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mc_mbar_try_wait(unsigned long long *bar, unsigned int parity) {
    unsigned int ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(mc_smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}

// This CTA's slice of the edge map.  The first S keylines of the slice live in dynamic shared memory (operands +
// residual buffers); S is sized for the maps the detector's auto-gain actually produces (ReferencePoints ~ 15 k), not
// for the capacity MaxPoints: the gathers through the field image only stay L1-resident between evaluations if the
// unified L1/shared array is not all shared memory.  Keylines beyond S (rare) re-load their operands from the global
// SoA and keep their residuals in the global residual buffers.
struct McView {
    double *x0, *y0, *z0, *s_rho;
    double *res[3];
    unsigned char *flag;  // 1: m_num < min(MatchNumThresh, FrameCount)
    double *gres[3];      // global Res0 / Res1 / Rest (overflow keylines)
    int S;
    int base, cnt, J;     // first keyline, keylines of this CTA, iterations per thread (uniform over the cluster)
};

// ---- a chain's LM variables in the registers of its warp (warp 0: main / prior-init chain, warp 1: zero-init chain) -----
// Lane k < 27 holds sum k in the layout the totals arrive in (k < 21: the upper triangle of JtJ row by row, 21..26: JtF):
// `acc` the accepted JtJ / JtF, `nw` the newest evaluation's JtJn / JtFn, so accepting a step is a select per lane instead
// of a 42-element copy.  Lanes 0-5 hold X, Xnew and h; the scalars are warp-uniform (every lane evaluates the same
// expression).  The LMState in shared memory is the hand-off: the merge reads the zero-init chain's try from it, and the
// epilogue reads the main chain from it once the rounds are over.  Fields nothing reads during the rounds (Xeval, res_in /
// res_out, Fnew, gain, last_score, Xt ..) are stored there as they are produced and never loaded back.
struct McChain {
    double acc, nw;        // lane k < 27: JtJ | JtF, JtJn | JtFn
    double x, xn, h;       // lane i < 6: X[i], Xnew[i], h[i]
    double F, F0, u, v;
    int eff, iR, iRN, iRt, n_eval;
};
struct McReq {             // the pose a step requests (uniform): Xeval and its residual buffers
    double x[6];
    int ri, ro;
};
#define MC_FULL 0xffffffffu
__device__ __forceinline__ int mc_up_row(int k) { return k < 6 ? 0 : k < 11 ? 1 : k < 15 ? 2 : k < 18 ? 3 : k < 20 ? 4 : 5; }
__device__ __forceinline__ int mc_up_col(int k, int a) {
    return k - (a == 0 ? 0 : a == 1 ? 6 : a == 2 ? 11 : a == 3 ? 15 : a == 4 ? 18 : 20) + a;
}
__device__ __forceinline__ double mc_lane6(const double (&a)[6], int lane) {   // a[lane] for lanes 0-5, no local memory
    double r = a[0];
#pragma unroll
    for (int i = 1; i < 6; i++) r = lane == i ? a[i] : r;
    return r;
}
__device__ __forceinline__ void mc_gather6(double v, double (&a)[6]) {   // lanes 0-5's v to every lane
#pragma unroll
    for (int i = 0; i < 6; i++) a[i] = __shfl_sync(MC_FULL, v, i);
}
__device__ __forceinline__ void mc_chain_load(McChain &c, const LMState &L, int lane) {
    {   // (every field is assigned on every lane, so nothing of the previous contents stays live)
        const int k = lane < 27 ? lane : 0;
        const int a = mc_up_row(k), b = mc_up_col(k, a);
        const int ij = k < 21 ? a * 6 + b : 0, jf = k < 21 ? 0 : k - 21;
        c.acc = k < 21 ? L.JtJ[ij] : L.JtF[jf];
        c.nw = k < 21 ? L.JtJn[ij] : L.JtFn[jf];
    }
    const int i = lane < 6 ? lane : 0;
    c.x = L.X[i];
    c.xn = L.Xnew[i];
    c.h = L.h[i];
    c.F = L.F;
    c.F0 = L.F0;
    c.u = L.u;
    c.v = L.v;
    c.eff = L.eff_steps;
    c.iR = L.iR;
    c.iRN = L.iRN;
    c.iRt = L.iRt;
    c.n_eval = L.n_eval;
}
__device__ __forceinline__ void mc_chain_store(const McChain &c, LMState &L, int lane) {
    if (lane < 21) {
        const int a = mc_up_row(lane), b = mc_up_col(lane, a);
        L.JtJ[a * 6 + b] = c.acc;
        L.JtJ[b * 6 + a] = c.acc;
        L.JtJn[a * 6 + b] = c.nw;
        L.JtJn[b * 6 + a] = c.nw;
    } else if (lane < 27) {
        L.JtF[lane - 21] = c.acc;
        L.JtFn[lane - 21] = c.nw;
    }
    if (lane < 6) {
        L.X[lane] = c.x;
        L.Xnew[lane] = c.xn;
        L.h[lane] = c.h;
    }
    if (lane == 0) {
        L.F = c.F;
        L.F0 = c.F0;
        L.u = c.u;
        L.v = c.v;
        L.eff_steps = c.eff;
        L.iR = c.iR;
        L.iRN = c.iRN;
        L.iRt = c.iRt;
        L.n_eval = c.n_eval;
    }
}
// lm_request: the pose of the next evaluation; Xeval also goes to shared memory, where warps 3 / 4 read W.z
__device__ __forceinline__ void mc_request(McReq &q, LMState &L, const double (&X)[6], int ri, int ro, int lane) {
#pragma unroll
    for (int i = 0; i < 6; i++) q.x[i] = X[i];
    q.ri = ri;
    q.ro = ro;
    if (lane < 6) L.Xeval[lane] = mc_lane6(X, lane);
    if (lane == 0) {
        L.res_in = ri;
        L.res_out = ro;
    }
}
// F = TryVelRot(JtJ, JtF, X ...); F0 = F; u = tau*max_element(JtJ).  A row-by-row scan of JtJ keeps the first of the
// largest elements (a NaN is skipped unless it is JtJ[0]); the upper triangle in row order has the same first maximum
// (a mirrored element repeats an earlier one), and a butterfly that keeps the earlier operand unless the later one is
// larger, NaN as "no element", finds it in any grouping.
__device__ __forceinline__ void mc_take_first(McChain &c, double last, int lane) {
    c.F = last;
    c.acc = c.nw;
    c.F0 = c.F;
    double m = lane < 21 ? c.acc : __longlong_as_double(0x7FF8000000000000ll);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double q = __shfl_xor_sync(MC_FULL, m, o);
        const bool hi = (lane & o) != 0;
        const double lo_v = hi ? q : m, hi_v = hi ? m : q;
        m = isnan(lo_v) ? hi_v : (hi_v > lo_v ? hi_v : lo_v);
    }
    const double m0 = __shfl_sync(MC_FULL, c.acc, 0);
    c.u = 1e-3 * (isnan(m0) ? m0 : m);
}
// gain, then accept (F, X, JtJ / JtF from the evaluation, u shrinks) or reject (u *= v, v *= 2); returns true when the
// step was accepted
__device__ __forceinline__ bool mc_update(McChain &c, LMState &L, double last, bool gain_with_den, int lane) {
    const double Fnew = last;
    double gain;
    if (gain_with_den) {
        const double jf = __shfl_sync(MC_FULL, c.acc, (lane + 21) & 31);   // JtF[lane]
        const double p = (0.5 * c.h) * (c.u * c.h - jf);
        double den = 0;   // 0.5*h*(u*h-JtF): TooN dot of (0.5*h) and (u*h-JtF), left to right
#pragma unroll
        for (int i = 0; i < 6; i++) den += __shfl_sync(MC_FULL, p, i);
        gain = (c.F - Fnew) / den;
    } else {
        gain = c.F - Fnew;
    }
    if (lane == 0) {
        L.Fnew = Fnew;
        L.gain = gain;
    }
    if (gain > 0) {
        c.F = Fnew;
        c.x = c.xn;
        c.acc = c.nw;
        const double g = 2 * gain - 1;
        const double f = 1 - (g * g * g);
        c.u *= (0.33 > f ? 0.33 : f);  // std::max(0.33, ...)
        c.v = 2;
        c.eff++;
        return true;
    }
    c.u *= c.v;
    c.v *= 2;
    return false;
}
// h = (JtJ + u I)^-1 (-JtF), Xnew = X + h.  Every lane gathers ApI and factors it (lm.cuh's ldlt_factor / ldlt_backsub,
// without the zero-pivot stop; the same operations in the same order), so h and Xnew need no broadcast.  The main loop
// solves with Cholesky<6> (:766-767), the init tries with SVD<> (:659-661): where ldlt_solves_like_svd accepts the pivots,
// ApI is SPD with a condition number far below SVD.h's 1e9 cut, so the pseudo-inverse is the inverse and the LDL^T solve
// returns the same vector up to rounding; otherwise the Jacobi pseudo-inverse (lm_solve_fallback) solves, serial and cold.
__device__ __forceinline__ void mc_solve(McChain &c, LMState &L, bool use_svd, int lane, double (&xn)[6]) {
    double A[36], a[36], rhs[6], hh[6], xg[6], dmin, dmax;
    mc_gather6(c.x, xg);
#pragma unroll
    for (int a = 0; a < 6; a++)
#pragma unroll
        for (int b = a; b < 6; b++) {
            const double t = __shfl_sync(MC_FULL, c.acc, a * 6 - a * (a - 1) / 2 + (b - a));
            A[a * 6 + b] = t;
            A[b * 6 + a] = t;
        }
#pragma unroll
    for (int i = 0; i < 6; i++) {
        A[i * 6 + i] = A[i * 6 + i] + c.u;  // ApI = JtJ + Identity*u
        rhs[i] = -__shfl_sync(MC_FULL, c.acc, 21 + i);
    }
    ldlt_factor<6, false>(A, a, dmin, dmax);
    ldlt_backsub<6>(a, rhs, hh);
    if (use_svd && !ldlt_solves_like_svd(dmin, dmax)) {   // (uniform) rank-deficient ApI: SVD<> pseudo-inverse semantics
        if (lane < 21) {
            const int a = mc_up_row(lane), b = mc_up_col(lane, a);
            L.JtJ[a * 6 + b] = c.acc;
            L.JtJ[b * 6 + a] = c.acc;
        } else if (lane < 27) {
            L.JtF[lane - 21] = c.acc;
        }
        if (lane == 0) L.u = c.u;
        __syncwarp();
        if (lane == 0) lm_solve_fallback(L);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 6; i++) hh[i] = L.h[i];
        __syncwarp();
    }
#pragma unroll
    for (int i = 0; i < 6; i++) xn[i] = xg[i] + hh[i];
    c.h = mc_lane6(hh, lane);
    c.xn = mc_lane6(xn, lane);
}
// the LM step of a chain after an evaluation (global_tracker.cpp:651-683 zero-initialised try, :700-732 prior-initialised
// try, :755-816 main loop).  Returns whether it requested a pose; *fin: the main loop ended (lm_finalize follows the
// rounds).
__device__ __forceinline__ bool mc_step(McChain &c, McReq &q, LMState &L, int step, double last, int init_iter,
                                        int iter_max, bool &fin, int lane) {
    if (step == STEP_NONE) return false;
    const bool zero = step <= STEP_INIT_LAST_ZERO, init = step < STEP_MAIN_FIRST;
    const bool first = step == STEP_INIT_FIRST_ZERO || step == STEP_INIT_FIRST_PRIOR || step == STEP_MAIN_FIRST;
    const bool init_last = step == STEP_INIT_LAST_ZERO || step == STEP_INIT_LAST_PRIOR;
    if (first) {
        mc_take_first(c, last, lane);
        if (!zero) c.v = 2;   // (zero-init try: v = 2 from the declaration, :620)
    } else if (mc_update(c, L, last, !init_last, lane) && !init) {   // main loop: std::swap(ResidualNew,Residual)
        const int t = c.iRN;
        c.iRN = c.iR;
        c.iR = t;
    }
    // a first step solves when its loop iterates at all; the last step of each loop solves nothing
    const bool solve = first ? (init ? init_iter > 0 : iter_max > 0) : !(init_last || step == STEP_MAIN_LAST);
    fin = fin || (!init && !solve);
    if (!solve) return false;
    double xn[6];
    mc_solve(c, L, init, lane, xn);   // (init tries: SVD<> semantics; main loop: Cholesky<6>)
    mc_request(q, L, xn, init ? -1 : c.iR, zero ? c.iRt : c.iRN, lane);
    return true;
}
// "Save the scores in temporals" (:686-691) + "Check for the lowest score" (:734-747) once both tries are done: the
// main chain's warp reads the zero-init chain's try from z (which its warp stored before the named barrier)
__device__ __forceinline__ void mc_merge(McChain &c, McReq &q, LMState &s, const LMState &z, int lane) {
    const double Xt = z.X[lane < 6 ? lane : 0];
    const double Ft = z.F, F0t = z.F0, ut = z.u, vt = z.v;
    const int eff_t = z.eff_steps;
    if (lane < 6) s.Xt[lane] = Xt;
    if (lane == 0) {
        s.Ft = Ft;
        s.F0t = F0t;
        s.ut = ut;
        s.vt = vt;
        s.eff_steps_t = eff_t;
    }
    if (c.F > Ft) {
        c.x = Xt;
        c.F = Ft;
        c.F0 = F0t;
        c.u = ut;
        c.v = vt;
        c.eff = eff_t;
        c.iRN = c.iRt;
    }
    const int t = c.iRN;
    c.iRN = c.iR;
    c.iR = t;
    double X[6];
    mc_gather6(c.x, X);
    mc_request(q, s, X, c.iR, c.iRN, lane);
}
__device__ __forceinline__ void mc_merge_publish(const McChain &z, LMState &Z, int lane) {   // what mc_merge reads
    if (lane < 6) Z.X[lane] = z.x;
    if (lane == 0) {
        Z.F = z.F;
        Z.F0 = z.F0;
        Z.u = z.u;
        Z.v = z.v;
        Z.eff_steps = z.eff;
    }
}


// ---- exchange between clusters: self-validating 8-byte {sequence number, payload word} slots in global memory ----------
// (a poller that sees the sequence number has the payload: no fence, no counter -- the NCCL-LL idea).  A double takes two
// slots.  Slot block of (round parity, cluster, rank, pose): 64 words.
__device__ __forceinline__ unsigned long long *mc_slots(unsigned long long *ll, int G, int par, int c, int rank, int p) {
    return ll + ((size_t)(((par * G + c) * MC_C + rank) * 2 + p)) * 64;
}
__device__ __forceinline__ void mc_slot_put(unsigned long long *s, int k, unsigned int seq, double v) {
    st_volatile_u64(s + 2 * k, ((unsigned long long)seq << 32) | (unsigned int)__double2loint(v));
    st_volatile_u64(s + 2 * k + 1, ((unsigned long long)seq << 32) | (unsigned int)__double2hiint(v));
}
// value k of every other cluster's same-rank CTA; own value at position c.  false: timed out
__device__ __forceinline__ bool mc_slot_gather(unsigned long long *ll, int G, int par, int c, int rank, int p, int k,
                                               unsigned int seq, double own, double (&v)[MC_GMAX]) {
    bool done[MC_GMAX];
#pragma unroll
    for (int q = 0; q < MC_GMAX; q++) {
        done[q] = q >= G || q == c;
        v[q] = q == c ? own : 0.0;
    }
    const long long t0 = clock64();
    for (;;) {
        bool all = true;
#pragma unroll
        for (int q = 0; q < MC_GMAX; q++)
            if (!done[q]) {
                const unsigned long long *s = mc_slots(ll, G, par, q, rank, p);
                unsigned long long lo, hi;   // one 16-byte request for the two slots (each slot validates itself)
                asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];" : "=l"(lo), "=l"(hi) : "l"(s + 2 * k) : "memory");
                if ((unsigned int)(lo >> 32) == seq && (unsigned int)(hi >> 32) == seq) {
                    v[q] = __hiloint2double((int)(unsigned int)hi, (int)(unsigned int)lo);
                    done[q] = true;
                } else {
                    all = false;
                }
            }
        if (all) return true;
        if (clock64() - t0 > MC_SPIN_LIMIT) return false;
    }
}
template <int T>
struct __align__(16) McSmem {
    double gather[2][MC_C][MC_XW];   // [round parity][source rank][value]
    double part[T / 32][32];
    double xout[64];
    double xcol[64];                 // column sums (this CTA's sums + those of the equal-rank CTAs of the other clusters)
    double req[2][16];               // per pose: R[9] V[3] RotM[4]
    int req_res[2][2];               // per pose: res_in, res_out
    double wcarry[3][MC_NV];         // per residual buffer: the stale fi that leading misses of a virtual warp inherit
    double vw_last[2][MC_NV];
    int vw_has[2][MC_NV];
    unsigned long long mbar[2];
    LMState lm, lmz;                 // main / prior-init chain, zero-init chain
    int abort;
};

// one TryVelRot evaluation of pose slot p over this CTA's keylines; leaves the CTA's 28 sums and stale-fi summary in
// sm.xout[p * MC_PW ..]
template <int T, bool RW, bool PJ>
__device__ __forceinline__ void mc_eval_pose(McSmem<T> &sm, const McView &v, int p, const KLSoA &old, const TvrConst &tc,
                                             const CamC &cam, const unsigned long long *__restrict__ field,
                                             const float4 *__restrict__ fpack, bool write_mid, int tid, int lane,
                                             int wid) {
    const double *sR = sm.req[p], *sV = sR + 9, *sRM = sR + 12;
    const int res_in = sm.req_res[p][0], res_out = sm.req_res[p][1];
    const bool has_rin = RW && res_in >= 0;
    const double *rin = v.res[has_rin ? res_in : 0], *grin = v.gres[has_rin ? res_in : 0];
    double *rout = v.res[res_out], *grout = v.gres[res_out];
    int *mid_out = write_mid ? old.m_id_f : nullptr;
    constexpr int U = 1;   // keylines of a thread evaluated side by side (2, 3 measured slower: register pressure)
    double acc[28];
#pragma unroll
    for (int k = 0; k < 28; k++) acc[k] = 0;
    MC_BSTAMP(10);
    for (int j0 = 0; j0 < v.J; j0 += U) {
        if (j0 == U) MC_BSTAMP(11);
        double x0[U], y0[U], z0[U], s_rho[U], r_prev[U], fi_own[U];
        float2 m[U];
        float n_m[U];
        bool skip[U], act[U], matched[U], need[U], outside[U];
        int gi[U], li[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            li[u] = (j0 + u) * T + tid;
            gi[u] = v.base + li[u];
            act[u] = li[u] < v.cnt;
            // lanes without a keyline run on harmless operands and contribute exact zeros
            x0[u] = y0[u] = 0.0;
            z0[u] = s_rho[u] = 1.0;
            m[u] = make_float2(0.f, 0.f);
            n_m[u] = 0.f;
            bool fl = false;
            if (act[u]) {
                if (li[u] < v.S) {
                    x0[u] = v.x0[li[u]];
                    y0[u] = v.y0[li[u]];
                    z0[u] = v.z0[li[u]];
                    s_rho[u] = v.s_rho[li[u]];
                    fl = v.flag[li[u]] != 0;
                } else {
                    const KlOp o = load_klop(old, gi[u], cam);
                    x0[u] = o.x0;
                    y0[u] = o.y0;
                    z0[u] = o.z0;
                    s_rho[u] = o.s_rho;
                    fl = (unsigned int)o.m_num < tc.mnt;
                }
                m[u] = __ldg(&old.m_m[gi[u]]);
                n_m[u] = __ldg(&old.n_m[gi[u]]);
            }
            skip[u] = !act[u] || s_rho[u] > tc.s_rho_min || fl;   // :356
            double r = 0.0;
            if (has_rin && act[u]) {
                r = li[u] < v.S ? rin[li[u]] : grin[gi[u]];
                if ((unsigned long long)__double_as_longlong(r) == RES_SENTINEL) r = sm.wcarry[res_in][(j0 + u) * (T / 32) + wid];
            }
            r_prev[u] = r;
        }
        tvr_keyline<RW, PJ, U>(x0, y0, z0, s_rho, m, n_m, skip, act, has_rin, r_prev, sR, sV, sRM, tc, cam, field,
                                  fpack, mid_out, gi, acc, matched, need, fi_own, outside);
        // "DResidualNew[ikl]=fi" keeps the fi of the last matched keyline before ikl (:341,399-408): in-warp scan here,
        // earlier warps / CTAs through wcarry once the round's exchange is complete
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (j0 + u >= v.J) break;
            const int vw = (j0 + u) * (T / 32) + wid;
            const unsigned int bal = __ballot_sync(0xffffffffu, matched[u]);
            const unsigned int lower = bal & ((1u << lane) - 1u);
            const double prev_fi = __shfl_sync(0xffffffffu, fi_own[u], lower ? 31 - __clz(lower) : 0);
            const double wl = __shfl_sync(0xffffffffu, fi_own[u], bal ? 31 - __clz(bal) : 0);
            if (lane == 0) {
                sm.vw_has[p][vw] = bal != 0;
                sm.vw_last[p][vw] = wl;
            }
            if (act[u] && (matched[u] || need[u] || outside[u])) {
                const double rv = matched[u] ? fi_own[u]
                                  : need[u]  ? (lower ? prev_fi : __longlong_as_double((long long)RES_SENTINEL))
                                             : tc.max_r;
                if (li[u] < v.S) rout[li[u]] = rv;
                else grout[gi[u]] = rv;
            }
        }
    }
    MC_BSTAMP(12);
    // block sums in a fixed order
    __syncthreads();   // previous user of sm.part / sm.vw_* readers are done
    MC_BSTAMP(13);
    if (PJ) {
        const double w = warp_transpose_sum28(acc, lane);
        sm.part[wid][lane] = w;
    } else {
        double s = acc[27];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) sm.part[wid][27] = s;
    }
    MC_BSTAMP(14);
    __syncthreads();
    MC_BSTAMP(15);
    if (tid < 28) {
        double t = 0;
        if (PJ || tid == 27) {
            t = sm.part[0][tid];
#pragma unroll
            for (int ww = 1; ww < T / 32; ww++) t += sm.part[ww][tid];
        }
        sm.xout[p * MC_PW + tid] = t;
    } else if (tid == 32) {
        int has = 0;
        double lastv = 0;
        for (int q = v.J * (T / 32) - 1; q >= 0; q--)
            if (sm.vw_has[p][q]) {
                has = 1;
                lastv = sm.vw_last[p][q];
                break;
            }
        sm.xout[p * MC_PW + 28] = has ? 1.0 : 0.0;
        sm.xout[p * MC_PW + 29] = lastv;
    }
}

// next pose of a chain: R = exp(W), V, residual buffer ids (:309-311) / the z rotation RotM = exp((0,0,W.z)) (:313-314)
template <int T>
__device__ __forceinline__ void mc_req_R(McSmem<T> &sm, int p, const double *X, int res_in, int res_out) {
    so3_exp(X + 3, sm.req[p]);
    for (int k = 0; k < 3; k++) sm.req[p][9 + k] = X[k];
    sm.req_res[p][0] = res_in;
    sm.req_res[p][1] = res_out;
}
template <int T>
__device__ __forceinline__ void mc_req_RM(McSmem<T> &sm, int p, const LMState &s) {
    double wz[3] = {0, 0, s.Xeval[5]}, RMf[9];
    so3_exp(wz, RMf);
    sm.req[p][12] = RMf[0];
    sm.req[p][13] = RMf[1];
    sm.req[p][14] = RMf[3];
    sm.req[p][15] = RMf[4];
}

template <int T>
__global__ void __cluster_dims__(MC_C, 1, 1) __launch_bounds__(T, 1)
    k_minimizer_cluster(KLSoA old, const MapState *__restrict__ old_st, const unsigned long long *__restrict__ field,
                        const float4 *__restrict__ fpack, MapState *f_st, LMState *lm_out, int *abort_out, CamC cam,
                        McPlan plan, MinSetup su, FrameState *post_fs, FmBest *fm_best, int kpc_cap, ResPtrs gres,
                        unsigned long long *ll, MinCtl *ctl) {
    MC_STAMP(15, 0);
    // early_operands (set by the per-frame pipeline, whose previous kernel on this stream -- EstimateQuantile -- writes no
    // keyline array): the old map's operands are staged into shared memory BEFORE waiting for that kernel, i.e. while it runs
    const bool early = su.early_operands != 0 && su.a.match_num_thresh <= 255u;
    // (the dependents are released at the start of the last round, below: the grid after this kernel -- k_match of the
    // per-frame pipeline -- then becomes resident a round before it may start, instead of occupying the SMs this kernel
    // leaves free, where the detector stream runs the next frame, for the whole minimisation)
    if (!early) pdl_wait();
    MC_STAMP(15, 1);
    extern __shared__ __align__(16) unsigned char mc_dyn[];
    __shared__ McSmem<T> sm;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int rank = (int)mc_cluster_rank();
    const int G = (int)(gridDim.x / MC_C), cl = (int)(blockIdx.x / MC_C);   // clusters of this minimisation, mine
    const bool first_cta = blockIdx.x == 0;
    const unsigned int seq0 = G > 1 ? __ldcg(&ctl->gen) : 0u;   // sequence numbers of this minimisation: seq0 + 1 + round
    const int K0 = old_st->kn;
    if (K0 <= 0) {   // "if(klist.KNum()<=0) return 0;" (:601): Vel / W0 / RVel / RW0 stay what the caller passed, no FrameCount++
        if (early) {
            pdl_wait();
            pdl_launch();
        }
        if (first_cta && tid == 0) {
            lm_out->no_keylines = 1;
            lm_out->score = 0;
            for (int i = 0; i < 3; i++) {
                lm_out->Vel[i] = su.VW[i];
                lm_out->W0[i] = su.VW[3 + i];
            }
            if (post_fs) d_frame_post_min(post_fs, *lm_out);
        }
        return;   // (every CTA of every cluster: nobody reaches a barrier)
    }
    McView v;
    {
        double *d = reinterpret_cast<double *>(mc_dyn);
        v.x0 = d;
        v.y0 = d + kpc_cap;
        v.z0 = d + 2 * kpc_cap;
        v.s_rho = d + 3 * kpc_cap;
        v.res[0] = d + 4 * kpc_cap;
        v.res[1] = d + 5 * kpc_cap;
        v.res[2] = d + 6 * kpc_cap;
        v.flag = reinterpret_cast<unsigned char *>(d + 7 * kpc_cap);
        v.S = kpc_cap;
        v.gres[0] = gres.r[0];
        v.gres[1] = gres.r[1];
        v.gres[2] = gres.r[2];
        int kpc = (K0 + MC_C * G - 1) / (MC_C * G);
        kpc = (kpc + 31) & ~31;               // whole virtual warps
        if (kpc > MC_KPC_MAX) kpc = MC_KPC_MAX;   // (the host only launches this kernel when the capacity fits)
        v.base = (rank * G + cl) * kpc;        // slices in (rank, cluster) order: a column = the CTAs of equal rank
        v.cnt = K0 - v.base;
        v.cnt = v.cnt < 0 ? 0 : (v.cnt > kpc ? kpc : v.cnt);
        v.J = (kpc + T - 1) / T;
    }
    TvrConst tc;
    tc.max_r = su.max_r;
    tc.match_thresh = su.a.match_thresh;
    tc.k_huber = su.a.reweight_distance;
    tc.s_rho_min = 0;
    tc.mnt = 0;
    if (!early) {
        tc.s_rho_min = su.s_rho_from_state ? old_st->s_rho_q : su.max_s_rho;
        const unsigned int fc = su.fc_from_state ? f_st->frame_count : su.frame_count;
        tc.mnt = su.a.match_num_thresh < fc ? su.a.match_num_thresh : fc;
    }
    // ---- prologue: operands -> shared memory, LM state, barriers -----------------------------------------------
    for (int li = tid; li < v.cnt; li += T) {
        if (li < v.S) {
            const KlOp o = load_klop(old, v.base + li, cam);
            v.x0[li] = o.x0;
            v.y0[li] = o.y0;
            v.z0[li] = o.z0;
            v.s_rho[li] = o.s_rho;
            const unsigned int mn = (unsigned int)o.m_num;
            v.flag[li] = early ? (unsigned char)(mn < 255u ? mn : 255u) : (unsigned char)(mn < tc.mnt ? 1 : 0);
            v.res[0][li] = 0.0;   // for (auto &r : Residual) r = 0   (:625)
        } else {
            v.gres[0][v.base + li] = 0.0;
        }
    }
    if (early) {   // now the quantile and the frame counter of the previous kernel are needed
        pdl_wait();
        tc.s_rho_min = su.s_rho_from_state ? old_st->s_rho_q : su.max_s_rho;
        const unsigned int fc = su.fc_from_state ? f_st->frame_count : su.frame_count;
        tc.mnt = su.a.match_num_thresh < fc ? su.a.match_num_thresh : fc;   // (<= 255)
        const int ns = v.cnt < v.S ? v.cnt : v.S;
        for (int li = tid; li < ns; li += T) v.flag[li] = (unsigned int)v.flag[li] < tc.mnt ? 1 : 0;   // (own bytes)
    }
    const bool fused = plan.merge_round >= 0;
    if (tid == 0) {
        sm.abort = su.debug_abort;
        lm_begin(sm.lm, old_st, f_st, su.VW, su.a, su.max_r, su.max_s_rho, su.s_rho_from_state, su.frame_count,
                 su.fc_from_state);
        if (fused) {   // the prior-initialised try starts beside the zero-initialised one (:696-700)
            for (int i = 0; i < 3; i++) {
                sm.lm.X[i] = sm.lm.Vel_in[i];
                sm.lm.X[3 + i] = sm.lm.W0_in[i];
            }
            lm_request(sm.lm, sm.lm.X, -1, sm.lm.iRN);
        }
        mc_mbar_init(&sm.mbar[0], 1);
        mc_mbar_init(&sm.mbar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mc_req_R(sm, 0, sm.lm.Xeval, sm.lm.res_in, sm.lm.res_out);
        mc_req_RM(sm, 0, sm.lm);
    } else if (tid == 32 && fused) {
        lm_begin(sm.lmz, old_st, f_st, su.VW, su.a, su.max_r, su.max_s_rho, su.s_rho_from_state, su.frame_count,
                 su.fc_from_state);   // X = 0, request {0, -1, Rest}
        mc_req_R(sm, 1, sm.lmz.Xeval, sm.lmz.res_in, sm.lmz.res_out);
        mc_req_RM(sm, 1, sm.lmz);
    }
    __syncthreads();
    // the chains' LM variables live in registers of warps 0 / 1 for the whole minimisation (McChain).  Registers are
    // allocated per kernel, not per warp: the 512-thread form (capped at 128) spills part of the step (DESIGN.md §5)
    McChain ch;
    if (wid < 2) mc_chain_load(ch, wid == 0 ? sm.lm : sm.lmz, lane);
    bool fin = false;   // the main loop ended: lm_finalize after the rounds
    mc_cluster_sync();   // every CTA's barriers exist before anybody sends
    MC_STAMP(15, 2);

    // Round e: all warps evaluate the round's pose(s); the CTA's sums go to every CTA; then three warps work side by side
    // on the received data -- warp 0: totals, LM step, next pose of the main chain; warp 1: the same for the zero-init
    // chain; warp 2: stale-fi carries -- while warps 3 / 4 compute the z rotations of the two next poses as soon as the
    // LM steps are done (named barriers 1 / 2).  Two CTA-wide barriers per round.
    for (int e = 0; e < plan.n; e++) {
        const int sa = plan.sa[e], sb = plan.sb[e];
        const bool two = sa != STEP_NONE;
        const bool RW = sb >= STEP_MAIN_FIRST;
        const bool PJ = !(sb == STEP_INIT_LAST_ZERO || sb == STEP_INIT_LAST_PRIOR);
        const int par = e & 1;
        const unsigned int nval = two ? 2 * MC_PW : MC_PW;
        const bool last = e == plan.n - 1;
        const bool merge = e == plan.merge_round;                 // this round ends the two init tries
        const bool next_two = !last && plan.sa[e + 1] != STEP_NONE;
        const int res_out_p[2] = {sm.req_res[0][1], sm.req_res[1][1]};   // (warp 0 / 1 rewrite req_res for the next round)
        MC_STAMP(e, 0);
        if (last) pdl_launch();
        // ---- keylines ---------------------------------------------------------------------------------------
        if (RW) mc_eval_pose<T, true, true>(sm, v, 0, old, tc, cam, field, fpack, last, tid, lane, wid);
        else if (PJ) mc_eval_pose<T, false, true>(sm, v, 0, old, tc, cam, field, fpack, last, tid, lane, wid);
        else mc_eval_pose<T, false, false>(sm, v, 0, old, tc, cam, field, fpack, last, tid, lane, wid);
        if (two) {
            if (PJ) mc_eval_pose<T, false, true>(sm, v, 1, old, tc, cam, field, fpack, false, tid, lane, wid);
            else mc_eval_pose<T, false, false>(sm, v, 1, old, tc, cam, field, fpack, false, tid, lane, wid);
        }
        __syncthreads();
        MC_STAMP(e, 1);
        // ---- exchange.  Several clusters: the CTAs of equal rank first exchange their sums through L2 slots (published
        // right after the keyline pass, so that the store latency hides behind the slowest CTA) and add them in cluster
        // order; then every CTA sends its column sum to every CTA of its cluster through distributed shared memory.
        const unsigned int seq = seq0 + 1u + (unsigned int)e;
        if (tid == 0) mc_mbar_expect_tx(&sm.mbar[par], nval * MC_C * 8u);
        if (wid < 2 && (wid == 0 || two)) {
            const int p = wid;
            double t = lane < MC_PW ? sm.xout[p * MC_PW + lane] : 0.0;
            if (G > 1) {
                double vq[MC_GMAX];
                if (lane < MC_PW) {
                    mc_slot_put(mc_slots(ll, G, par, cl, rank, p), lane, seq, t);
                    MC_GT(e, 0);
                    if (!mc_slot_gather(ll, G, par, cl, rank, p, lane, seq, t, vq)) sm.abort = 1;
                    MC_GT(e, 1);
                }
                if (lane < 28) {
                    t = vq[0];
#pragma unroll
                    for (int q = 1; q < MC_GMAX; q++)
                        if (q < G) t += vq[q];
                }
                // column summary for the later columns: the last cluster of this column that has a match
                int qs = -1;
                if (lane == 28)
#pragma unroll
                    for (int q = 0; q < MC_GMAX; q++)
                        if (q < G && vq[q] != 0.0) qs = q;
                qs = __shfl_sync(0xffffffffu, qs, 28);
                if (lane == 28) t = qs >= 0 ? 1.0 : 0.0;
                if (lane == 29) {
                    t = 0.0;
#pragma unroll
                    for (int q = 0; q < MC_GMAX; q++)
                        if (q == qs) t = vq[q];
                }
            }
            if (lane < MC_PW) sm.xcol[p * MC_PW + lane] = t;
            __syncwarp();
            for (int idx = lane; idx < (MC_PW / 2) * MC_C; idx += 32) {
                const unsigned int dst = idx / (MC_PW / 2), pair = idx - dst * (MC_PW / 2);
                const unsigned int la = mc_smem_u32(&sm.gather[par][rank][p * MC_PW + 2 * pair]);
                const double a = sm.xcol[p * MC_PW + 2 * pair], b = sm.xcol[p * MC_PW + 2 * pair + 1];
                mc_st_async_v2(mc_mapa(la, dst), a, b, mc_mapa(mc_smem_u32(&sm.mbar[par]), dst));
            }
        }
        MC_STAMP(e, 2);
        if (wid < 3) {   // only the warps that consume the data wait for it
            const unsigned int ph = (unsigned int)(e >> 1) & 1u;
            const long long t0 = clock64();
            while (!mc_mbar_try_wait(&sm.mbar[par], ph)) {
                if (clock64() - t0 > MC_SPIN_LIMIT) {
                    sm.abort = 1;
                    break;
                }
            }
            MC_STAMP(e, 3);
            if (wid == 2) {   // stale-fi carries of this CTA's virtual warps
                // what enters this CTA from the earlier clusters of its column: their {has a match, last matched fi}
                double ccarry[2] = {0.0, 0.0};
                bool chas[2] = {false, false};
                if (G > 1) {
                    for (int p = 0; p < (two ? 2 : 1); p++) {
                        // lane q = 4 * cluster + word reads one slot word of {has, last} of an earlier cluster
                        const int qc = lane >> 2, qw = lane & 3;
                        unsigned int w32 = 0;
                        if (qc < cl) {
                            const unsigned long long *sl = mc_slots(ll, G, par, qc, rank, p) + 2 * 28 + qw;
                            const long long t0 = clock64();
                            unsigned long long x;
                            while ((unsigned int)((x = ld_volatile_u64(sl)) >> 32) != seq)
                                if (clock64() - t0 > MC_SPIN_LIMIT) {
                                    sm.abort = 1;
                                    break;
                                }
                            w32 = (unsigned int)x;
                        }
                        bool found = false;
                        for (int q = cl - 1; q >= 0; q--) {   // (uniform)
                            const double has = __hiloint2double((int)__shfl_sync(0xffffffffu, w32, 4 * q + 1),
                                                                (int)__shfl_sync(0xffffffffu, w32, 4 * q));
                            const double lst = __hiloint2double((int)__shfl_sync(0xffffffffu, w32, 4 * q + 3),
                                                                (int)__shfl_sync(0xffffffffu, w32, 4 * q + 2));
                            if (!found && has != 0.0) {
                                ccarry[p] = lst;
                                chas[p] = true;
                                found = true;
                            }
                        }
                    }
                }
                const int nvw = v.J * (T / 32);
                for (int q = lane; q < (two ? 2 : 1) * nvw; q += 32) {
                    const int p = q / nvw, vw = q - p * nvw;
                    double cy = 0;
                    bool found = false;
                    for (int w2 = vw - 1; w2 >= 0 && !found; w2--)
                        if (sm.vw_has[p][w2]) {
                            cy = sm.vw_last[p][w2];
                            found = true;
                        }
                    if (!found && chas[p]) {
                        cy = ccarry[p];
                        found = true;
                    }
                    for (int r = rank - 1; r >= 0 && !found; r--)   // earlier columns (their summaries came with the sums)
                        if (sm.gather[par][r][p * MC_PW + 28] != 0.0) {
                            cy = sm.gather[par][r][p * MC_PW + 29];
                            found = true;
                        }
                    sm.wcarry[res_out_p[p]][vw] = cy;
                }
            } else if (wid == 0 || two) {   // totals in rank order, then this chain's LM step and next pose
                const int p = wid;
                LMState &L = p == 0 ? sm.lm : sm.lmz;
                // lane k: total k in rank order, filed straight into this lane's JtJn / JtFn (lm_ingest, sign fix-ups
                // :484-490); lane 27: the score
                double t = 0;
                if (lane < 28) {
                    t = sm.gather[par][0][p * MC_PW + lane];
#pragma unroll
                    for (int r = 1; r < MC_C; r++) t += sm.gather[par][r][p * MC_PW + lane];
                }
                if (lane == 27) L.last_score = t;
                if (PJ && lane < 27) {
                    if (lane < 21) {
                        const int a = mc_up_row(lane), b = mc_up_col(lane, a);
                        const bool neg = (a < 2 && (b == 2 || b == 3)) || ((a == 2 || a == 3) && b >= 4);
                        ch.nw = neg ? -t : t;
                    } else {
                        const int a = lane - 21;
                        ch.nw = (a == 2 || a == 3) ? -t : t;
                    }
                }
                const double last_score = __shfl_sync(MC_FULL, t, 27);
                MC_STAMP(e, 4);
                const bool ab = __any_sync(MC_FULL, sm.abort != 0);   // (one decision for the whole warp)
                McReq q;
                bool req = false;
                if (!ab) {
                    ch.n_eval++;
                    MC_STAMP(e, 5);
                    req = mc_step(ch, q, L, p == 0 ? sb : sa, last_score, su.a.init_iter, su.a.iter_max, fin, lane);
                    if (p == 0) MC_STAMP(e, 6);
                }
                if (merge) {   // (uniform) the main chain picks the better try once both LM steps are done
                    if (p == 1) mc_merge_publish(ch, sm.lmz, lane);
                    asm volatile("bar.sync 3, 64;" ::: "memory");
                    if (p == 0 && !ab) {
                        mc_merge(ch, q, sm.lm, sm.lmz, lane);
                        req = true;
                    }
                }
                if (!last) {
                    if (p == 0) {
                        asm volatile("bar.sync 1, 64;" ::: "memory");      // releases warp 3
                        if (lane == 0 && req) mc_req_R(sm, 0, q.x, q.ri, q.ro);
                    } else if (next_two) {
                        asm volatile("bar.sync 2, 64;" ::: "memory");      // releases warp 4
                        if (lane == 0 && req) mc_req_R(sm, 1, q.x, q.ri, q.ro);
                    }
                }
                MC_STAMP(e, 7);
            }
        } else if (last) {
            // FordwardMatch's arg-max over this CTA's keylines, whose m_id_f the pass above wrote: the CAS round trips
            // run on the warps that are idle during the last exchange and LM step, not between the pass and the exchange
            if (fm_best) {   // (two keylines per thread and step: loads and CAS round trips in flight together)
                const int nkn = f_st->kn, st = T - 96;
                for (int li = tid - 96; li < v.cnt; li += 2 * st)
                    d_fm_argmax_two(old, v.base + li, li + st < v.cnt ? v.base + li + st : -1, nkn, fm_best);
            }
        } else if (wid == 3) {
            asm volatile("bar.sync 1, 64;" ::: "memory");
            if (lane == 0) mc_req_RM(sm, 0, sm.lm);
        } else if (wid == 4 && next_two) {
            asm volatile("bar.sync 2, 64;" ::: "memory");
            if (lane == 0) mc_req_RM(sm, 1, sm.lmz);
        }
        __syncthreads();
        if (sm.abort) break;
    }
    // ---- epilogue ------------------------------------------------------------------------------------------------
    if (wid == 0) {   // the main chain's registers -> sm.lm, then the outputs of the main loop (:793-816)
        mc_chain_store(ch, sm.lm, lane);
        __syncwarp();
        if (lane == 0 && fin) lm_finalize(sm.lm, first_cta ? f_st : nullptr);
    }
    if (sm.abort && tid == 0) {
        *abort_out = 1;
        for (int k = 0; k < 3; k++) sm.lm.Vel[k] = sm.lm.W0[k] = __longlong_as_double(0x7FF8000000000000ll);
    }
    __syncthreads();
    if (!sm.abort) lm_finalize_cov(sm.lm, tid);   // the six columns of Cholesky<6>(JtJ).get_inverse() side by side
    // the per-frame pipeline's stage after the minimiser, folded in: what needs only V / W beside the covariance
    if (first_cta && tid == 32 && post_fs) d_frame_post_min_pose(post_fs, sm.lm);
    __syncthreads();
    if (first_cta) {
        // the next minimisation gets fresh sequence numbers: this one used seq0 + 1 .. seq0 + plan.n <= seq0 + MIN_MAX_ROUNDS
        if (tid == 0 && G > 1) ctl->gen = seq0 + MIN_MAX_ROUNDS + 1u;
        const double *src = reinterpret_cast<const double *>(&sm.lm);
        double *dst = reinterpret_cast<double *>(lm_out);
        for (int k = tid; k < (int)(sizeof(LMState) / sizeof(double)); k += T) dst[k] = src[k];
        if (tid == 0 && post_fs) d_frame_post_min_cov(post_fs, sm.lm);
    }
    MC_STAMP(15, 3);
    mc_cluster_sync();   // no CTA exits while a peer may still send to it
    MC_STAMP(15, 4);
}

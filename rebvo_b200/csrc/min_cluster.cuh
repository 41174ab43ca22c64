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

// "Save the scores in temporals" (:686-691) + "Check for the lowest score" (:734-747) once both tries are done
__device__ __forceinline__ void mc_lm_merge(LMState &s, const LMState &z) {
    for (int i = 0; i < 6; i++) s.Xt[i] = z.X[i];
    s.Ft = z.F;
    s.F0t = z.F0;
    s.ut = z.u;
    s.vt = z.v;
    s.eff_steps_t = z.eff_steps;
    lm_after_prior_pass(s);
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
__device__ __forceinline__ void mc_req_R(McSmem<T> &sm, int p, const LMState &s) {
    so3_exp(s.Xeval + 3, sm.req[p]);
    for (int k = 0; k < 3; k++) sm.req[p][9 + k] = s.Xeval[k];
    sm.req_res[p][0] = s.res_in;
    sm.req_res[p][1] = s.res_out;
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
        mc_req_R(sm, 0, sm.lm);
        mc_req_RM(sm, 0, sm.lm);
    } else if (tid == 32 && fused) {
        lm_begin(sm.lmz, old_st, f_st, su.VW, su.a, su.max_r, su.max_s_rho, su.s_rho_from_state, su.frame_count,
                 su.fc_from_state);   // X = 0, request {0, -1, Rest}
        mc_req_R(sm, 1, sm.lmz);
        mc_req_RM(sm, 1, sm.lmz);
    }
    __syncthreads();
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
                if (lane < 28) {   // lane k: total k in rank order, filed straight into JtJn / JtFn (lm_ingest, sign fix-ups :484-490)
                    double t = sm.gather[par][0][p * MC_PW + lane];
#pragma unroll
                    for (int r = 1; r < MC_C; r++) t += sm.gather[par][r][p * MC_PW + lane];
                    if (lane == 27) {
                        L.last_score = t;
                    } else if (PJ && lane < 27) {
                        if (lane < 21) {
                            // upper-triangle index -> (row, column), branch-free
                            const int a = lane < 6 ? 0 : lane < 11 ? 1 : lane < 15 ? 2 : lane < 18 ? 3 : lane < 20 ? 4 : 5;
                            const int b = lane - (a == 0 ? 0 : a == 1 ? 6 : a == 2 ? 11 : a == 3 ? 15 : a == 4 ? 18 : 20) + a;
                            const bool neg = (a < 2 && (b == 2 || b == 3)) || ((a == 2 || a == 3) && b >= 4);
                            t = neg ? -t : t;
                            L.JtJn[a * 6 + b] = t;
                            L.JtJn[b * 6 + a] = t;
                        } else {
                            const int a = lane - 21;
                            L.JtFn[a] = (a == 2 || a == 3) ? -t : t;
                        }
                    }
                }
                __syncwarp();
                MC_STAMP(e, 4);
                if (lane == 0 && !sm.abort) {
                    L.n_eval++;
                    MC_STAMP(e, 5);
                    if (p == 0) {
                        lm_step_main(sm.lm, sb, first_cta ? f_st : nullptr);
                        MC_STAMP(e, 6);
                    } else {
                        lm_step_zero(sm.lmz, sa);
                    }
                }
                __syncwarp();
                if (merge) {   // (uniform) the main chain picks the better try once both LM steps are done
                    asm volatile("bar.sync 3, 64;" ::: "memory");
                    if (p == 0 && lane == 0 && !sm.abort) mc_lm_merge(sm.lm, sm.lmz);
                    __syncwarp();
                }
                if (!last) {
                    if (p == 0) {
                        asm volatile("bar.sync 1, 64;" ::: "memory");      // releases warp 3
                        if (lane == 0) mc_req_R(sm, 0, sm.lm);
                    } else if (next_two) {
                        asm volatile("bar.sync 2, 64;" ::: "memory");      // releases warp 4
                        if (lane == 0) mc_req_R(sm, 1, sm.lmz);
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

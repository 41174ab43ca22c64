// stage_reduce.cuh -- the block reduction of the stage-level keyline evaluations: TryVelRot (k_try_vel_rot, tracker.cu),
// TryVel (k_tv_eval) and ExtRotVel (k_extrotvel, imu_track.cu).  Each runs one old keyline per thread in blocks of
// STAGE_T; a block writes its NV sums to partials[k][block] (block_sum_to) and, where the evaluation writes residuals, the
// stale-fi summary of its matches (block_stale_fi).  A second launch, k_blocks_finish, folds the partials in block order
// and hands the stale fi across blocks.  Sums are in a fixed order: deterministic, not the reference's pairwise tree.
#pragma once
#include "common.cuh"

#define STAGE_T 256                          // threads (one keyline each) per block; partials hold up to STAGE_T blocks
#define RES_SENTINEL 0x7FF8DEADBEEF0001ull   // residual bits of a miss whose stale fi comes from an earlier block

// sum of acc[k] over the block: xor tree per warp, then warps in order; dst[k * dst_stride] = sum k
template <int NV>
__device__ __forceinline__ void block_sum_to(const double (&acc)[NV], double (*s_part)[STAGE_T / 32], int lane, int wid,
                                             double *dst, int dst_stride) {
#pragma unroll
    for (int k = 0; k < NV; k++) {
        double v = acc[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0) s_part[k][wid] = v;
    }
    __syncthreads();
    if (wid == 0 && lane < NV) {
        double t = 0;
#pragma unroll
        for (int ww = 0; ww < STAGE_T / 32; ww++) t += s_part[lane][ww];
        dst[lane * dst_stride] = t;
    }
}

struct StaleSmem {
    int whas[STAGE_T / 32];
    double wlast[STAGE_T / 32];
};
// The reference's residual of a miss is the fi of the last matched keyline before it (fi is a function-level variable:
// "DResidualNew[ikl]=fi" in TryVelRot, "Residuals[ikl]=fabs(fi)" in TryVel).  Called by every thread of the block, with
// its keyline's match and fi: returns the fi of the block's last match before this keyline (|fi| when abs), or
// RES_SENTINEL when the block has none before it, for k_blocks_finish to replace.  Writes the block's summary (has a
// match, last matched fi) to blk_has / blk_last_fi.
__device__ __forceinline__ double block_stale_fi(bool matched, double fi_own, bool abs, StaleSmem &sm, int *blk_has,
                                                 double *blk_last_fi, int lane, int wid) {
    const unsigned int bal = __ballot_sync(0xffffffffu, matched);
    const unsigned int lower = bal & ((1u << lane) - 1u);
    const double prev_fi = __shfl_sync(0xffffffffu, fi_own, lower ? 31 - __clz(lower) : 0);
    const double wl = __shfl_sync(0xffffffffu, fi_own, bal ? 31 - __clz(bal) : 0);
    if (lane == 0) {
        sm.whas[wid] = bal != 0;
        sm.wlast[wid] = wl;
    }
    __syncthreads();
    bool found = lower != 0;
    double v = prev_fi;
    if (!found)
        for (int ww = wid - 1; ww >= 0; ww--)
            if (sm.whas[ww]) {
                v = sm.wlast[ww];
                found = true;
                break;
            }
    if (lane == 0 && wid == 0) {
        int has = 0;
        double lv = 0;
        for (int ww = 0; ww < STAGE_T / 32; ww++)
            if (sm.whas[ww]) {
                has = 1;
                lv = sm.wlast[ww];
            }
        blk_has[blockIdx.x] = has;
        blk_last_fi[blockIdx.x] = lv;
    }
    if (!found) return __longlong_as_double((long long)RES_SENTINEL);
    return abs ? fabs(v) : v;
}

// After an evaluation of nb blocks: out[k] = partials[k][0] + .. + partials[k][nb - 1] in block order (block 0, thread
// k < NV).  With res, each residual of keyline i < st->kn that holds RES_SENTINEL takes the last matched fi of the nearest
// earlier block that has a match, 0 when none (|fi| when abs); such a launch has nb blocks of STAGE_T, one without res a
// single block of at least NV threads.
template <int NV>
__global__ void __launch_bounds__(STAGE_T) k_blocks_finish(const double *__restrict__ partials, int nb,
                                                           double *__restrict__ out, double *__restrict__ res,
                                                           const int *__restrict__ blk_has,
                                                           const double *__restrict__ blk_last_fi,
                                                           const MapState *__restrict__ st, bool abs) {
    const int tid = threadIdx.x;
    if (blockIdx.x == 0 && tid < NV) {
        double t = 0;
        for (int b = 0; b < nb; b++) t += partials[tid * STAGE_T + b];
        out[tid] = t;
    }
    const int i = blockIdx.x * STAGE_T + tid;
    if (!res || i >= st->kn || reinterpret_cast<unsigned long long *>(res)[i] != RES_SENTINEL) return;
    double carry = 0;
    for (int b = blockIdx.x - 1; b >= 0; b--)
        if (blk_has[b]) {
            carry = blk_last_fi[b];
            break;
        }
    res[i] = abs ? fabs(carry) : carry;
}

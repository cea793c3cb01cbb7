// observe_mse.cuh -- the MSE observer's shrink-grid search (ct_mse_block, include/ct_b200.h) for the fused observer kernels.
//
// A group's min / max are in registers already; every candidate i shrinks them by p_i, takes calculate_qparams of the result
// (observe_core.cuh) and sums |fake_quantize(x) - x|^norm over the group in float32.  The caller supplies that per-lane partial sum;
// the lanes of a group combine it with the same xor shuffles as their min / max, so every lane holds the same sum and takes the same
// decision.  The search is compute-bound: `steps` fake-quantize passes over registers, two MUFU operations per element and step for a
// norm other than 2.
#pragma once

#include <cfloat>

#include "observe_core.cuh"

namespace ctb {

// |d|^norm in float32: d * d for norm 2, else exp2(norm * log2|d|) on the MUFU (|d| = 0 gives exp2(-inf) = 0, inf stays inf)
__device__ __forceinline__ float mse_pow(float d, float norm, bool square) {
    const float a = fabsf(d);
    if (square) return a * a;
    float l, r;
    asm("lg2.approx.f32 %0, %1;" : "=f"(l) : "f"(a));
    const float t = norm * l;
    asm("ex2.approx.f32 %0, %1;" : "=f"(r) : "f"(t));
    return r;
}

// stop step S from the call's `any` bits: the first step ending `patience` steps without an improvement, steps - 1 if none
__device__ __forceinline__ int mse_stop(uint64_t any, int steps, int patience) {
    int run = 0;
    for (int i = 0; i < steps; ++i) {
        run = ((any >> i) & 1ull) ? 0 : run + 1;
        if (run >= patience) return i;
    }
    return steps - 1;
}

// |fake_quantize(x) - x|^norm of one element with integer (FP8 = false) or float8_e4m3fn codes, every op rounded to x's dtype T as
// ct_fake_quantize rounds it (forward_helpers.py:180-215); c is make_scale_ctx(s), zq the zero point (ASYM)
template <class P, bool ASYM, bool FP8>
__device__ __forceinline__ float mse_elem(float xv, float s, float zq, const ScaleCtx& c, float qmin, float qmax, float norm, bool square) {
    float t = rnd_dt(c.slow ? __fdiv_rn(xv, s) : quot<P, false>(xv, c), P::DT);
    if (ASYM) t = rnd_dt(t + zq, P::DT);
    t = fminf(fmaxf(t, qmin), qmax);
    t = FP8 ? hd_e4m3_to_f32(hd_f32_to_e4m3(t)) : rintf(t);
    if (ASYM) t = rnd_dt(t - zq, P::DT);
    return mse_pow(rnd_dt(t * s, P::DT) - xv, norm, square);
}

// the stop step's mask of steps 0 .. S
__device__ __forceinline__ uint64_t mse_keep(const ct_mse_block* B) {
    const int stop = mse_stop(B->any, B->steps, B->patience);
    return stop >= 63 ? ~0ull : ((1ull << (stop + 1)) - 1ull);
}
// the last improving step <= S of a group with mask m (0 if none)
__device__ __forceinline__ int mse_last(uint64_t m, uint64_t keep) {
    const uint64_t k = m & keep;
    return k ? 63 - __clzll((long long)k) : 0;
}

// the step a group is written with before the stop step is known: its last improving step (0 if it never improved).  `partial(i, lo,
// hi)` is this lane's error sum for candidate i with the shrunk range [lo, hi]; `err_row` (or nullptr) receives e(i) from one lane.
template <class P, int LPG, class Partial>
__device__ __forceinline__ int mse_search(const ct_mse_block* B, float lo, float hi, Partial partial, uint64_t& mask, float* err_row) {
    const int steps = B->steps;
    const unsigned act = LPG > 1 ? __activemask() : 0u;   // whole groups are active or inactive together
    float best = FLT_MAX;
    int best_i = 0;
    mask = 0;
    for (int i = 0; i < steps; ++i) {
        const float p = __ldg(&B->shrink[i]);
        float e = partial(rnd_dt(lo * p, P::DT), rnd_dt(hi * p, P::DT));
#pragma unroll
        for (int d = 1; d < LPG; d <<= 1) e += __shfl_xor_sync(act, e, d);
        if (err_row) err_row[i] = e;
        if (e < best) {   // NaN / inf never improve
            best = e;
            best_i = i;
            mask |= 1ull << i;
        }
    }
    return best_i;
}

// the group's mask into scratch and its new bits into the call's `any` (one lane per group); `any` only gains bits, so a stale read
// costs a redundant atomic, never a lost bit
__device__ __forceinline__ void mse_publish(ct_mse_block* B, uint64_t gi, uint64_t mask) {
    B->masks[gi] = mask;
    const unsigned long long seen = __ldcg(reinterpret_cast<const unsigned long long*>(&B->any));
    if (mask & ~seen) atomicOr(reinterpret_cast<unsigned long long*>(&B->any), (unsigned long long)mask);
}

}  // namespace ctb

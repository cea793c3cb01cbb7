// fast_observe.cu -- one-pass "observe + quantize + pack" for group-quantized integer weights:
//   x (bf16 / fp16)  ->  packed int32 codes + scale (+ int8 zero point)
// i.e. the memoryless min-max observer rule of the reference, calculate_qparams
// (quantization/utils/helpers.py:50-137), fused in front of quantize + pack_to_int32
// (pack_quantized/base.py:96-104), so the weight is read from HBM once instead of twice.
// This is row (f)1 of SURVEY.md section 8.
//
// A thread owns a unit of 32 elements (4 chunks); a quantization group of 32 * LPG elements is owned by
// LPG adjacent lanes, which combine their packed min / max with warp shuffles.  The qparams are then
// computed redundantly by every lane of the group with the reference's per-op rounding to the weight
// dtype T, and lane 0 of the group stores them.
#include "engine.h"
#include "observe_core.cuh"
#include "ops.cuh"

namespace ctb {

template <class P, int BITS, int ASYM, int LPG>
struct ObserveQuantPackOp {
    static constexpr int IN_BYTES = 16;
    static constexpr int GROUP = 4;
    static constexpr int OUT_WORDS = BITS / 4;   // per chunk
    using Raw = NoRaw;
    __device__ static __forceinline__ Raw prefetch(const Job&, uint32_t) { return {}; }

    __device__ static __forceinline__ void run(const Job& J, const Common& cm, const Raw&, uint32_t gc0, const uint32_t (&w)[4][4], int off) {
        // ---- observer: min / max of the group ----
        uint32_t mn2 = w[0][0], mx2 = w[0][0];
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                mn2 = min2_nan<P>(mn2, w[g][k]);
                mx2 = max2_nan<P>(mx2, w[g][k]);
            }
        if (LPG > 1) {
            const unsigned act = __activemask();   // whole groups are active or inactive together
#pragma unroll
            for (int d = 1; d < LPG; d <<= 1) {
                mn2 = min2_nan<P>(mn2, __shfl_xor_sync(act, mn2, d));
                mx2 = max2_nan<P>(mx2, __shfl_xor_sync(act, mx2, d));
            }
        }
        float lo, hi;
        obs_range2<P>(mn2, mx2, lo, hi);

        // ---- calculate_qparams, each op rounded to T (helpers.py:74-131) ----
        float zq;
        const float s = obs_scale_zp<P::DT>(lo, hi, ASYM, cm.qmin, cm.qmax, zq);

        const uint32_t gi = fd_div(gc0, J.dc);
        if ((threadIdx.x & (LPG - 1)) == 0) {
            reinterpret_cast<unsigned short*>(const_cast<void*>(J.scale))[gi] = (unsigned short)P::from_float1(s);
            if (ASYM) reinterpret_cast<int8_t*>(const_cast<void*>(J.zp))[gi] = (int8_t)(int)zq;
        }

        // ---- quantize + pack with the fresh qparams ----
        const ScaleCtx sc = make_scale_ctx(s);
        const uint32_t zp2 = ASYM ? dup2<P>(zq) : 0u;
        uint32_t o[4 * OUT_WORDS];
        using QP = QuantPackOp<P, BITS, ASYM, 4>;
        if (sc.slow) {
#pragma unroll
            for (int g = 0; g < 4; ++g) QP::template chunk<true>(w[g], sc, zp2, cm, o + g * OUT_WORDS);
        } else {
#pragma unroll
            for (int g = 0; g < 4; ++g) QP::template chunk<false>(w[g], sc, zp2, cm, o + g * OUT_WORDS);
        }
        rotate_out<4, OUT_WORDS>(o, off);
        store_words<4 * OUT_WORDS>(J.out + (size_t)gc0 * (4 * OUT_WORDS), o);
    }
};

#define SIG_FAIL(sig)                                                                              \
    do {                                                                                           \
        set_error("no fused observer kernel for dtype=%d bits=%d asym=%d lanes/group=%d", sig.p_dt, sig.sel, sig.zp, sig.group); \
        return CT_E_UNSUPPORTED;                                                                   \
    } while (0)

template <class P, int BITS, int ASYM>
static int observe_lpg(const FastSig& s, const LaunchPlan& lp, int device, cudaStream_t st) {
    switch (s.group) {
    case 1: return launch_stream<ObserveQuantPackOp<P, BITS, ASYM, 1>>(lp, device, st);
    case 2: return launch_stream<ObserveQuantPackOp<P, BITS, ASYM, 2>>(lp, device, st);
    case 4: return launch_stream<ObserveQuantPackOp<P, BITS, ASYM, 4>>(lp, device, st);
    case 8: return launch_stream<ObserveQuantPackOp<P, BITS, ASYM, 8>>(lp, device, st);
    }
    SIG_FAIL(s);
}
template <class P>
static int observe_p(const FastSig& s, const LaunchPlan& lp, int device, cudaStream_t st) {
    if (s.sel == 4 && s.zp == 0) return observe_lpg<P, 4, 0>(s, lp, device, st);
    if (s.sel == 4 && s.zp == 1) return observe_lpg<P, 4, 1>(s, lp, device, st);
    if (s.sel == 8 && s.zp == 0) return observe_lpg<P, 8, 0>(s, lp, device, st);
    if (s.sel == 8 && s.zp == 1) return observe_lpg<P, 8, 1>(s, lp, device, st);
    SIG_FAIL(s);
}

int launch_fast_observe(const FastSig& s, const LaunchPlan& lp, int device, cudaStream_t st) {
    if (s.p_dt == CT_BF16) return observe_p<BF16>(s, lp, device, st);
    if (s.p_dt == CT_F16) return observe_p<F16>(s, lp, device, st);
    SIG_FAIL(s);
}

}  // namespace ctb

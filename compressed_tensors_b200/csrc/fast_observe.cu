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
//
// MSE mode (d->aux = ct_mse_block): between the min / max and the qparams, the group searches its shrink grid from registers
// (observe_mse.cuh) and is written with its best improving step; mse_fixup_pack_kernel then applies the call's stop step.
#include "engine.h"
#include "generic.cuh"
#include "observe_core.cuh"
#include "observe_mse.cuh"
#include "ops.cuh"

namespace ctb {

template <class P, int BITS, int ASYM, int LPG, bool MSE = false>
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
        const uint32_t gi = fd_div(gc0, J.dc);

        if constexpr (MSE) {
            ct_mse_block* B = reinterpret_cast<ct_mse_block*>(const_cast<void*>(J.aux));
            const bool lead = (threadIdx.x & (LPG - 1)) == 0;
            const bool square = B->norm == 2.0f;
            const float norm = B->norm;
            auto partial = [&](float clo, float chi) {
                float czq;
                const float cs = obs_scale_zp<P::DT>(clo, chi, ASYM, cm.qmin, cm.qmax, czq);
                const ScaleCtx c = make_scale_ctx(cs);
                float e = 0.f;
#pragma unroll
                for (int g = 0; g < 4; ++g)
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        e += mse_elem<P, ASYM, false>(P::lo(w[g][k]), cs, czq, c, cm.qmin, cm.qmax, norm, square) +
                             mse_elem<P, ASYM, false>(P::hi(w[g][k]), cs, czq, c, cm.qmin, cm.qmax, norm, square);
                return e;
            };
            uint64_t mask;
            float* err_row = (B->errors && lead) ? B->errors + (size_t)gi * B->steps : nullptr;
            const int best = mse_search<P, LPG>(B, lo, hi, partial, mask, err_row);
            if (lead) mse_publish(B, gi, mask);
            const float p = __ldg(&B->shrink[best]);
            lo = rnd_dt(lo * p, P::DT);
            hi = rnd_dt(hi * p, P::DT);
        }

        // ---- calculate_qparams, each op rounded to T (helpers.py:74-131) ----
        float zq;
        const float s = obs_scale_zp<P::DT>(lo, hi, ASYM, cm.qmin, cm.qmax, zq);

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

template <class P, int BITS, int ASYM, bool MSE>
static StreamKernel observe_lpg(int lanes_per_group) {
    switch (lanes_per_group) {
    case 1: return stream_kernel<ObserveQuantPackOp<P, BITS, ASYM, 1, MSE>>();
    case 2: return stream_kernel<ObserveQuantPackOp<P, BITS, ASYM, 2, MSE>>();
    case 4: return stream_kernel<ObserveQuantPackOp<P, BITS, ASYM, 4, MSE>>();
    case 8: return stream_kernel<ObserveQuantPackOp<P, BITS, ASYM, 8, MSE>>();
    }
    return {};
}
template <class P, bool MSE>
static StreamKernel observe_p(int bits, bool asym, int lanes_per_group) {
    if (bits == 4 && !asym) return observe_lpg<P, 4, 0, MSE>(lanes_per_group);
    if (bits == 4 && asym) return observe_lpg<P, 4, 1, MSE>(lanes_per_group);
    if (bits == 8 && !asym) return observe_lpg<P, 8, 0, MSE>(lanes_per_group);
    if (bits == 8 && asym) return observe_lpg<P, 8, 1, MSE>(lanes_per_group);
    return {};
}

StreamKernel observe_kernel(int p_dt, int bits, bool asym, int lanes_per_group, bool mse) {
    if (p_dt == CT_BF16) return mse ? observe_p<BF16, true>(bits, asym, lanes_per_group) : observe_p<BF16, false>(bits, asym, lanes_per_group);
    if (p_dt == CT_F16) return mse ? observe_p<F16, true>(bits, asym, lanes_per_group) : observe_p<F16, false>(bits, asym, lanes_per_group);
    return {};
}

// The MSE mode's second launch: the stop step S from the call's `any` bits, then every group whose mask has a bit above S rewritten,
// by one thread, with its last improving step <= S (0 if none): min / max, calculate_qparams, codes and packed words with the same
// per-element arithmetic as the streaming pass (quant_scalar's IEEE division equals its reciprocal quotient, ct_selftest_division).
// Groups with no bit above S already hold that step and are only read (their mask).
template <class P, int BITS, int ASYM>
__global__ void __launch_bounds__(256) mse_fixup_pack_kernel(const ct_mse_block* B, const void* x, void* scale, int8_t* zp, uint32_t* packed,
                                                             int64_t n_groups, int group, float qmin, float qmax) {
    const uint64_t keep = mse_keep(B);
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t m = B->masks[g];
        if ((m & ~keep) == 0) continue;
        const int best = mse_last(m, keep);
        const int64_t e0 = g * group;
        float mn = 0.f, mx = 0.f;   // min(min_vals, 0), max(max_vals, 0); a group that improved is finite
        for (int j = 0; j < group; ++j) {
            const float v = load_as_f32(x, e0 + j, P::DT);
            mn = fminf(mn, v);
            mx = fmaxf(mx, v);
        }
        const float p = B->shrink[best];
        float zq;
        const float s = obs_scale_zp<P::DT>(rnd_dt(mn * p, P::DT), rnd_dt(mx * p, P::DT), ASYM, qmin, qmax, zq);
        reinterpret_cast<unsigned short*>(scale)[g] = (unsigned short)P::from_float1(s);
        if (ASYM) zp[g] = (int8_t)(int)zq;
        for (int u = 0; u < group; u += 32) {
            uint32_t words[BITS];
            pack_group<BITS>(words, 32, [&](int j) { return (int32_t)quant_scalar(load_as_f32(x, e0 + u + j, P::DT), s, ASYM, zq, P::DT, CT_Q_INT, qmin, qmax); });
#pragma unroll
            for (int w = 0; w < BITS; ++w) packed[(e0 + u) / 32 * BITS + w] = words[w];
        }
    }
}

template <class P, int BITS, int ASYM>
static void fixup_launch(const ct_mse_block* B, const void* x, void* scale, int8_t* zp, uint32_t* packed, int64_t n_groups, int group,
                         float qmin, float qmax, cudaStream_t st) {
    const int64_t blocks = (n_groups + 255) / 256;
    mse_fixup_pack_kernel<P, BITS, ASYM><<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(B, x, scale, zp, packed, n_groups, group, qmin, qmax);
}

int launch_mse_fixup_pack(const ct_quant_desc& d, const void* x, void* scale, void* zp, int32_t* packed, cudaStream_t st) {
    const int64_t n_groups = d.rows * d.cols / d.cdiv;
    if (n_groups == 0) return CT_OK;
    const float r = (float)(1 << d.num_bits), qmin = -r / 2, qmax = r / 2 - 1;
    const ct_mse_block* B = reinterpret_cast<const ct_mse_block*>(d.aux);
    int8_t* z = reinterpret_cast<int8_t*>(zp);
    uint32_t* pk = reinterpret_cast<uint32_t*>(packed);
    const int grp = (int)d.cdiv;
#define CT_FIXUP(P, B_, A_) fixup_launch<P, B_, A_>(B, x, scale, z, pk, n_groups, grp, qmin, qmax, st)
    if (d.x_dtype == CT_BF16) {
        if (d.num_bits == 4) { if (z) CT_FIXUP(BF16, 4, 1); else CT_FIXUP(BF16, 4, 0); }
        else { if (z) CT_FIXUP(BF16, 8, 1); else CT_FIXUP(BF16, 8, 0); }
    } else {
        if (d.num_bits == 4) { if (z) CT_FIXUP(F16, 4, 1); else CT_FIXUP(F16, 4, 0); }
        else { if (z) CT_FIXUP(F16, 8, 1); else CT_FIXUP(F16, 8, 0); }
    }
#undef CT_FIXUP
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

}  // namespace ctb

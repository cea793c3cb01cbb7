// observe_core.cuh -- the observer's calculate_qparams rule (quantization/utils/helpers.py:50-137) in one place, for every kernel that
// derives scales on the device: the group / channel / tensor observers (fast_observe.cu, observe_channel.cu, observe_tensor.cu), NVFP4's
// group scale (fp4_ops.cuh) and the dynamic activation observers (dynamic_fake.cu).
//
// The reference evaluates each op of the rule as a separate torch op on qparam-sized tensors in the observer's dtype DT (x's dtype:
// min / max come from torch.amin / amax of x), so every op rounds to DT; these functions round the same way.  DT = CT_F32 rounds nothing.
// min / max are taken as already clamped around 0 (min(min_vals, 0), max(max_vals, 0)) by the caller.
//
// NaN.  torch.amin / amax, torch.min / max and torch.clamp give NaN where any operand is NaN, so a NaN in a row or group makes its scale
// NaN (and every fake-quantized value of it).  The reductions therefore use fmin_nan / fmax_nan and the packed min2_nan / max2_nan
// (quant_core.cuh), never fminf / fmaxf or min2 / max2, which drop a NaN operand.
#pragma once

#include "quant_core.cuh"

namespace ctb {

// packed min / max of a reduction -> min(min_vals, 0), max(max_vals, 0) as floats
template <class P> __device__ __forceinline__ void obs_range2(uint32_t mn2, uint32_t mx2, float& lo, float& hi) {
    lo = fmin_nan(fmin_nan(P::lo(mn2), P::hi(mn2)), 0.f);
    hi = fmax_nan(fmax_nan(P::lo(mx2), P::hi(mx2)), 0.f);
}
// one 16-byte chunk folded into a packed running min / max
template <class P> __device__ __forceinline__ void obs_chunk_minmax(const uint4& v, uint32_t& mn2, uint32_t& mx2) {
    mn2 = min2_nan<P>(min2_nan<P>(mn2, v.x), min2_nan<P>(v.y, min2_nan<P>(v.z, v.w)));
    mx2 = max2_nan<P>(max2_nan<P>(mx2, v.x), max2_nan<P>(v.y, max2_nan<P>(v.z, v.w)));
}

template <int DT> CT_HD float obs_round(float v) { return rnd_dt(v, DT); }
// torch.finfo(DT).eps: the scale that replaces a zero one when the args give no scale_dtype
template <int DT> CT_HD float obs_eps() { return DT == CT_BF16 ? 0.0078125f : (DT == CT_F16 ? 0.0009765625f : 1.1920928955078125e-07f); }
template <int DT> CT_HD float obs_tiny() { return DT == CT_F16 ? 6.103515625e-05f : 1.1754943508222875e-38f; }

// symmetric scale before any scale_dtype rounding: max(|min|, |max|) / (bit_range / 2) in DT (the halved range is exact in every DT)
template <int DT> CT_HD float obs_sym_scale(float lo, float hi, float qmin, float qmax) {
    return obs_round<DT>(hd_div(fmax_nan(fabsf(lo), fabsf(hi)), (qmax - qmin) * 0.5f));
}

// integer scale (x dtype, no scale_dtype) and zero point of one observed range: symmetric, or asymmetric with the zero point
// round(clamp(qmin - min / scale, qmin, qmax)) as int8 (0 for 0 / 0); a zero scale becomes eps after the zero point is formed
template <int DT> CT_HD float obs_scale_zp(float lo, float hi, bool asym, float qmin, float qmax, float& zq) {
    float s;
    zq = 0.f;
    if (asym) {
        s = obs_round<DT>(hd_div(obs_round<DT>(hd_sub(hi, lo)), qmax - qmin));
        float z = obs_round<DT>(hd_sub(qmin, obs_round<DT>(hd_div(lo, s))));
        z = clamp_nan(z, qmin, qmax);
        z = clamp_nan(z, -128.f, 127.f);
        zq = (z != z) ? 0.f : rintf(z);                        // round(...).to(int8); NaN (0/0) -> 0
    } else {
        s = obs_sym_scale<DT>(lo, hi, qmin, qmax);
    }
    return s == 0.f ? obs_eps<DT>() : s;
}

// scale_dtype = float8_e4m3fn: clamp to +-448, .to(float8_e4m3fn) (round_to_quantized_type_dtype) and back; a zero scale becomes 0.125.
// `byte` is the stored e4m3 code (0x7f for NaN).  v is the scale in the dtype the reference holds it in (fp32 after a global scale).
CT_HD float obs_fp8_scale(float v, uint32_t& byte) {
    byte = hd_f32_to_e4m3(clamp_nan(v, -448.0f, 448.0f));
    float sf = hd_e4m3_to_f32(byte);
    if (sf == 0.f) { sf = 0.125f; byte = 0x20u; }             // eps of the scale dtype; 0x20 = 0.125 in e4m3
    if (sf != sf) byte = 0x7fu;
    return sf;
}

// MX scales (scale_dtype = uint8, group 32): generate_mx_scales of max |x| (mxfp_utils.py:70-139: round_to_power_2 on DT's bits, then
// 127 + floor(log2(.)) - floor(log2(element max))), rounded to uint8, and maybe_convert_from_mx_exp (2^(e - 127) in float32, .to(DT)).
// A power of two that underflows DT gives 0, which becomes the uint8 eps, 1.  amax >= 0 in DT; returns the scale in DT.
template <int DT> CT_HD float obs_mx_scale(float amax, int num_bits) {
    static_assert(DT == CT_BF16 || DT == CT_F16, "MX scales are generated in bf16 / fp16");
    // a NaN amax takes the scale of a zero one.  The reference works on the NaN's bits: most NaNs its CPU reductions return (0x7fff,
    // 0xffff) mask to +-0 as here, a canonical one to +inf, and which one it returns varies with the NaN's position in the group
    float p;
    if constexpr (DT == CT_BF16) {
        const uint32_t u = ((uint32_t)hd_bf16_bits(amax) + 32u) & 0xff80u;   // + 2^(7 - 1 - 1), keep sign and exponent
        p = hd_bf16_value((uint16_t)(u & 0xffffu));
    } else {
        const uint32_t h = (uint32_t)__half_as_ushort(__float2half_rn(amax));
        const uint32_t u = (h + 256u) & 0xfc00u;                               // + 2^(10 - 1 - 1)
        p = __half2float(__ushort_as_half((unsigned short)(u & 0xffffu)));
    }
    if (amax != amax) p = 0.f;
    // p is 0, a power of two or inf: log2 is exact, and so is every sum below in DT (integers of magnitude < 256)
    const float e = p == 0.f ? -INFINITY : (p == INFINITY ? INFINITY : (float)ilogbf(p));
    const float biased = e + 127.0f - (num_bits == 4 ? 2.0f : 8.0f);
    const int code = (int)rintf(fminf(fmaxf(biased, 0.0f), 255.0f));          // round_to_quantized_type_dtype(uint8)
    const float s = obs_round<DT>(code == 255 ? INFINITY : ldexpf(1.0f, code - 127));
    return s == 0.f ? 1.0f : s;
}

// compress_mx_scale (compressors/mx_utils.py:18-31) of one scale v held in dtype dt: 127 + floor(log2(v)) with log2 and floor in dt,
// .to(int32), .to(uint8) (wraps).  Exact for powers of two (what obs_mx_scale produces); log2f elsewhere.  inf / NaN / 0 take int32's
// minimum, as torch's conversion gives on x86, so they store 127.
CT_HD uint32_t mx_scale_code(float v, int dt) {
    float l;
    uint32_t u;
    memcpy(&u, &v, 4);
    if (v > 0.f && (u & 0x007fffffu) == 0u && (u >> 23) != 0u && (u >> 23) != 255u) l = (float)((int)(u >> 23) - 127);
    else l = floorf(rnd_dt(log2f(v), dt));
    const int e = (l != l || isinf(l)) ? (int)0x80000000 : (int)l;
    return (uint32_t)(uint8_t)(uint32_t)(127 + (long long)e);
}

}  // namespace ctb

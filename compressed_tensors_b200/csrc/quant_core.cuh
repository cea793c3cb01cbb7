// quant_core.cuh -- register-level arithmetic of quantize / dequantize, bit-exact with the
// reference's per-op rounding (forward_helpers.py:523-572, quant_args.py:460-496).
//
// The reference evaluates x/scale, +zero_point, clamp, round and the final cast as SEPARATE
// torch ops, each rounding to the tensor dtype ("compute dtype" T).  For 16-bit T the kernels
// keep pairs of values packed in one 32-bit register (T2) and use the native packed
// add/min/max/mul instructions, whose single IEEE rounding equals ATen's
// "widen to fp32, op, narrow with RNE" because sums/products of two 8- or 11-bit significands
// are exact in fp32.
//
// Division.  ATen computes T(fp32(x) / fp32(s)).  For T = bf16 the quotient of two 8-bit
// significands is never within 2^-17 (relative) of a bf16 rounding boundary unless it lies exactly
// on a representable value, and exact ties cannot occur, so T(x * rcp(s)) with a 1-ulp reciprocal
// gives the identical result.  For T = fp16 (11-bit significands) the margin is 2^-23, so the
// product is refined to the correctly rounded fp32 quotient with one residual FMA step first.
// ct_selftest_division() proves both claims on the device for all 2^32 operand pairs.  Scales
// outside [2^-100, 2^100] (where the reciprocal could over/underflow) and fp32 operands use true
// IEEE division (div.rn.f32).
#pragma once

#include <cmath>
#include <cstring>

#include "common.cuh"

namespace ctb {

// ------------------------------------------------------------------------------------
// 16-bit pair traits
// ------------------------------------------------------------------------------------
struct BF16 {
    using T2 = __nv_bfloat162;
    static constexpr int DT = CT_BF16;
    // magic for round-to-integer by addition: 1.5 * 2^7, ulp 1 on [128, 256)
    static constexpr uint32_t MAGIC2 = 0x43404340u;  // 192.0 | 192.0
    static constexpr int MAGIC_MAX_BITS = 7;          // |n| <= 64 keeps 192+n inside [128, 256)
    static constexpr uint32_t ONE_TWENTY_EIGHT2 = 0x43004300u;  // 128.0: exponent with ulp 1
    static constexpr uint32_t OFF8_2 = 0x43084308u;              // 136.0 = 128 + 8
    __device__ static __forceinline__ float lo(uint32_t v) { return __uint_as_float(v << 16); }
    __device__ static __forceinline__ float hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }
    __device__ static __forceinline__ uint32_t pack(float a, float b) {
        __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&t);
    }
    __device__ static __forceinline__ uint32_t from_float1(float a) { return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(a)); }
};
struct F16 {
    using T2 = __half2;
    static constexpr int DT = CT_F16;
    static constexpr uint32_t MAGIC2 = 0x66006600u;  // 1536.0 = 1.5 * 2^10, ulp 1 on [1024, 2048)
    static constexpr int MAGIC_MAX_BITS = 8;
    static constexpr uint32_t ONE_TWENTY_EIGHT2 = 0x64006400u;  // 1024.0: exponent with ulp 1
    static constexpr uint32_t OFF8_2 = 0x64086408u;              // 1032.0 = 1024 + 8
    __device__ static __forceinline__ float lo(uint32_t v) { return __low2float(*reinterpret_cast<__half2*>(&v)); }
    __device__ static __forceinline__ float hi(uint32_t v) { return __high2float(*reinterpret_cast<__half2*>(&v)); }
    __device__ static __forceinline__ uint32_t pack(float a, float b) {
        __half2 t = __floats2half2_rn(a, b);
        return *reinterpret_cast<uint32_t*>(&t);
    }
    __device__ static __forceinline__ uint32_t from_float1(float a) { return (uint32_t)__half_as_ushort(__float2half_rn(a)); }
};

template <class P> __device__ __forceinline__ uint32_t add2(uint32_t a, uint32_t b) {
    typename P::T2 r = __hadd2(*reinterpret_cast<typename P::T2*>(&a), *reinterpret_cast<typename P::T2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <class P> __device__ __forceinline__ uint32_t sub2(uint32_t a, uint32_t b) {
    typename P::T2 r = __hsub2(*reinterpret_cast<typename P::T2*>(&a), *reinterpret_cast<typename P::T2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <class P> __device__ __forceinline__ uint32_t mul2(uint32_t a, uint32_t b) {
    typename P::T2 r = __hmul2(*reinterpret_cast<typename P::T2*>(&a), *reinterpret_cast<typename P::T2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <class P> __device__ __forceinline__ uint32_t max2(uint32_t a, uint32_t b) {
    typename P::T2 r = __hmax2(*reinterpret_cast<typename P::T2*>(&a), *reinterpret_cast<typename P::T2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <class P> __device__ __forceinline__ uint32_t min2(uint32_t a, uint32_t b) {
    typename P::T2 r = __hmin2(*reinterpret_cast<typename P::T2*>(&a), *reinterpret_cast<typename P::T2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
// NaN-propagating packed min / max (max.NaN / min.NaN): torch.clamp, amin and amax give NaN where an operand is NaN, while
// max2 / min2 return the other operand
template <class P> __device__ __forceinline__ uint32_t max2_nan(uint32_t a, uint32_t b) {
    typename P::T2 r = __hmax2_nan(*reinterpret_cast<typename P::T2*>(&a), *reinterpret_cast<typename P::T2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <class P> __device__ __forceinline__ uint32_t min2_nan(uint32_t a, uint32_t b) {
    typename P::T2 r = __hmin2_nan(*reinterpret_cast<typename P::T2*>(&a), *reinterpret_cast<typename P::T2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}
template <class P> __device__ __forceinline__ uint32_t dup2(float v) {
    uint32_t h = P::from_float1(v);
    return h | (h << 16);
}

// ------------------------------------------------------------------------------------
// per-scale context
// ------------------------------------------------------------------------------------
struct ScaleCtx {
    float s;     // scale as fp32
    float r;     // reciprocal (fast path)
    bool slow;   // scale outside the proven-safe range -> IEEE division per element
};
__device__ __forceinline__ ScaleCtx make_scale_ctx(float s) {
    ScaleCtx c;
    c.s = s;
    float a = fabsf(s);
    c.slow = !(a >= 7.888609052210118e-31f && a <= 1.2676506002282294e30f);  // [2^-100, 2^100]; NaN -> slow
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(s));
    c.r = r;
    return c;
}

// fp32 quotient that rounds to T exactly like fp32(x)/fp32(s) does.  SLOW is decided once per
// chunk (scale outside the proven range) and selects IEEE division.
template <class P, bool SLOW = false>
__device__ __forceinline__ float quot(float x, const ScaleCtx& c) {
    if (SLOW) return __fdiv_rn(x, c.s);
    float q = __fmul_rn(x, c.r);
    if (P::DT == CT_F16) {
        // one residual step -> correctly rounded fp32 quotient.  Skipped when the first product is
        // +-0 (the FMA chain would turn -0 into +0) or +-inf / NaN (inf - inf).
        float rem = __fmaf_rn(-q, c.s, x);
        float q1 = __fmaf_rn(rem, c.r, q);
        const float a = fabsf(q);
        q = (a > 0.f && a < __int_as_float(0x7f800000)) ? q1 : q;
    }
    return q;
}

// x pair (raw T2 bits) -> clamped value in T, before rounding to the quantized grid.
// zp2: zero point already converted to T (zero_point.to(x.dtype)), duplicated in both halves.
// NAN_CLAMP keeps a NaN through the clamp as torch.clamp does (fake_quantize, whose output is a float); the ops that produce codes
// leave it off, since the code of a NaN is undefined in the reference.
template <class P, bool NAN_CLAMP>
__device__ __forceinline__ uint32_t clamp2(uint32_t t, uint32_t qmin2, uint32_t qmax2) {
    if constexpr (NAN_CLAMP) return min2_nan<P>(max2_nan<P>(t, qmin2), qmax2);
    else return min2<P>(max2<P>(t, qmin2), qmax2);
}
// out-of-line IEEE-division variant (rare: scale outside [2^-100, 2^100]); scalar by-value
// arguments so that nothing is forced into local memory
template <class P, bool HAS_ZP, bool NAN_CLAMP>
__device__ __noinline__ uint32_t scaled_clamped2_slow(uint32_t xv, float s, uint32_t zp2, uint32_t qmin2, uint32_t qmax2) {
    uint32_t t = P::pack(__fdiv_rn(P::lo(xv), s), __fdiv_rn(P::hi(xv), s));
    if (HAS_ZP) t = add2<P>(t, zp2);
    return clamp2<P, NAN_CLAMP>(t, qmin2, qmax2);
}
template <class P, bool HAS_ZP, bool SLOW, bool NAN_CLAMP = false>
__device__ __forceinline__ uint32_t scaled_clamped2(uint32_t xv, const ScaleCtx& c, uint32_t zp2, uint32_t qmin2, uint32_t qmax2) {
    if constexpr (SLOW) return scaled_clamped2_slow<P, HAS_ZP, NAN_CLAMP>(xv, c.s, zp2, qmin2, qmax2);
    float q0 = quot<P, false>(P::lo(xv), c);
    float q1 = quot<P, false>(P::hi(xv), c);
    uint32_t t = P::pack(q0, q1);                // scaled = x / scale          (rounds to T)
    if (HAS_ZP) t = add2<P>(t, zp2);             // scaled += zero_point.to(T)  (rounds to T)
    return clamp2<P, NAN_CLAMP>(t, qmin2, qmax2);   // torch.clamp
}

// round-half-even of a clamped T2 pair; result n has two's complement in the low bits of each half
// (valid when BITS <= P::MAGIC_MAX_BITS).
template <class P>
__device__ __forceinline__ uint32_t round_magic2(uint32_t t) { return add2<P>(t, P::MAGIC2); }

// the rounded value as T with the sign of zero preserved (torch.round(-0.3) == -0.0)
template <class P>
__device__ __forceinline__ uint32_t round_keep_sign2(uint32_t t) {
    uint32_t r = sub2<P>(add2<P>(t, P::MAGIC2), P::MAGIC2);
    return (r & 0x7fff7fffu) | (t & 0x80008000u);
}

// general (any BITS up to 8) integer rounding through fp32: returns the two int values
__device__ __forceinline__ int rint_magic_f32(float v) {
    // v already clamped to [-128, 127]
    return (int)(__float_as_uint(__fadd_rn(v, 12582912.0f)) & 0x7fffffu) - 0x400000;
}

// float pair -> two e4m3 bytes (lo in bits 0-7), RNE; inputs are already clamped to +-448
__device__ __forceinline__ uint32_t f32x2_to_e4m3x2(float lo, float hi) {
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return (uint32_t)r;
}
// two e4m3 bytes -> half2 bits (exact)
__device__ __forceinline__ uint32_t e4m3x2_to_f16x2(uint32_t two_bytes) {
    uint32_t r;
    uint16_t in = (uint16_t)two_bytes;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(in));
    return r;
}
// one word of four e4m3 bytes -> two half2 (bytes 0,1 -> h0; bytes 2,3 -> h1): the half-word selection is part of the conversion
// instruction (F2FP.F16.E4M3.UNPACK_B Rd, Rs.H1), no shift / mask
__device__ __forceinline__ void e4m3x4_to_f16x4(uint32_t w, uint32_t& h0, uint32_t& h1) {
    asm("{ .reg .b16 a, b;\n"
        "mov.b32 {a, b}, %2;\n"
        "cvt.rn.f16x2.e4m3x2 %0, a;\n"
        "cvt.rn.f16x2.e4m3x2 %1, b; }" : "=r"(h0), "=r"(h1) : "r"(w));
}
__device__ __forceinline__ float e4m3_to_f32(uint32_t byte) {
    uint32_t h2 = e4m3x2_to_f16x2(byte & 0xffu);
    return __low2float(*reinterpret_cast<__half2*>(&h2));
}

// ------------------------------------------------------------------------------------
// scalar (fp32 compute dtype / generic path) helpers.  `rnd` narrows to dtype dt and widens back.
// These are __host__ __device__: the generic kernels (generic.cu) and the CPU twins of the ABI (cpu_twin.cu, device = -1) run the
// SAME per-element arithmetic source.  On the host the IEEE operators stand in for the round-to-nearest intrinsics (the library is
// built without fast-math and with -ffp-contract=off) and cuda_fp8.h's software conversion for the e4m3 PTX instruction.
// ------------------------------------------------------------------------------------
#define CT_HD __host__ __device__ __forceinline__

CT_HD float hd_div(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}
CT_HD float hd_add(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}
CT_HD float hd_sub(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(a, b);
#else
    return a - b;
#endif
}
CT_HD float hd_mul(float a, float b) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
CT_HD uint8_t hd_f32_to_e4m3(float v) {
#ifdef __CUDA_ARCH__
    return (uint8_t)(f32x2_to_e4m3x2(v, 0.f) & 0xffu);
#else
    return (uint8_t)__nv_cvt_float_to_fp8(v, __NV_SATFINITE, __NV_E4M3);
#endif
}
CT_HD float hd_e4m3_to_f32(uint32_t byte) {
#ifdef __CUDA_ARCH__
    return e4m3_to_f32(byte);
#else
    const __half_raw h = __nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)(byte & 0xffu), __NV_E4M3);
    return __half2float(__half(h));
#endif
}
// bfloat16 round-to-nearest-even on raw bits: cuda_bf16.h's host conversions are correct but ~10x slower than this on a CPU
CT_HD uint16_t hd_bf16_bits(float v) {
#ifdef __CUDA_ARCH__
    return __bfloat16_as_ushort(__float2bfloat16_rn(v));
#else
    uint32_t u;
    memcpy(&u, &v, 4);
    if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x0040u);   // NaN stays NaN (quiet)
    u += 0x7fffu + ((u >> 16) & 1u);
    return (uint16_t)(u >> 16);
#endif
}
CT_HD float hd_bf16_value(uint16_t h) {
#ifdef __CUDA_ARCH__
    return __uint_as_float((uint32_t)h << 16);
#else
    const uint32_t u = (uint32_t)h << 16;
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
CT_HD float rnd_dt(float v, int dt) {
    if (dt == CT_BF16) return hd_bf16_value(hd_bf16_bits(v));
    if (dt == CT_F16) return __half2float(__float2half_rn(v));
    return v;
}
CT_HD float load_as_f32(const void* p, int64_t i, int dt) {
    switch (dt) {
    case CT_F32: return reinterpret_cast<const float*>(p)[i];
    case CT_F16: return __half2float(reinterpret_cast<const __half*>(p)[i]);
    case CT_BF16: return hd_bf16_value(reinterpret_cast<const uint16_t*>(p)[i]);
    case CT_I8: return (float)reinterpret_cast<const int8_t*>(p)[i];
    case CT_U8: return (float)reinterpret_cast<const uint8_t*>(p)[i];
    case CT_F8E4M3: return hd_e4m3_to_f32(reinterpret_cast<const uint8_t*>(p)[i]);
    case CT_I32: return (float)reinterpret_cast<const int32_t*>(p)[i];
    case CT_I64: return (float)reinterpret_cast<const int64_t*>(p)[i];
    case CT_E8M0: {   // stored MX scale: 2^(e - 127) decoded through bfloat16 (mx_utils.py:43-44), so e = 255 is +inf
        const int e = (int)reinterpret_cast<const uint8_t*>(p)[i];
        return e == 255 ? INFINITY : ldexpf(1.0f, e - 127);
    }
    default: return 0.f;
    }
}
// NaN-propagating min / max (min.NaN / max.NaN on the device), the scalar counterparts of min2_nan / max2_nan
CT_HD float fmin_nan(float a, float b) {
#ifdef __CUDA_ARCH__
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
#else
    return (a != a || b != b) ? a + b : fminf(a, b);
#endif
}
CT_HD float fmax_nan(float a, float b) {
#ifdef __CUDA_ARCH__
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
#else
    return (a != a || b != b) ? a + b : fmaxf(a, b);
#endif
}
CT_HD float clamp_nan(float v, float lo, float hi) {
    // torch.clamp propagates NaN
    return (v != v) ? v : fminf(fmaxf(v, lo), hi);
}
__device__ __forceinline__ uint8_t f32_to_e4m3_byte(float v) { return (uint8_t)(f32x2_to_e4m3x2(v, 0.f) & 0xffu); }

// FP4_E2M1_DATA.cast_to_fp4 (quantization/utils/fp4_utils.py:77-98) on one value: |x| snapped by the closed / open
// interval ladder, times torch.sign(x) -- so +-0 -> +0, small negatives -> -0, NaN stays NaN
CT_HD float fp4_round(float v) {
    const float a = fabsf(v);
    float r = a <= 0.25f ? 0.0f : a < 0.75f ? 0.5f : a <= 1.25f ? 1.0f : a < 1.75f ? 1.5f : a <= 2.5f ? 2.0f : a < 3.5f ? 3.0f : a <= 5.0f ? 4.0f : 6.0f;
    if (v != v) return v;
    return v > 0.f ? r : (v < 0.f ? -r : 0.0f);
}
// nibble of an fp4 VALUE (compressors/nvfp4/helpers.py:141-156): index of |v| in the E2M1 table, bit 3 = sign bit
__device__ __forceinline__ uint32_t fp4_nibble(float v) {
    const int a = abs((int)(int8_t)(int)(v * 2.0f));
    const uint32_t idx = a == 1 ? 1u : a == 2 ? 2u : a == 3 ? 3u : a == 4 ? 4u : a == 6 ? 5u : a == 8 ? 6u : a >= 12 ? 7u : 0u;
    return idx | ((__float_as_uint(v) >> 28) & 8u);
}
__device__ __forceinline__ float fp4_value(uint32_t nib) {
    const float mag = (nib & 4u) ? ((nib & 2u) ? ((nib & 1u) ? 6.0f : 4.0f) : ((nib & 1u) ? 3.0f : 2.0f))
                                 : ((nib & 2u) ? ((nib & 1u) ? 1.5f : 1.0f) : ((nib & 1u) ? 0.5f : 0.0f));
    return (nib & 8u) ? -mag : mag;
}

// value of `quantized_ground` before the final .to(dtype), in compute dtype cd
CT_HD float quant_scalar(float x, float s, bool has_zp, float zp_in_xdt, int cd, int qtype, float qmin, float qmax) {
    float t = rnd_dt(hd_div(x, s), cd);
    if (has_zp) t = rnd_dt(hd_add(t, zp_in_xdt), cd);
    t = clamp_nan(t, qmin, qmax);
    if (qtype == CT_Q_INT) t = rintf(t);
    else if (qtype == CT_Q_FP4) t = fp4_round(t);
    else t = (t != t) ? t : hd_e4m3_to_f32(hd_f32_to_e4m3(t));
    return t;
}
CT_HD void store_from_f32(void* p, int64_t i, int dt, float v) {
    switch (dt) {
    case CT_F32: reinterpret_cast<float*>(p)[i] = v; break;
    case CT_F16: reinterpret_cast<__half*>(p)[i] = __float2half_rn(v); break;
    case CT_BF16: reinterpret_cast<uint16_t*>(p)[i] = hd_bf16_bits(v); break;
    case CT_I8: reinterpret_cast<int8_t*>(p)[i] = (v != v || v - v != 0.f) ? (int8_t)0 : (int8_t)(int)v; break;   // NaN / inf -> 0
    case CT_F8E4M3: reinterpret_cast<uint8_t*>(p)[i] = hd_f32_to_e4m3(v); break;
    case CT_I32: reinterpret_cast<int32_t*>(p)[i] = (int)v; break;
    default: break;
    }
}
__device__ __forceinline__ void q_range(int qtype, int bits, float& qmin, float& qmax) {
    if (qtype == CT_Q_INT) {
        float r = (float)(1 << bits);
        qmax = r * 0.5f - 1.f;
        qmin = -r * 0.5f;
    } else {
        qmax = 448.f;
        qmin = -448.f;
    }
}

}  // namespace ctb

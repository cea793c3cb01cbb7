// fp4_ops.cuh -- streaming functors of the FP4 formats (stream.cuh pipelines):
//   Fp4NvQuantPackOp   x (bf16 / fp16) -> E2M1 nibbles, fp32 arithmetic with  scale / global_scale  per group of 16 (NVFP4)
//   Fp4MxQuantPackOp   x (bf16 / fp16) -> E2M1 nibbles, arithmetic in x's dtype, one scale per group (MXFP4: group 32)
//   Fp4UnpackDequantOp nibbles -> bf16 / fp16, scale as float, as stored fp8 (NVFP4) or as stored E8M0 exponent (MX)
// Hopper has no E2M1 conversion instruction, so rounding to E2M1 is done in integer arithmetic on the float's bits:
// round-to-nearest-even on the E2M1 grid with saturation at +-6, which IS the closed / open interval ladder of the reference's
// cast_to_fp4 (quantization/utils/fp4_utils.py:89-96; the ties 0.25, 1.25, 2.5, 5.0 go down, 0.75, 1.75, 3.5 go up) preceded
// by the clamp to +-6 (quant_args.py:481).  The sign bit is kept (small negatives give code 8, -0.0), NaN gives +6 (code 7).
// The one difference -- the reference maps an exact -0.0 to +0.0 because it multiplies by torch.sign(x) -- is removed by
// adding +0.0f first.
#pragma once

#include "observe_core.cuh"
#include "observe_mse.cuh"
#include "ops.cuh"

namespace ctb {

// one float -> one E2M1 code (4 bits).  For |x| as an unsigned integer the ladder is a count of thresholds passed; a strict
// threshold t (the ties that go down) is "|x| >= t + 1 ulp"
__device__ __forceinline__ uint32_t f32_to_e2m1(float x) {
    const uint32_t u = __float_as_uint(x), a = u & 0x7fffffffu;
    uint32_t c = (uint32_t)(a >= 0x3e800001u) + (uint32_t)(a >= 0x3f400000u) + (uint32_t)(a >= 0x3fa00001u) + (uint32_t)(a >= 0x3fe00000u)
               + (uint32_t)(a >= 0x40200001u) + (uint32_t)(a >= 0x40600000u) + (uint32_t)(a >= 0x40a00001u);   // 0.25 .75 1.25 1.75 2.5 3.5 5
    c |= (u >> 28) & 8u;
    return a > 0x7f800000u ? 7u : c;
}
// two floats -> one byte of two E2M1 codes, `lo` in the low nibble (compressors/nvfp4/helpers.py:154-156)
__device__ __forceinline__ uint32_t f32x2_to_e2m1x2(float lo, float hi) { return f32_to_e2m1(lo) | (f32_to_e2m1(hi) << 4); }

// eight floats -> one word of eight E2M1 codes, element 0 in the low nibble of byte 0
__device__ __forceinline__ uint32_t f32x8_to_e2m1x8(float f0, float f1, float f2, float f3, float f4, float f5, float f6, float f7) {
    return f32_to_e2m1(f0) | (f32_to_e2m1(f1) << 4) | (f32_to_e2m1(f2) << 8) | (f32_to_e2m1(f3) << 12) | (f32_to_e2m1(f4) << 16)
         | (f32_to_e2m1(f5) << 20) | (f32_to_e2m1(f6) << 24) | (f32_to_e2m1(f7) << 28);
}
// one word of eight E2M1 codes -> four half2 (byte j -> h[j], low nibble in the low half; exact, code 8 is -0.0).
// Code s|eem placed at fp16 bits 15 and 11..9 is the fp16 number (e2m1 value) * 2^-14 -- E2M1's subnormal (e = 0) lands on fp16's
// subnormals with the same scale -- so one packed multiply by 2^14 finishes two elements
__device__ __forceinline__ void e2m1x8_to_f16x8(uint32_t w, uint32_t (&h)[4]) {
    const __half2 two14 = __half2half2(__ushort_as_half((unsigned short)0x7400u));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t b = w >> (8 * j);
        const uint32_t t = (b & 0xfu) | ((b & 0xf0u) << 12);                      // nibble 0 -> bits 0..3, nibble 1 -> bits 16..19
        uint32_t v = ((t & 0x00070007u) << 9) | ((t & 0x00080008u) << 12);
        __half2 x = __hmul2(*reinterpret_cast<__half2*>(&v), two14);
        h[j] = *reinterpret_cast<uint32_t*>(&x);
    }
}

// RN(x / s) through r = RN(1 / s) and one residual step: q0 = x r, e = fma(-q0, s, x), q1 = fma(e, r, q0).  No branches; the
// callers keep the operands in ranges where nothing over- or underflows and ct_selftest_fp4_division checks the result
// against div.rn exhaustively (every 16-bit x, every float32 significand of s).
__device__ __forceinline__ float recip_div(float x, float s, float rcp) {
    const float q0 = __fmul_rn(x, rcp);
    const float e = __fmaf_rn(-q0, s, x);
    return __fmaf_rn(e, rcp, q0);
}

enum Fp4ScaleKind { FS_SAME = 0, FS_F32 = 1, FS_F8 = 2, FS_E8M0 = 3 };   // how the scale tensor is held
enum Fp4ZpKind { FZ_NONE = 0, FZ_F8 = 1, FZ_U8 = 2, FZ_I8 = 3 };         // zero point of a symmetric scheme (zeros), added like the reference does

template <int ZK>
__device__ __forceinline__ float fp4_zp_value(uint32_t byte) {
    if constexpr (ZK == FZ_F8) return e4m3_to_f32(byte);
    else if constexpr (ZK == FZ_U8) return (float)(byte & 0xffu);
    else if constexpr (ZK == FZ_I8) return (float)(int)(int8_t)(byte & 0xffu);
    else return 0.f;
}

// ------------------------------------------------------------------------------------
// NVFP4 quantize + pack.  unit = 4 chunks = 32 elements = two groups of 16 -> one 16-byte store.
//   reference: scale = scale / global_scale (fp32); scaled = x / scale (fp32); scaled += zp.to(x.dtype); clamp; cast_to_fp4;
//   .to(x.dtype); pack_fp4_to_uint8      (forward_helpers.py:535-546, nvfp4/base.py:82-90)
// Division: q = RN(x / s) through the correctly rounded reciprocal r = RN(1/s) and one residual step
//   q0 = x r,  e = fma(-q0, s, x),  q1 = fma(e, r, q0)
// (exhaustively checked against div.rn for every 16-bit x and every scale significand by ct_selftest_fp4_division);
// groups whose effective scale falls outside [2^-100, 2^10] (negative ones included) take div.rn per element.
// ------------------------------------------------------------------------------------
// per-tile constants of the ops that divide a scale by the tensor's global scale
struct Fp4DqTile {
    float gs, rgs;   // global scale of the tensor and its correctly rounded reciprocal
    bool has, fast;  // fast: |gs| in [2^-60, 2^60] -> scale / gs by recip_div for |scale| in [2^-40, 2^14] (exhaustively checked)
};

struct Fp4NvRaw {
    uint32_t s0, s1;   // the unit's two group scales (bit patterns)
    uint32_t z;        // two zero-point bytes
    float gs;
};

template <class P, int SK, int ZK>
struct Fp4NvQuantPackOp {
    static_assert(SK == FS_SAME || SK == FS_F32, "NVFP4 quantization takes float scales");
    static constexpr int IN_BYTES = 16;
    static constexpr int GROUP = 4;
    using Raw = Fp4NvRaw;

    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc0) {
        Raw r;
        const uint32_t si = gc0 >> 1;   // group of 16 elements = 2 chunks; gc0 % 4 == 0 so si is even
        if constexpr (SK == FS_F32) {
            const uint2 v = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const float*>(J.scale) + si));
            r.s0 = v.x; r.s1 = v.y;
        } else {
            // raw word only: nothing in prefetch() may depend on a load (it would wait for it a whole tile early); run() splits it
            r.s0 = __ldg(reinterpret_cast<const uint32_t*>(reinterpret_cast<const unsigned short*>(J.scale) + si));
            r.s1 = 0;
        }
        r.z = 0;
        if constexpr (ZK != FZ_NONE) r.z = __ldg(reinterpret_cast<const unsigned short*>(reinterpret_cast<const uint8_t*>(J.zp) + si));
        r.gs = __ldg(reinterpret_cast<const float*>(J.aux));
        return r;
    }
    __device__ static __forceinline__ float scale_value(uint32_t bits) {
        if constexpr (SK == FS_F32) return __uint_as_float(bits);
        else { RawQP q; q.s = bits; q.z = 0; return scale_f32<P>(q); }
    }
    // fast quotient: reciprocal + one residual step (no branches).  |x| <= 2^14 here (clamp_x), |1/s| <= 2^100: no overflow
    __device__ static __forceinline__ float quotient(float x, float s, float rcp) { return recip_div(x, s, rcp); }
    // x pair clamped to +-2^14 (packed min / max).  With |s| <= 2^10 every |x| >= 2^14 quantizes to +-6 anyway (|x / s| >= 16),
    // so the codes do not change, and the products above can no longer overflow to inf (inf - inf = NaN in the residual).
    __device__ static __forceinline__ uint32_t clamp_x(uint32_t w) {
        constexpr uint32_t HI = (P::DT == CT_BF16) ? 0x46804680u : 0x74007400u;   // 16384.0 as bf16 / fp16, both halves
        return min2<P>(max2<P>(w, HI | 0x80008000u), HI);
    }
    // one chunk (8 elements, 4 packed words) -> 4 bytes of nibbles.  CLAMP = false: the caller knows every |x| <= 2^14 already
    // (the fused observer has the group's max |x| in hand), so clamp_x would be the identity
    template <bool CLAMP = true>
    __device__ static __forceinline__ uint32_t chunk_fast(const uint32_t (&w)[4], float s, float rcp, float z) {
        float t[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t xc = CLAMP ? clamp_x(w[j]) : w[j];
            t[2 * j] = quotient(P::lo(xc), s, rcp);
            t[2 * j + 1] = quotient(P::hi(xc), s, rcp);
            // the reference's in-place add of the zero point.  Without one nothing is added: with s in (0, 2^10] the residual step
            // already turns x = -0.0 into +0.0 (fma(+0, r, -0) = +0) and no non-zero 16-bit x underflows to -0.0
            if constexpr (ZK != FZ_NONE) { t[2 * j] = __fadd_rn(t[2 * j], z); t[2 * j + 1] = __fadd_rn(t[2 * j + 1], z); }
        }
        return f32x8_to_e2m1x8(t[0], t[1], t[2], t[3], t[4], t[5], t[6], t[7]);
    }
    // out of line, everything by value: a unit whose effective scale is outside [2^-100, 2^10] (or <= 0 / inf / NaN) -> IEEE division
    // per element.  One call per unit so that the caller's registers never have to be spilled to be indexed.
    __device__ static __noinline__ uint4 unit_slow(uint4 c0, uint4 c1, uint4 c2, uint4 c3, float s0, float s1, float z0, float z1, int off) {
        const uint4 c[4] = {c0, c1, c2, c3};
        uint32_t o[4];
#pragma unroll 1
        for (int k = 0; k < 4; ++k) {
            const bool g = ((k + off) >> 1) & 1;
            const float s = g ? s1 : s0, z = g ? z1 : z0;
            const uint32_t w[4] = {c[k].x, c[k].y, c[k].z, c[k].w};
            uint32_t word = 0;
#pragma unroll 1
            for (int j = 0; j < 4; ++j) {
                // the trailing + 0.0f maps a zero quotient to +0.0 as the reference's torch.sign does: x / s is -0.0 for x = -0.0
                // under s > 0 and for x = +0.0 under s < 0, and a -0.0 zero point (fp8 byte 0x80) keeps it so
                const float t0 = __fadd_rn(__fadd_rn(__fdiv_rn(P::lo(w[j]), s), z), 0.0f);
                const float t1 = __fadd_rn(__fadd_rn(__fdiv_rn(P::hi(w[j]), s), z), 0.0f);
                word |= f32x2_to_e2m1x2(t0, t1) << (8 * j);
            }
            o[k] = word;
        }
        return make_uint4(o[0], o[1], o[2], o[3]);
    }
    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw& r, uint32_t gc0, const uint32_t (&w)[4][4], int off) {
        float s[2], rc[2], z[2];
        const uint32_t b0 = (SK == FS_F32) ? r.s0 : (r.s0 & 0xffffu), b1 = (SK == FS_F32) ? r.s1 : (r.s0 >> 16);
        s[0] = __fdiv_rn(scale_value(b0), r.gs);
        s[1] = __fdiv_rn(scale_value(b1), r.gs);
        bool slow = false;
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            // [2^-100, 2^10]; a negative or NaN scale goes slow too: under a negative s the residual step turns x = +0.0 into -0.0,
            // where the reference's torch.sign gives +0.0
            slow |= !(s[g] >= 7.888609052210118e-31f && s[g] <= 1024.0f);
            rc[g] = __frcp_rn(s[g]);
            // zero_point.to(x.dtype): fp8 / small integers are exact in bf16 and fp16
            z[g] = fp4_zp_value<ZK>(r.z >> (8 * g));
        }
        uint32_t o[4];
        if (slow) {
            const uint4 v = unit_slow(make_uint4(w[0][0], w[0][1], w[0][2], w[0][3]), make_uint4(w[1][0], w[1][1], w[1][2], w[1][3]),
                                      make_uint4(w[2][0], w[2][1], w[2][2], w[2][3]), make_uint4(w[3][0], w[3][1], w[3][2], w[3][3]),
                                      s[0], s[1], z[0], z[1], off);
            o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const bool g = ((k + off) >> 1) & 1;   // chunk (k + off) mod 4 belongs to group 0 or 1 of the unit
                o[k] = chunk_fast(w[k], g ? s[1] : s[0], g ? rc[1] : rc[0], g ? z[1] : z[0]);
            }
        }
        rotate_out<4, 1>(o, off);
        store_words<4>(J.out + (size_t)gc0 * 4, o);
    }
};

// ------------------------------------------------------------------------------------
// NVFP4 observe + quantize + pack: the per-group part of the observer fused in front of Fp4NvQuantPackOp.
//   reference: min / max per group of 16 -> calculate_qparams(args NVFP4, global_scale) (quantization/utils/helpers.py:50-137:
//   max|x| / 6 in T, x global_scale in float32, clamp to +-448 and .to(float8_e4m3fn), 0 -> 0.125) -> quantize -> pack.
//   The global scale (generate_gparam over the whole tensor, helpers.py:308-337) is an INPUT: it needs a grid-wide reduction
//   that has to finish before any group can be scaled.  Outputs: nibbles and the group scales as stored (float8_e4m3fn).
// J.scale is written here (uint8 [n / 16]); J.aux = global scale.
// MSE = true: J.zp (no zero point exists for this op) = the call's ct_mse_block; each group of 16 searches its max |x| shrink grid
// (observe_mse.cuh) with the global scale fixed, and is written with its best improving step (mse_fixup_nvfp4_kernel applies the stop).
// ------------------------------------------------------------------------------------
template <class P, bool MSE = false>
struct Fp4NvObserveQuantPackOp {
    static constexpr int IN_BYTES = 16;
    static constexpr int GROUP = 4;
    using Raw = NoRaw;
    __device__ static __forceinline__ Raw prefetch(const Job&, uint32_t) { return {}; }
    // per tile: the tensor's global scale, its reciprocal, and whether scale / global_scale may use recip_div (as in Fp4DqTile)
    using Tile = Fp4DqTile;
    __device__ static __forceinline__ Tile tile(const Job& J) {
        Tile t;
        t.has = true;
        t.gs = __ldg(reinterpret_cast<const float*>(J.aux));
        t.rgs = __frcp_rn(t.gs);
        const float a = fabsf(t.gs);
        t.fast = a >= 8.673617379884035e-19f && a <= 1.152921504606847e18f;
        return t;
    }
    // packed max(|a|, |b|): max.xorsign.abs takes the larger magnitude (its sign is the xor of the input signs, cleared at the end)
    __device__ static __forceinline__ uint32_t amax2(uint32_t a, uint32_t b) {
        uint32_t r;
        if constexpr (P::DT == CT_BF16) asm("max.xorsign.abs.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
        else asm("max.xorsign.abs.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
        return r;
    }
    // max |x| of one chunk as packed T2
    __device__ static __forceinline__ uint32_t chunk_amax2(const uint32_t (&w)[4]) { return amax2(amax2(w[0], w[1]), amax2(w[2], w[3])) & 0x7fff7fffu; }
    // group scale as the reference derives it from max |x| (calculate_qparams, helpers.py:50-137): the stored e4m3 byte and its value
    //   DIV = true : IEEE divisions; DIV = false: recip_div, valid for amax == 0 or amax in [2^-40, 2^14] (selftest mode 1; 6.0 is
    //   one of the float32 significands it covers) -- the caller checks the range
    template <bool DIV>
    __device__ static __forceinline__ float group_scale(float amax, float gs, uint32_t& byte) {
        const float q6 = DIV ? __fdiv_rn(amax, 6.0f) : recip_div(amax, 6.0f, 0.16666667163372039794921875f);   // max_val_pos / (bit_range / 2)
        return obs_fp8_scale(__fmul_rn(gs, obs_round<P::DT>(q6)), byte);          // ... in T, x global_scale (float32), as e4m3
    }
    struct SlowOut {
        uint4 nibbles;
        uint32_t codes;
    };
    // out of line, everything by value: a unit with a group outside the ranges the shortcuts are proven for (max |x| above 2^14 or
    // below 2^-40, a global scale outside [2^-60, 2^60], an effective scale outside [2^-100, 2^10] or negative, NaN) -> IEEE division everywhere
    __device__ static __noinline__ SlowOut unit_slow_observe(uint4 c0, uint4 c1, uint4 c2, uint4 c3, float amax0, float amax1, float gs, int off) {
        using Q = Fp4NvQuantPackOp<P, FS_F32, FZ_NONE>;
        uint32_t b0, b1;
        const float s0 = __fdiv_rn(group_scale<true>(amax0, gs, b0), gs);
        const float s1 = __fdiv_rn(group_scale<true>(amax1, gs, b1), gs);
        SlowOut r;
        r.nibbles = Q::unit_slow(c0, c1, c2, c3, s0, s1, 0.f, 0.f, off);
        r.codes = b0 | (b1 << 8);
        return r;
    }
    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw&, uint32_t gc0, const uint32_t (&w)[4][4], int off, const Tile& tc) {
        using Q = Fp4NvQuantPackOp<P, FS_F32, FZ_NONE>;
        const uint32_t m0 = chunk_amax2(w[0]), m1 = chunk_amax2(w[1]), m2 = chunk_amax2(w[2]), m3 = chunk_amax2(w[3]);
        // register k holds chunk (k + off) mod 4; groups are chunks {0, 1} and {2, 3}
        const bool odd = off & 1;
        const uint32_t pa = odd ? max2<P>(m3, m0) : max2<P>(m0, m1);      // the pair that contains register 0
        const uint32_t pb = odd ? max2<P>(m1, m2) : max2<P>(m2, m3);
        const bool a_is_g0 = off < 2;                                        // off 0: regs {0,1} = chunks {0,1}; off 1: regs {3,0} = chunks {0,1}
        const uint32_t g0 = a_is_g0 ? pa : pb, g1 = a_is_g0 ? pb : pa;
        float amax[2], s[2], rc[2];
        uint32_t codes = 0;
        bool slow = !tc.fast;
        amax[0] = fmaxf(P::lo(g0), P::hi(g0));                                             // max(|min(min, 0)|, |max(max, 0)|) = max |x|
        amax[1] = fmaxf(P::lo(g1), P::hi(g1));
        if constexpr (MSE) {
            ct_mse_block* B = reinterpret_cast<ct_mse_block*>(const_cast<void*>(J.zp));
            const float norm = B->norm;
            const bool square = norm == 2.0f;
#pragma unroll
            for (int g = 0; g < 2; ++g) {
                // candidate i: max |x| of the shrunk range is T(max |x| * p_i); the scale as the reference forms it, IEEE divisions
                auto partial = [&](float, float a) {
                    uint32_t byte;
                    const float cs = __fdiv_rn(group_scale<true>(a, tc.gs, byte), tc.gs);
                    float e = 0.f;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if ((((k + off) >> 1) & 1) != g) continue;
#pragma unroll
                        for (int j = 0; j < 4; ++j)
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const float xv = h ? P::hi(w[k][j]) : P::lo(w[k][j]);
                                const float q = fp4_round(fminf(fmaxf(__fdiv_rn(xv, cs), -6.0f), 6.0f));
                                e += mse_pow(rnd_dt(__fmul_rn(q, cs), P::DT) - xv, norm, square);
                            }
                    }
                    return e;
                };
                const uint64_t gi = (uint64_t)(gc0 >> 1) + g;
                uint64_t mask;
                const int best = mse_search<P, 1>(B, 0.f, amax[g], partial, mask, B->errors ? B->errors + gi * B->steps : nullptr);
                mse_publish(B, gi, mask);
                amax[g] = rnd_dt(amax[g] * __ldg(&B->shrink[best]), P::DT);
            }
        }
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            // amax <= 2^14 also means clamp_x is the identity for every element of the group (chunk_fast<false> below)
            slow |= !(amax[g] <= 16384.0f && (amax[g] >= 9.094947017729282e-13f || amax[g] == 0.f));
            uint32_t byte;
            const float sf = group_scale<false>(amax[g], tc.gs, byte);
            codes |= byte << (8 * g);
            // scale / global_scale: an e4m3 value (within [2^-9, 448]) over the global scale, same shortcut as the decompress kernel
            s[g] = recip_div(sf, tc.gs, tc.rgs);
            slow |= !(s[g] >= 7.888609052210118e-31f && s[g] <= 1024.0f);                // [2^-100, 2^10]; negative (gs < 0), NaN -> slow
            rc[g] = __frcp_rn(s[g]);
        }
        uint32_t o[4];
        if (slow) {
            const SlowOut v = unit_slow_observe(make_uint4(w[0][0], w[0][1], w[0][2], w[0][3]), make_uint4(w[1][0], w[1][1], w[1][2], w[1][3]),
                                                make_uint4(w[2][0], w[2][1], w[2][2], w[2][3]), make_uint4(w[3][0], w[3][1], w[3][2], w[3][3]),
                                                amax[0], amax[1], tc.gs, off);
            o[0] = v.nibbles.x; o[1] = v.nibbles.y; o[2] = v.nibbles.z; o[3] = v.nibbles.w;
            codes = v.codes;
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const bool g = ((k + off) >> 1) & 1;
                o[k] = Q::template chunk_fast<false>(w[k], g ? s[1] : s[0], g ? rc[1] : rc[0], 0.f);
            }
        }
        reinterpret_cast<unsigned short*>(const_cast<void*>(J.scale))[gc0 >> 2] = (unsigned short)codes;   // two fp8 scales of this unit
        rotate_out<4, 1>(o, off);
        store_words<4>(J.out + (size_t)gc0 * 4, o);
    }
};

// ------------------------------------------------------------------------------------
// MXFP4-style quantize + pack: arithmetic in x's dtype T (scale has the same dtype, no global scale), one scale per unit.
//   unit = 4 chunks = 32 elements (needs group_size % 32 == 0)
// ------------------------------------------------------------------------------------
struct Fp4MxRaw {
    uint32_t s;
    uint32_t z;
};
template <class P, int ZK>
struct Fp4MxQuantPackOp {
    static constexpr int IN_BYTES = 16;
    static constexpr int GROUP = 4;
    using Raw = Fp4MxRaw;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc0) {
        Raw r;
        const uint32_t si = scale_index(J, gc0);
        r.s = __ldg(reinterpret_cast<const unsigned short*>(J.scale) + si);
        r.z = 0;
        if constexpr (ZK != FZ_NONE) r.z = __ldg(reinterpret_cast<const uint8_t*>(J.zp) + si);
        return r;
    }
    template <bool SLOW>
    __device__ static __forceinline__ uint32_t chunk(const uint32_t (&w)[4], const ScaleCtx& sc, uint32_t zp2, const Common& cm) {
        float f[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const uint32_t t = scaled_clamped2<P, ZK != FZ_NONE, SLOW>(w[j], sc, zp2, cm.qmin2, cm.qmax2);
            f[2 * j] = __fadd_rn(P::lo(t), 0.0f);
            f[2 * j + 1] = __fadd_rn(P::hi(t), 0.0f);
        }
        return f32x8_to_e2m1x8(f[0], f[1], f[2], f[3], f[4], f[5], f[6], f[7]);
    }
    __device__ static __forceinline__ void run(const Job& J, const Common& cm, const Raw& r, uint32_t gc0, const uint32_t (&w)[4][4], int off) {
        RawQP q; q.s = r.s; q.z = 0;
        const ScaleCtx sc = make_scale_ctx(scale_f32<P>(q));
        const uint32_t zp2 = (ZK != FZ_NONE) ? dup2<P>(fp4_zp_value<ZK>(r.z)) : 0u;
        uint32_t o[4];
        if (sc.slow) {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = chunk<true>(w[k], sc, zp2, cm);
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = chunk<false>(w[k], sc, zp2, cm);
        }
        rotate_out<4, 1>(o, off);
        store_words<4>(J.out + (size_t)gc0 * 4, o);
    }
};

// ------------------------------------------------------------------------------------
// unpack + dequantize: 8 nibbles (4 bytes) per chunk -> 8 x T; unit = 1 chunk, so that a thread's output is ONE 16-byte store
// (a 2-chunk unit writes 32 bytes per thread in two half-coalesced stores: twice the L1->L2 write sectors).
//   reference: unpack_fp4_from_uint8 -> (scale.to(T)) -> scale / global_scale -> x_q.to(scale.dtype) * scale -> .to(T)
//   (nvfp4/base.py:111-128, forward_helpers.py:559-570).  A product of an E2M1 value (2 significant bits) and a scale of
//   <= 24 bits is rounded once, to T, whichever of fp32 (global scale) or T the reference multiplies in.
// ------------------------------------------------------------------------------------
struct Fp4DqRaw {
    uint32_t s;
};

template <class P, int SK>
struct Fp4UnpackDequantOp {
    static constexpr int IN_BYTES = 4;
    static constexpr int GROUP = 1;
    // launch shape: the default ring, 4 stages x 3 CTAs per SM (stream.cuh: ring_shape)
    using Raw = Fp4DqRaw;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc0) {
        Raw r;
        const uint32_t si = scale_index(J, gc0);
        if constexpr (SK == FS_SAME) r.s = __ldg(reinterpret_cast<const unsigned short*>(J.scale) + si);
        else r.s = __ldg(reinterpret_cast<const uint8_t*>(J.scale) + si);
        return r;
    }
    using Tile = Fp4DqTile;
    __device__ static __forceinline__ Tile tile(const Job& J) {
        Tile t;
        t.has = J.aux != nullptr;
        t.gs = t.has ? __ldg(reinterpret_cast<const float*>(J.aux)) : 1.0f;
        t.rgs = __frcp_rn(t.gs);
        const float a = fabsf(t.gs);
        t.fast = a >= 8.673617379884035e-19f && a <= 1.152921504606847e18f;
        return t;
    }
    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw& r, uint32_t gc0, const uint32_t (&w)[1][1], int, const Tile& tc) {
        float s;
        if constexpr (SK == FS_SAME) { RawQP q; q.s = r.s; q.z = 0; s = scale_f32<P>(q); }
        else if constexpr (SK == FS_F8) s = e4m3_to_f32(r.s);                                   // .to(T) of an e4m3 value is exact
        else s = P::lo(P::pack((r.s & 0xffu) == 255u ? __int_as_float(0x7f800000) : ldexpf(1.0f, (int)(r.s & 0xffu) - 127), 0.f));  // 2^(e-127) -> bf16 -> T
        if (tc.has) {   // scale / global_scale, float32
            const float a = fabsf(s);
            if (tc.fast && a >= 9.094947017729282e-13f && a <= 16384.0f) s = recip_div(s, tc.gs, tc.rgs);
            else s = __fdiv_rn(s, tc.gs);
        }
        uint32_t o[4], h[4];
        e2m1x8_to_f16x8(w[0][0], h);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float a = __low2float(*reinterpret_cast<__half2*>(&h[j])), b = __high2float(*reinterpret_cast<__half2*>(&h[j]));
            o[j] = P::pack(__fmul_rn(a, s), __fmul_rn(b, s));
        }
        store_words<4>(J.out + (size_t)gc0 * 16, o);
    }
};

}  // namespace ctb

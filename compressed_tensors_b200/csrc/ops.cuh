// ops.cuh -- the per-unit functors plugged into the streaming pipelines (stream.cuh).
//
// Fast-path contract (checked on the host in dispatch.cu): x, scale and compute dtype are the
// same float dtype P; zero point absent (ZP=0) or int8 (ZP=1); scale index = chunk / dc
// (TENSOR, CHANNEL, GROUP with full rows of scales) or the 2-D form (row / rd) * srs + col_chunk / dc
// (BLOCK, one-row group scales), and dc % GROUP == 0 so that every unit has exactly one scale.
// The FP4 functors (two scales per unit, float32 arithmetic) are in fp4_ops.cuh.
#pragma once

#include "quant_core.cuh"
#include "stream.cuh"

namespace ctb {

struct F32 {
    static constexpr int DT = CT_F32;
};

enum QKind { QI_NARROW = 0, QI_WIDE = 1, QF8 = 2 };

template <class P> struct ElemBytes { static constexpr int v = 2; };
template <> struct ElemBytes<F32> { static constexpr int v = 4; };

// ------------------------------------------------------------------------------------
// raw scale / zero-point fetch (plain loads, nothing dependent) and its decoding
// ------------------------------------------------------------------------------------
struct RawQP {
    uint32_t s;   // 16-bit P: the scale's bit pattern (low half); F32: float bits
    int32_t z;    // int8 zero point (ZP == 1) / float8_e4m3fn zero-point byte (ZP == 2: what the FP8 presets register, quant_args.py zp_dtype)
};
struct NoRaw {};

// index of the scale / zero point of chunk gc (the whole unit shares it)
__device__ __forceinline__ uint32_t scale_index(const Job& J, uint32_t gc) {
    if (J.cpr.d == 0) return fd_div(gc, J.dc);                       // flat: TENSOR / CHANNEL / GROUP
    const uint32_t r = fd_div(gc, J.cpr);                             // 2-D: BLOCK, one-row group scales
    const uint32_t cc = gc - r * J.cpr.d;
    return fd_div(r, J.rd) * J.srs + fd_div(cc, J.dc);
}

template <class P, int ZP>
__device__ __forceinline__ RawQP load_qp(const void* scale, const void* zp, uint32_t si) {
    RawQP r;
    if constexpr (P::DT == CT_F32) r.s = __float_as_uint(__ldg(reinterpret_cast<const float*>(scale) + si));
    else r.s = __ldg(reinterpret_cast<const unsigned short*>(scale) + si);
    r.z = 0;
    if constexpr (ZP == 1) r.z = __ldg(reinterpret_cast<const int8_t*>(zp) + si);
    if constexpr (ZP == 2) r.z = __ldg(reinterpret_cast<const uint8_t*>(zp) + si);
    return r;
}
template <class P, int ZP>
__device__ __forceinline__ RawQP fetch_qp(const Job& J, uint32_t gc) { return load_qp<P, ZP>(J.scale, J.zp, scale_index(J, gc)); }
template <class P> __device__ __forceinline__ float scale_f32(const RawQP& r) {
    if constexpr (P::DT == CT_BF16) return __uint_as_float(r.s << 16);
    else if constexpr (P::DT == CT_F16) return __half2float(__ushort_as_half((unsigned short)r.s));
    else return __uint_as_float(r.s);
}
// scale in T duplicated in both halves (16-bit P) / float bits (F32)
template <class P> __device__ __forceinline__ uint32_t scale_t2(const RawQP& r) {
    if constexpr (P::DT == CT_F32) return r.s;
    else return r.s | (r.s << 16);
}
// zero_point.to(T) duplicated (16-bit P) / float bits (F32); int8 and e4m3 values are exact in every T
template <class P, int ZP> __device__ __forceinline__ uint32_t zp_t2(const RawQP& r) {
    if constexpr (ZP == 0) return 0u;
    else {
        const float z = (ZP == 2) ? e4m3_to_f32((uint32_t)r.z) : (float)r.z;
        if constexpr (P::DT == CT_F32) return __float_as_uint(z);
        else return dup2<P>(z);
    }
}

// fp32 compute dtype: clamped, un-rounded value (NAN_CLAMP as in clamp2)
template <int ZP, bool NAN_CLAMP = false>
__device__ __forceinline__ float scaled_clamped_f32(float x, float s, uint32_t zpbits, const Common& cm) {
    float t = __fdiv_rn(x, s);
    if (ZP) t = __fadd_rn(t, __uint_as_float(zpbits));
    if constexpr (NAN_CLAMP) return fmin_nan(fmax_nan(t, cm.qmin), cm.qmax);
    else return fminf(fmaxf(t, cm.qmin), cm.qmax);
}

// rounded (integer-valued, sign of zero preserved) pair in T
template <class P, bool WIDE>
__device__ __forceinline__ uint32_t round_int2(uint32_t t) {
    if constexpr (!WIDE) return round_keep_sign2<P>(t);
    else return P::pack(rintf(P::lo(t)), rintf(P::hi(t)));
}
// fp8-grid pair in T: T -> e4m3 (RNE) -> T
template <class P>
__device__ __forceinline__ uint32_t round_fp8_2(uint32_t t) {
    uint32_t h2 = e4m3x2_to_f16x2(f32x2_to_e4m3x2(P::lo(t), P::hi(t)));
    if constexpr (P::DT == CT_F16) return h2;
    else return P::pack(__low2float(*reinterpret_cast<__half2*>(&h2)), __high2float(*reinterpret_cast<__half2*>(&h2)));
}

// unsigned 4-bit codes of 4 rounded pairs -> one packed word (element 0 in bits 0-3)
__device__ __forceinline__ uint32_t nibbles_to_word(uint32_t t0, uint32_t t1, uint32_t t2, uint32_t t3) {
    uint32_t a = __byte_perm(t0, t1, 0x6420) & 0x0f0f0f0fu;
    uint32_t b = __byte_perm(t2, t3, 0x6420) & 0x0f0f0f0fu;
    a |= a >> 4;
    b |= b >> 4;
    return __byte_perm(a, b, 0x6420) ^ 0x88888888u;
}

template <int N>
__device__ __forceinline__ void store_words(uint8_t* p, const uint32_t (&o)[N]) {
    if constexpr (N == 1) stg_stream4(p, o[0]);
    else if constexpr (N == 2) stg_stream8(p, make_uint2(o[0], o[1]));
    else {
#pragma unroll
        for (int k = 0; k < N; k += 4) stg_stream16(p + 4 * k, make_uint4(o[k], o[k + 1], o[k + 2], o[k + 3]));
    }
}

// ------------------------------------------------------------------------------------
// QuantPack: x (GROUP x 8 x T) -> GROUP * BITS bytes of the int32 bitstream
//   replaces quantize(dtype=int8) + pack_to_int32 (pack_quantized/base.py:96-104)
//   GROUP = 4 with 4-bit codes: 32 elements -> one 16-byte store
// ------------------------------------------------------------------------------------
template <class P, int BITS, int ZP, int G>
struct QuantPackOp {
    static_assert(BITS == 4 || BITS == 8, "fast path packs 4- and 8-bit codes");
    static constexpr int TILE = (P::DT == CT_F32) ? TILE_CHUNKS : BIG_TILE_CHUNKS;   // engine.h: sig_tile_chunks
    static constexpr int PREF_STAGES = (P::DT == CT_F32) ? 4 : 3;
    static constexpr int PREF_CTAS = (P::DT == CT_F32) ? 3 : 2;
    static constexpr bool INPUT_EVICT_FIRST = false;   // reads 2-8x what it writes: see InputEvictFirst
    static constexpr int IN_BYTES = 8 * ElemBytes<P>::v;
    static constexpr int GROUP = G;
    static constexpr int OUT_WORDS = BITS / 4;   // per chunk
    using Raw = RawQP;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) { return fetch_qp<P, ZP>(J, gc); }

    template <bool SLOW>
    __device__ static __forceinline__ void chunk(const uint32_t (&w)[IN_BYTES / 4], const ScaleCtx& sc, uint32_t zp2, const Common& cm, uint32_t* o) {
        if constexpr (P::DT == CT_F32) {
            uint32_t lo = 0, hi = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const float t = scaled_clamped_f32<ZP>(__uint_as_float(w[k]), sc.s, zp2, cm);
                const uint32_t u = (uint32_t)(rint_magic_f32(t) + (1 << (BITS - 1))) & ((1u << BITS) - 1u);
                if (BITS == 4) lo |= u << (4 * k);
                else if (k < 4) lo |= u << (8 * k);
                else hi |= u << (8 * (k - 4));
            }
            o[0] = lo;
            if (BITS == 8) o[BITS / 4 - 1] = hi;
        } else if constexpr (BITS == 4) {
            uint32_t t[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) t[k] = round_magic2<P>(scaled_clamped2<P, ZP != 0, SLOW>(w[k], sc, zp2, cm.qmin2, cm.qmax2));
            o[0] = nibbles_to_word(t[0], t[1], t[2], t[3]);
        } else {
            uint32_t b[8];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t t = scaled_clamped2<P, ZP != 0, SLOW>(w[k], sc, zp2, cm.qmin2, cm.qmax2);
                b[2 * k] = (uint32_t)(rint_magic_f32(P::lo(t)) + 128) & 0xffu;
                b[2 * k + 1] = (uint32_t)(rint_magic_f32(P::hi(t)) + 128) & 0xffu;
            }
            o[0] = b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24);
            o[BITS / 4 - 1] = b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24);
        }
    }

    __device__ static __forceinline__ void run(const Job& J, const Common& cm, const Raw& r, uint32_t gc0, const uint32_t (&w)[G][IN_BYTES / 4], int off) {
        const ScaleCtx sc = make_scale_ctx(scale_f32<P>(r));
        const uint32_t zp2 = zp_t2<P, ZP>(r);
        uint32_t o[G * OUT_WORDS];
        if (sc.slow && P::DT != CT_F32) {
#pragma unroll
            for (int g = 0; g < G; ++g) chunk<true>(w[g], sc, zp2, cm, o + g * OUT_WORDS);
        } else {
#pragma unroll
            for (int g = 0; g < G; ++g) chunk<false>(w[g], sc, zp2, cm, o + g * OUT_WORDS);
        }
        rotate_out<G, OUT_WORDS>(o, off);
        store_words<G * OUT_WORDS>(J.out + (size_t)gc0 * (4 * OUT_WORDS), o);
    }
};

// ------------------------------------------------------------------------------------
// Quantize: x (GROUP x 8 x T) -> GROUP x 8 one-byte codes (int8 or float8_e4m3fn)
//   replaces quantize(dtype=args.pytorch_dtype()) (naive_quantized/base.py:79-86)
//   GROUP = 2: 16 elements -> one 16-byte store
// ------------------------------------------------------------------------------------
template <class P, int KIND, int ZP, int G>
struct QuantizeOp {
    static constexpr int TILE = (P::DT == CT_F32) ? TILE_CHUNKS : BIG_TILE_CHUNKS;   // engine.h: sig_tile_chunks
    static constexpr int PREF_STAGES = (P::DT == CT_F32) ? 4 : 3;
    static constexpr int PREF_CTAS = (P::DT == CT_F32) ? 3 : 2;
    static constexpr int IN_BYTES = 8 * ElemBytes<P>::v;
    static constexpr int GROUP = G;
    using Raw = RawQP;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) { return fetch_qp<P, ZP>(J, gc); }

    template <bool SLOW>
    __device__ static __forceinline__ void chunk(const uint32_t (&w)[IN_BYTES / 4], const ScaleCtx& sc, uint32_t zp2, const Common& cm, uint32_t* o) {
        uint32_t b[8];
        if constexpr (P::DT == CT_F32) {
#pragma unroll
            for (int k = 0; k < 8; k += 2) {
                const float t0 = scaled_clamped_f32<ZP>(__uint_as_float(w[k]), sc.s, zp2, cm);
                const float t1 = scaled_clamped_f32<ZP>(__uint_as_float(w[k + 1]), sc.s, zp2, cm);
                if constexpr (KIND == QF8) {
                    const uint32_t e = f32x2_to_e4m3x2(t0, t1);
                    b[k] = e & 0xffu;
                    b[k + 1] = e >> 8;
                } else {
                    b[k] = (uint32_t)rint_magic_f32(t0) & 0xffu;
                    b[k + 1] = (uint32_t)rint_magic_f32(t1) & 0xffu;
                }
            }
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t t = scaled_clamped2<P, ZP != 0, SLOW>(w[k], sc, zp2, cm.qmin2, cm.qmax2);
                if constexpr (KIND == QF8) {
                    const uint32_t e = f32x2_to_e4m3x2(P::lo(t), P::hi(t));
                    b[2 * k] = e & 0xffu;
                    b[2 * k + 1] = e >> 8;
                } else {
                    b[2 * k] = (uint32_t)rint_magic_f32(P::lo(t)) & 0xffu;
                    b[2 * k + 1] = (uint32_t)rint_magic_f32(P::hi(t)) & 0xffu;
                }
            }
        }
        o[0] = b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24);
        o[1] = b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24);
    }

    __device__ static __forceinline__ void run(const Job& J, const Common& cm, const Raw& r, uint32_t gc0, const uint32_t (&w)[G][IN_BYTES / 4], int off) {
        const ScaleCtx sc = make_scale_ctx(scale_f32<P>(r));
        const uint32_t zp2 = zp_t2<P, ZP>(r);
        uint32_t o[G * 2];
        if (sc.slow && P::DT != CT_F32) {
#pragma unroll
            for (int g = 0; g < G; ++g) chunk<true>(w[g], sc, zp2, cm, o + 2 * g);
        } else {
#pragma unroll
            for (int g = 0; g < G; ++g) chunk<false>(w[g], sc, zp2, cm, o + 2 * g);
        }
        rotate_out<G, 2>(o, off);
        store_words<G * 2>(J.out + (size_t)gc0 * 8, o);
    }
};

// ------------------------------------------------------------------------------------
// dequantization tail shared by Dequantize / UnpackDequant / FakeQuant
//   v = q.to(T); v -= zp.to(T); v *= scale     (forward_helpers.py:562-567)
// ------------------------------------------------------------------------------------
template <class P, int ZP>
__device__ __forceinline__ uint32_t dq_tail2(uint32_t v, uint32_t zp2, uint32_t s2) {
    if (ZP) v = sub2<P>(v, zp2);
    return mul2<P>(v, s2);
}
template <int ZP>
__device__ __forceinline__ float dq_tail_f32(float v, uint32_t zpbits, uint32_t sbits) {
    if (ZP) v = __fsub_rn(v, __uint_as_float(zpbits));
    return __fmul_rn(v, __uint_as_float(sbits));
}

// unsigned byte u (0..255) -> exact float u - bias, via the 2^23 exponent trick
__device__ __forceinline__ float ubyte_to_f32(uint32_t word, int k, float bias_plus_2p23) {
    // selector picks byte k of `word` as byte 0, bytes 1..3 from 0x4B000000
    const uint32_t bits = __byte_perm(word, 0x4B000000u, 0x7650u + (uint32_t)k);
    return __fsub_rn(__uint_as_float(bits), bias_plus_2p23);
}

template <class P>
__device__ __forceinline__ void store_out8(uint8_t* out, uint32_t gc, const uint32_t (&o)[8 * ElemBytes<P>::v / 4]) {
    store_words<8 * ElemBytes<P>::v / 4>(out + (size_t)gc * (8 * ElemBytes<P>::v), o);
}

// ------------------------------------------------------------------------------------
// Dequantize: 8 one-byte codes -> 8 x T       (naive_quantized/base.py:119-124)
// ------------------------------------------------------------------------------------
template <class P, int KIND /* QI_* = int8 codes, QF8 = e4m3 codes */, int ZP>
struct DequantizeOp {
    static constexpr int TILE = (P::DT == CT_F32) ? TILE_CHUNKS : BIG_TILE_CHUNKS;   // engine.h: sig_tile_chunks
    static constexpr int PREF_STAGES = (P::DT == CT_F32) ? 4 : 3;
    static constexpr int PREF_CTAS = (P::DT == CT_F32) ? 3 : 2;
    static constexpr int IN_BYTES = 8;
    static constexpr int GROUP = 1;
    using Raw = RawQP;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) { return fetch_qp<P, ZP>(J, gc); }

    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw& r, uint32_t gc, const uint32_t (&wg)[1][2], int) {
        const uint32_t(&w)[2] = wg[0];
        const uint32_t s2 = scale_t2<P>(r), zp2 = zp_t2<P, ZP>(r);
        float f[8];
        if constexpr (KIND == QF8) {
            uint32_t h[4];
            e4m3x4_to_f16x4(w[0], h[0], h[1]);
            e4m3x4_to_f16x4(w[1], h[2], h[3]);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                f[2 * k] = __low2float(*reinterpret_cast<__half2*>(&h[k]));
                f[2 * k + 1] = __high2float(*reinterpret_cast<__half2*>(&h[k]));
            }
        } else {
            const uint32_t w0 = w[0] ^ 0x80808080u, w1 = w[1] ^ 0x80808080u;  // int8 -> offset-128 unsigned
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                f[k] = ubyte_to_f32(w0, k, 8388608.0f + 128.0f);
                f[4 + k] = ubyte_to_f32(w1, k, 8388608.0f + 128.0f);
            }
        }
        uint32_t o[8 * ElemBytes<P>::v / 4];
        if constexpr (P::DT == CT_F32) {
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = __float_as_uint(dq_tail_f32<ZP>(f[k], zp2, s2));
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = dq_tail2<P, ZP>(P::pack(f[2 * k], f[2 * k + 1]), zp2, s2);
        }
        store_out8<P>(J.out, gc, o);
    }
};

// ------------------------------------------------------------------------------------
// Dequantize with a float32 scale and a 16-bit output: (q.to(float32) * scale).to(T) -- two roundings, fp32 then T
//   (the FP8 block checkpoints of entrypoints/convert/converters/fp8block_dequantizer.py:111-158: fp8 weight, float32
//   weight_scale_inv per 128x128 block, bf16 result; also dequantize() with a float32 scale on the group path)
// ------------------------------------------------------------------------------------
template <class P>
struct DequantF32ScaleOp {
    static constexpr int TILE = (P::DT == CT_F32) ? TILE_CHUNKS : BIG_TILE_CHUNKS;   // engine.h: sig_tile_chunks
    static constexpr int PREF_STAGES = (P::DT == CT_F32) ? 4 : 3;
    static constexpr int PREF_CTAS = (P::DT == CT_F32) ? 3 : 2;
    static constexpr int IN_BYTES = 8;
    static constexpr int GROUP = 1;
    struct Raw { uint32_t s; };
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) {
        Raw r;
        r.s = __float_as_uint(__ldg(reinterpret_cast<const float*>(J.scale) + scale_index(J, gc)));
        return r;
    }
    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw& r, uint32_t gc, const uint32_t (&wg)[1][2], int) {
        const float s = __uint_as_float(r.s);
        uint32_t o[4], h[4];
        e4m3x4_to_f16x4(wg[0][0], h[0], h[1]);
        e4m3x4_to_f16x4(wg[0][1], h[2], h[3]);
#pragma unroll
        for (int k = 0; k < 4; ++k)
            o[k] = P::pack(__fmul_rn(__low2float(*reinterpret_cast<__half2*>(&h[k])), s), __fmul_rn(__high2float(*reinterpret_cast<__half2*>(&h[k])), s));
        store_words<4>(J.out + (size_t)gc * 16, o);
    }
};

// ------------------------------------------------------------------------------------
// UnpackDequant: BITS*8 bits of the int32 bitstream -> 8 x T
//   replaces unpack_from_int32 + dequantize (pack_quantized/base.py:159-166)
// ------------------------------------------------------------------------------------
template <class P, int BITS, int ZP>
struct UnpackDequantOp {
    static_assert(BITS == 4 || BITS == 8, "fast path unpacks 4- and 8-bit codes");
    static constexpr int TILE = (P::DT == CT_F32) ? TILE_CHUNKS : BIG_TILE_CHUNKS;   // engine.h: sig_tile_chunks
    static constexpr int PREF_STAGES = (P::DT == CT_F32) ? 4 : 3;
    static constexpr int PREF_CTAS = (P::DT == CT_F32) ? 3 : 2;
    static constexpr int IN_BYTES = BITS;
    static constexpr int GROUP = 1;
    using Raw = RawQP;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) { return fetch_qp<P, ZP>(J, gc); }

    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw& r, uint32_t gc, const uint32_t (&wg)[1][BITS / 4], int) {
        const uint32_t(&w)[BITS / 4] = wg[0];
        const uint32_t s2 = scale_t2<P>(r), zp2 = zp_t2<P, ZP>(r);
        uint32_t o[8 * ElemBytes<P>::v / 4];
        if constexpr (BITS == 4 && P::DT != CT_F32) {
            // nibble u = n + 8 in [0, 15]; (EXP | u) is the T value EXPVAL + u exactly; subtract EXPVAL + 8
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t lo = (w[0] >> (8 * k)) & 0xfu;
                const uint32_t hi = (w[0] >> (8 * k + 4)) & 0xfu;
                const uint32_t p = P::ONE_TWENTY_EIGHT2 | lo | (hi << 16);
                o[k] = dq_tail2<P, ZP>(sub2<P>(p, P::OFF8_2), zp2, s2);
            }
        } else {
            float f[8];
            if constexpr (BITS == 4) {
#pragma unroll
                for (int k = 0; k < 8; ++k) f[k] = (float)((int)((w[0] >> (4 * k)) & 0xfu) - 8);
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    f[k] = ubyte_to_f32(w[0], k, 8388608.0f + 128.0f);
                    f[4 + k] = ubyte_to_f32(w[BITS / 4 - 1], k, 8388608.0f + 128.0f);
                }
            }
            if constexpr (P::DT == CT_F32) {
#pragma unroll
                for (int k = 0; k < 8; ++k) o[k] = __float_as_uint(dq_tail_f32<ZP>(f[k], zp2, s2));
            } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) o[k] = dq_tail2<P, ZP>(P::pack(f[2 * k], f[2 * k + 1]), zp2, s2);
            }
        }
        store_out8<P>(J.out, gc, o);
    }
};

// ------------------------------------------------------------------------------------
// FakeQuant: x (8 x T) -> quantize -> dequantize -> 8 x T   (forward_helpers.py:180-215)
//   a NaN input or scale gives NaN, as in the reference: the clamp propagates it
// ------------------------------------------------------------------------------------
template <class P, int KIND, int ZP>
struct FakeQuantOp {
    static constexpr int IN_BYTES = 8 * ElemBytes<P>::v;
    static constexpr int GROUP = 1;
    using Raw = RawQP;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) { return fetch_qp<P, ZP>(J, gc); }

    template <bool SLOW>
    __device__ static __forceinline__ void body(const Common& cm, const ScaleCtx& sc, uint32_t s2, uint32_t zp2,
                                                const uint32_t (&w)[IN_BYTES / 4], uint32_t (&o)[IN_BYTES / 4]) {
        if constexpr (P::DT == CT_F32) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                float t = scaled_clamped_f32<ZP, true>(__uint_as_float(w[k]), sc.s, zp2, cm);
                if constexpr (KIND == QF8) t = e4m3_to_f32(f32_to_e4m3_byte(t));
                else t = rintf(t);
                o[k] = __float_as_uint(dq_tail_f32<ZP>(t, zp2, s2));
            }
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                uint32_t t = scaled_clamped2<P, ZP != 0, SLOW, true>(w[k], sc, zp2, cm.qmin2, cm.qmax2);
                if constexpr (KIND == QF8) t = round_fp8_2<P>(t);
                else t = round_int2<P, KIND == QI_WIDE>(t);
                o[k] = dq_tail2<P, ZP>(t, zp2, s2);
            }
        }
    }
    // one chunk w -> o with the raw scale / zero point r; the streaming run() below and the strided kernel of fake_heads.cu share it
    __device__ static __forceinline__ void apply(const Common& cm, const Raw& r, const uint32_t (&w)[IN_BYTES / 4], uint32_t (&o)[IN_BYTES / 4]) {
        const ScaleCtx sc = make_scale_ctx(scale_f32<P>(r));
        const uint32_t s2 = scale_t2<P>(r), zp2 = zp_t2<P, ZP>(r);
        if (sc.slow && P::DT != CT_F32) body<true>(cm, sc, s2, zp2, w, o);
        else body<false>(cm, sc, s2, zp2, w, o);
    }
    __device__ static __forceinline__ void run(const Job& J, const Common& cm, const Raw& r, uint32_t gc, const uint32_t (&wg)[1][IN_BYTES / 4], int) {
        uint32_t o[IN_BYTES / 4];
        apply(cm, r, wg[0], o);
        store_out8<P>(J.out, gc, o);
    }
};

// ------------------------------------------------------------------------------------
// standalone bit packing of int8 codes (compressors/pack_quantized/helpers.py:20-180), 4 and 8 bits.
// For these two ops a "chunk" is 16 codes (the host passes n_chunks = numel / 16).
//   pack   4-bit: GROUP = 2 -> 32 codes (2 x 16 B) in, 16 B out;  8-bit: 16 B in, 16 B out
//   unpack 4-bit: 8 B in -> 16 codes = 16 B out;                  8-bit: 16 B in, 16 B out
// ------------------------------------------------------------------------------------
// word = sum_j (v_j + 8) << 4j  (mod 2^32), the reference's scatter_add semantics, which also fixes
// the result for out-of-range int8 inputs.  dp4a forms v0 + 16*v1 etc.
__device__ __forceinline__ uint32_t pack8_codes(uint32_t w0, uint32_t w1) {
    const int s01 = __dp4a((int)w0, 0x00001001, 0);   // weights (1, 16, 0, 0)
    const int s23 = __dp4a((int)w0, 0x10010000, 0);   // weights (0, 0, 1, 16)
    const int s45 = __dp4a((int)w1, 0x00001001, 0);
    const int s67 = __dp4a((int)w1, 0x10010000, 0);
    return (uint32_t)s01 + ((uint32_t)s23 << 8) + ((uint32_t)s45 << 16) + ((uint32_t)s67 << 24) + 0x88888888u;
}
template <int BITS>
struct PackOp {
    static constexpr int IN_BYTES = 16;
    static constexpr int GROUP = (BITS == 4) ? 2 : 1;
    using Raw = NoRaw;
    __device__ static __forceinline__ Raw prefetch(const Job&, uint32_t) { return {}; }
    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw&, uint32_t gc0, const uint32_t (&w)[GROUP][4], int off) {
        if constexpr (BITS == 8) {
            uint32_t o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = w[0][k] ^ 0x80808080u;
            store_words<4>(J.out + (size_t)gc0 * 16, o);
        } else {
            uint32_t o[4];
#pragma unroll
            for (int g = 0; g < 2; ++g) {
                o[2 * g] = pack8_codes(w[g][0], w[g][1]);
                o[2 * g + 1] = pack8_codes(w[g][2], w[g][3]);
            }
            rotate_out<2, 2>(o, off);
            store_words<4>(J.out + (size_t)gc0 * 8, o);
        }
    }
};
// 8 unsigned nibbles of `word` -> 8 int8 codes (value - 8) in two words
__device__ __forceinline__ void unpack8_codes(uint32_t word, uint32_t& a, uint32_t& b) {
    const uint32_t lo = word & 0x0f0f0f0fu, hi = (word >> 4) & 0x0f0f0f0fu;
    a = __byte_perm(lo, hi, 0x5140);   // elements 0..3 (codes 0..15 per byte)
    b = __byte_perm(lo, hi, 0x7362);   // elements 4..7
    // code - 8 per byte without inter-byte borrows: keep low 3 bits, set 0xF8 when bit 3 is clear
    a = (a & 0x07070707u) | ((~a & 0x08080808u) * 31u);
    b = (b & 0x07070707u) | ((~b & 0x08080808u) * 31u);
}
template <int BITS>
struct UnpackOp {
    static constexpr int IN_BYTES = 2 * BITS;   // 16 codes
    static constexpr int GROUP = 1;
    using Raw = NoRaw;
    __device__ static __forceinline__ Raw prefetch(const Job&, uint32_t) { return {}; }
    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw&, uint32_t gc0, const uint32_t (&w)[1][IN_BYTES / 4], int) {
        uint32_t o[4];
        if constexpr (BITS == 8) {
#pragma unroll
            for (int k = 0; k < 4; ++k) o[k] = w[0][k] ^ 0x80808080u;
        } else {
            unpack8_codes(w[0][0], o[0], o[1]);
            unpack8_codes(w[0][IN_BYTES / 4 - 1], o[2], o[3]);
        }
        store_words<4>(J.out + (size_t)gc0 * 16, o);
    }
};

}  // namespace ctb

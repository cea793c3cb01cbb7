// fast_sparse24q.cu -- BASELINE config 4: "Sparse24BitMask + int4" in one pass each way.
//
//   compress  : dense x [R, C] (bf16 / fp16), group / channel / tensor scales (+ int8 zero points)
//                 -> per quad keep the 2 of largest |x| (ties: lower column; sparse.cu's rule)
//                 -> quantize the KEPT values with the qparams of their original column (forward_helpers.py:523-546)
//                 -> weight_packed int32 [R, C/16]  = pack_to_int32(kept codes [R, C/2], 4)  (pack_quantized/helpers.py:20-101)
//                    bitmask uint8 [R, C/8]         = pack_bitmasks(mask)                    (utils/helpers.py:306-317)
//   decompress: the inverse -- codes scattered back to their columns, dequantized (forward_helpers.py:549-572), dropped columns = +0
//
// This is the composition  Sparse24BitMaskCompressor . PackedQuantizationCompressor  restated from the pieces that survive in the
// reference (the quantize arithmetic, the int32 bitstream and the mask bit order are golden-pinned; the 2:4 selection rule and the
// composition itself are "parity unpinned", SURVEY.md 8 a12 / a14).  Algorithmic traffic with g128 bf16: 2 + 0.25 + 0.125 + 2/128
// = 2.39 B per dense element (SURVEY 8(d)); neither the dense int8 codes, the kept bf16 values nor a byte mask ever touch HBM.
//
// Both directions are functors on the streaming pipelines of stream.cuh (TMA ring + dynamic tile claims):
//   Sparse24QuantPackOp    chunk = 8 dense elements (16 B in), unit = 4 chunks: 8 quads -> 8 B of nibbles + 4 mask bytes
//   Sparse24UnpackDequantOp chunk = unit = 16 dense elements (4 B of nibbles in, streamed through the ring; the 2 mask bytes come with
//                           the scale prefetch): 32 B out as one 256-bit store
// The second tensor (the bitmask) travels in Job::aux.
#include "engine.h"
#include "ops.cuh"
#include "sparse_common.cuh"

namespace ctb {

template <class P, int ZP>
struct Sparse24QuantPackOp {
    static constexpr int IN_BYTES = 16;
    static constexpr int GROUP = 4;
    using Raw = RawQP;
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) { return fetch_qp<P, ZP>(J, gc); }

    // one chunk = 2 quads: mask byte + 4 nibbles (16 bits of the packed stream)
    template <bool SLOW>
    __device__ static __forceinline__ void chunk(const uint32_t (&w)[4], const ScaleCtx& sc, uint32_t zp2, const Common& cm, uint32_t& hw, uint32_t& mb) {
        uint32_t p0, p1;
        const uint32_t k0 = quad_select16(w[0], w[1], p0);
        const uint32_t k1 = quad_select16(w[2], w[3], p1);
        mb = k0 | (k1 << 4);
        const uint32_t t0 = round_magic2<P>(scaled_clamped2<P, ZP != 0, SLOW>(p0, sc, zp2, cm.qmin2, cm.qmax2));
        const uint32_t t1 = round_magic2<P>(scaled_clamped2<P, ZP != 0, SLOW>(p1, sc, zp2, cm.qmin2, cm.qmax2));
        uint32_t a = __byte_perm(t0, t1, 0x6420) & 0x0f0f0f0fu;     // the four codes' low nibbles, one per byte
        a |= a >> 4;
        hw = __byte_perm(a, 0u, 0x4420);                             // (n0 | n1 << 4) | (n2 | n3 << 4) << 8
    }

    __device__ static __forceinline__ void run(const Job& J, const Common& cm, const Raw& r, uint32_t gc0, const uint32_t (&w)[4][4], int off) {
        const ScaleCtx sc = make_scale_ctx(scale_f32<P>(r));
        const uint32_t zp2 = zp_t2<P, ZP>(r);
        uint32_t hw[4], mb[4];
        if (sc.slow) {
#pragma unroll
            for (int g = 0; g < 4; ++g) chunk<true>(w[g], sc, zp2, cm, hw[g], mb[g]);
        } else {
#pragma unroll
            for (int g = 0; g < 4; ++g) chunk<false>(w[g], sc, zp2, cm, hw[g], mb[g]);
        }
        rotate_out<4, 1>(hw, off);
        rotate_out<4, 1>(mb, off);
        const uint32_t w0 = (hw[0] | (hw[1] << 16)) ^ 0x88888888u;   // + 8: two's complement nibble -> offset-binary (helpers.py:66-68)
        const uint32_t w1 = (hw[2] | (hw[3] << 16)) ^ 0x88888888u;
        stg_stream8(J.out + (size_t)gc0 * 2, make_uint2(w0, w1));
        stg_stream4(reinterpret_cast<uint8_t*>(const_cast<void*>(J.aux)) + gc0, mb[0] | (mb[1] << 8) | (mb[2] << 16) | (mb[3] << 24));
    }
};

template <class P, int ZP>
struct Sparse24UnpackDequantOp {
    static constexpr int IN_BYTES = 4;    // per chunk of 16 dense elements: 8 kept codes
    static constexpr int GROUP = 1;       // one thread = one chunk = 32 contiguous output bytes (two 16-byte stores)
    struct Raw {
        RawQP qp;
        uint32_t mask;   // the chunk's 2 mask bytes
    };
    __device__ static __forceinline__ Raw prefetch(const Job& J, uint32_t gc) {
        Raw r;
        r.qp = fetch_qp<P, ZP>(J, gc);
        r.mask = __ldg(reinterpret_cast<const unsigned short*>(J.aux) + gc);
        return r;
    }
    // kept pair v = {first kept, second kept} of a quad, b = its 4 mask bits -> the quad's 4 elements in two words.
    // element e takes the first kept value if it is the lowest set bit, the second if any lower bit is set, zero if its bit is clear
    __device__ static __forceinline__ void scatter_quad(uint32_t v, uint32_t b, uint32_t& o01, uint32_t& o23) {
        // byte selectors per element: first kept = bytes (0,1) = 0x10, second = (2,3) = 0x32, zero = (4,4) = 0x44 (second prmt operand = 0):
        //   sel_e = 0x44 - 0x34 * bit_e + 0x22 * (bit_e and a lower bit is set)
        // all four at once: the bits that have a lower set bit are b & (b - 1); a multiply by 1 + 2^7 + 2^14 + 2^21 and a mask move bit e
        // of a nibble to byte e (no two partial products meet, so nothing carries)
        const uint32_t later = b & (b - 1u);
        const uint32_t B = (b * 0x00204081u) & 0x01010101u, L = (later * 0x00204081u) & 0x01010101u;
        const uint32_t S = 0x44444444u - B * 0x34u + L * 0x22u;
        asm("prmt.b32 %0, %1, %2, %3;" : "=r"(o01) : "r"(v), "r"(0u), "r"(S));          // PRMT reads the selector's low 16 bits
        asm("prmt.b32 %0, %1, %2, %3;" : "=r"(o23) : "r"(v), "r"(0u), "r"(S >> 16));
    }
    __device__ static __forceinline__ void run(const Job& J, const Common&, const Raw& r, uint32_t gc, const uint32_t (&w)[1][1], int) {
        const uint32_t s2 = scale_t2<P>(r.qp), zp2 = zp_t2<P, ZP>(r.qp);
        const uint32_t word = w[0][0];
        uint32_t o[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            // nibble u = code + 8 in [0, 15]; (EXP | u) is the T value EXPVAL + u exactly; subtract EXPVAL + 8 (UnpackDequantOp's trick)
            const uint32_t lo = (word >> (8 * q)) & 0xfu, hi = (word >> (8 * q + 4)) & 0xfu;
            const uint32_t v = dq_tail2<P, ZP>(sub2<P>(P::ONE_TWENTY_EIGHT2 | lo | (hi << 16), P::OFF8_2), zp2, s2);
            scatter_quad(v, (r.mask >> (4 * q)) & 0xfu, o[2 * q], o[2 * q + 1]);
        }
        stg_stream32(J.out + (size_t)gc * 32, o);
    }
};

template <class P>
static StreamKernel s24_p(bool compress, int zp_kind) {
    if (compress && zp_kind == 0) return stream_kernel<Sparse24QuantPackOp<P, 0>>();
    if (compress && zp_kind == 1) return stream_kernel<Sparse24QuantPackOp<P, 1>>();
    if (!compress && zp_kind == 0) return stream_kernel<Sparse24UnpackDequantOp<P, 0>>();
    if (!compress && zp_kind == 1) return stream_kernel<Sparse24UnpackDequantOp<P, 1>>();
    return {};
}

StreamKernel sparse24q_kernel(bool compress, int p_dt, int zp_kind) {
    if (p_dt == CT_BF16) return s24_p<BF16>(compress, zp_kind);
    if (p_dt == CT_F16) return s24_p<F16>(compress, zp_kind);
    return {};
}

}  // namespace ctb

// fast_pack.cu -- streaming instantiations: fused quantize+pack, fused unpack+dequantize,
// standalone int8 <-> int32 bit packing.
#include "engine.h"
#include "ops.cuh"

namespace ctb {

// unit sizes: 4-bit codes -> 4 chunks (32 elements -> 16 B out); 8-bit codes -> 2 chunks; fp32 -> 1 chunk
template <class P, int BITS, int ZP>
static StreamKernel quantpack_u(int max_unit) {
    constexpr int GMAX = (BITS == 4) ? 4 : 2;
    if constexpr (P::DT != CT_F32) {
        if (max_unit >= GMAX) return stream_kernel<QuantPackOp<P, BITS, ZP, GMAX>>();
    }
    return stream_kernel<QuantPackOp<P, BITS, ZP, 1>>();
}
template <class P>
static StreamKernel quantpack_p(int bits, int zp_kind, int max_unit) {
    if (bits == 4 && zp_kind == 0) return quantpack_u<P, 4, 0>(max_unit);
    if (bits == 4 && zp_kind == 1) return quantpack_u<P, 4, 1>(max_unit);
    if (bits == 8 && zp_kind == 0) return quantpack_u<P, 8, 0>(max_unit);
    if (bits == 8 && zp_kind == 1) return quantpack_u<P, 8, 1>(max_unit);
    return {};
}
StreamKernel quantpack_kernel(int p_dt, int bits, int zp_kind, int max_unit) {
    switch (p_dt) {
    case CT_BF16: return quantpack_p<BF16>(bits, zp_kind, max_unit);
    case CT_F16: return quantpack_p<F16>(bits, zp_kind, max_unit);
    case CT_F32: return quantpack_p<F32>(bits, zp_kind, max_unit);
    }
    return {};
}

template <class P>
static StreamKernel unpackdeq_p(int bits, int zp_kind) {
    if (bits == 4 && zp_kind == 0) return stream_kernel<UnpackDequantOp<P, 4, 0>>();
    if (bits == 4 && zp_kind == 1) return stream_kernel<UnpackDequantOp<P, 4, 1>>();
    if (bits == 8 && zp_kind == 0) return stream_kernel<UnpackDequantOp<P, 8, 0>>();
    if (bits == 8 && zp_kind == 1) return stream_kernel<UnpackDequantOp<P, 8, 1>>();
    return {};
}
StreamKernel unpackdeq_kernel(int p_dt, int bits, int zp_kind) {
    switch (p_dt) {
    case CT_BF16: return unpackdeq_p<BF16>(bits, zp_kind);
    case CT_F16: return unpackdeq_p<F16>(bits, zp_kind);
    case CT_F32: return unpackdeq_p<F32>(bits, zp_kind);
    }
    return {};
}

StreamKernel bits_kernel(bool pack, int bits) {
    if (pack && bits == 4) return stream_kernel<PackOp<4>>();
    if (pack && bits == 8) return stream_kernel<PackOp<8>>();
    if (!pack && bits == 4) return stream_kernel<UnpackOp<4>>();
    if (!pack && bits == 8) return stream_kernel<UnpackOp<8>>();
    return {};
}

}  // namespace ctb

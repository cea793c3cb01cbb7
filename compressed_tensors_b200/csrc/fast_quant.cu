// fast_quant.cu -- streaming instantiations: quantize (to int8 / float8_e4m3fn) and dequantize.
#include "engine.h"
#include "ops.cuh"

namespace ctb {

// the NARROW / WIDE integer kinds share one kernel here
template <class P, int KIND, int ZP>
static StreamKernel quant_u(int max_unit) {
    if constexpr (P::DT != CT_F32) {
        if (max_unit >= 2) return stream_kernel<QuantizeOp<P, KIND, ZP, 2>>();
    }
    return stream_kernel<QuantizeOp<P, KIND, ZP, 1>>();
}
template <class P>
static StreamKernel quant_p(bool fp8, int zp_kind, int max_unit) {
    if (fp8 && zp_kind == 0) return quant_u<P, QF8, 0>(max_unit);
    if (fp8 && zp_kind == 1) return quant_u<P, QF8, 1>(max_unit);
    if (fp8 && zp_kind == 2) return quant_u<P, QF8, 2>(max_unit);   // float8_e4m3fn zero point (the FP8 presets)
    if (!fp8 && zp_kind == 0) return quant_u<P, QI_WIDE, 0>(max_unit);
    if (!fp8 && zp_kind == 1) return quant_u<P, QI_WIDE, 1>(max_unit);
    return {};
}
StreamKernel quant_kernel(int p_dt, bool fp8, int zp_kind, int max_unit) {
    switch (p_dt) {
    case CT_BF16: return quant_p<BF16>(fp8, zp_kind, max_unit);
    case CT_F16: return quant_p<F16>(fp8, zp_kind, max_unit);
    case CT_F32: return quant_p<F32>(fp8, zp_kind, max_unit);
    }
    return {};
}

template <class P>
static StreamKernel dequant_p(bool fp8, int zp_kind, bool f32_scale) {
    if (f32_scale) {
        if constexpr (P::DT != CT_F32) {
            if (fp8 && zp_kind == 0) return stream_kernel<DequantF32ScaleOp<P>>();
        }
        return {};
    }
    if (fp8 && zp_kind == 0) return stream_kernel<DequantizeOp<P, QF8, 0>>();
    if (fp8 && zp_kind == 1) return stream_kernel<DequantizeOp<P, QF8, 1>>();
    if (fp8 && zp_kind == 2) return stream_kernel<DequantizeOp<P, QF8, 2>>();
    if (!fp8 && zp_kind == 0) return stream_kernel<DequantizeOp<P, QI_WIDE, 0>>();
    if (!fp8 && zp_kind == 1) return stream_kernel<DequantizeOp<P, QI_WIDE, 1>>();
    return {};
}
StreamKernel dequant_kernel(int p_dt, bool fp8, int zp_kind, bool f32_scale) {
    switch (p_dt) {
    case CT_BF16: return dequant_p<BF16>(fp8, zp_kind, f32_scale);
    case CT_F16: return dequant_p<F16>(fp8, zp_kind, f32_scale);
    case CT_F32: return dequant_p<F32>(fp8, zp_kind, f32_scale);
    }
    return {};
}

}  // namespace ctb

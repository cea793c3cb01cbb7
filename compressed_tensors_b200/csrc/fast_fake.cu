// fast_fake.cu -- streaming instantiations: fused quantize->dequantize (fake_quantize).
#include "engine.h"
#include "ops.cuh"

namespace ctb {

template <class P>
static StreamKernel fake_p(int kind, int zp_kind) {
    if (kind == QF8 && zp_kind == 0) return stream_kernel<FakeQuantOp<P, QF8, 0>>();
    if (kind == QF8 && zp_kind == 1) return stream_kernel<FakeQuantOp<P, QF8, 1>>();
    if (kind == QF8 && zp_kind == 2) return stream_kernel<FakeQuantOp<P, QF8, 2>>();
    if (kind == QI_WIDE && zp_kind == 0) return stream_kernel<FakeQuantOp<P, QI_WIDE, 0>>();
    if (kind == QI_WIDE && zp_kind == 1) return stream_kernel<FakeQuantOp<P, QI_WIDE, 1>>();
    if constexpr (P::DT != CT_F32) {   // fp32 has no packed-magic rounding: fake_kind never picks NARROW for it
        if (kind == QI_NARROW && zp_kind == 0) return stream_kernel<FakeQuantOp<P, QI_NARROW, 0>>();
        if (kind == QI_NARROW && zp_kind == 1) return stream_kernel<FakeQuantOp<P, QI_NARROW, 1>>();
    }
    return {};
}

StreamKernel fake_kernel(int p_dt, int qtype, int bits, int zp_kind) {
    const int kind = fake_kind(p_dt, qtype, bits);
    switch (p_dt) {
    case CT_BF16: return fake_p<BF16>(kind, zp_kind);
    case CT_F16: return fake_p<F16>(kind, zp_kind);
    case CT_F32: return fake_p<F32>(kind, zp_kind);
    }
    return {};
}

}  // namespace ctb

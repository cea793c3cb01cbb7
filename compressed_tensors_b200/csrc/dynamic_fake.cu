// dynamic_fake.cu -- ct_dynamic_fake_quantize: dynamic activation quantization in one pass.  The observer of
// compute_dynamic_scales_and_zp (quantization/utils/helpers.py:140-195: min / max over the strategy's reduction dims, then
// calculate_qparams) fused with fake_quantize (forward.py:148-181), which forward_quantize runs on every forward of a quantized Linear
// whose input activations are dynamic.  The reference reads the activation three times (amin, amax, fake_quantize) and runs a dozen
// qparam-sized kernels in between; here it crosses HBM once in and once out, with the qparams written beside it.
//   TOKEN                 one CTA per row (everything after the first two dims), the row held in registers (up to 32768 columns)
//   GROUP / TENSOR_GROUP  groups of 16..128 elements inside a warp: 2..16 lanes of one 16-byte chunk each combine min / max by shuffles
//   TENSOR                ct_observe_tensor's grid-wide observer, then ct_fake_quantize on the device-resident scale (two launches)
// The qparams come from observe_core.cuh (the rule every device observer shares).  The per-element arithmetic is the one
// ct_fake_quantize runs on the same scale and zero-point tensors: FakeQuantOp where its dispatch (dispatch.cu, plan_one) takes the
// streaming kernel, the generic kernel's composition (generic.cuh, quant_at / dequant_at) where it takes that one (FP4, a global scale,
// a uint8 zero point).  So the fused result equals the two-step path bit for bit.
#include <cstring>

#include "engine.h"
#include "observe_core.cuh"
#include "ops.cuh"

namespace ctb {

enum ScaleRule { SR_PLAIN = 0, SR_FP8 = 1, SR_MX = 2 };   // args.scale_dtype: none, float8_e4m3fn (NVFP4), uint8 (MX, group 32)
constexpr int K_SCALAR = 3;                                // element rule after QKind: the generic kernel's composition
constexpr int TOKEN_MAX_COLS = 32768;
constexpr int GROUP_UNITS = 4;                             // chunks per thread of the group kernel (one per warp-wide span of 32 chunks)

struct DynParams {
    Common cm;
    int srule;
    int asym;
    int scale_f32;      // scale_out holds float32 (a global scale promotes the scale), else x's dtype
    int zp_i8;          // zero point int8 (else float8_e4m3fn / uint8, whose zero is byte 0)
    int x_dt, cd, se_dt, qtype;   // K_SCALAR: x dtype, compute dtype and effective scale dtype of the matching fake_quantize
    const float* gs;    // global scale (one float32 on the device) or nullptr
};

// ------------------------------------------------------------------------------------
// TOKEN: one CTA of NT threads per row, up to NT * MAXU chunks of 8 elements
// ------------------------------------------------------------------------------------
template <class P, int KIND, int ZP, int ASYM, int NT, int MAXU>
__global__ void __launch_bounds__(NT) dyn_token_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, void* __restrict__ scale_out,
                                                       uint8_t* __restrict__ zp_out, int units /* cols / 8 */, const __grid_constant__ Common cm) {
    constexpr int NW = NT / 32;
    __shared__ uint32_t red[2][NW];
    __shared__ float qp[2];
    const int64_t r = blockIdx.x;
    const uint4* row = x + r * units;
    uint4 v[MAXU];
#pragma unroll
    for (int u = 0; u < MAXU; ++u) {
        const int i = u * NT + threadIdx.x;
        v[u] = (i < units) ? ldg_stream16(row + i) : make_uint4(0, 0, 0, 0);   // 0 is neutral: the observer clamps min <= 0 <= max
    }
    uint32_t mn2 = v[0].x, mx2 = v[0].x;
#pragma unroll
    for (int u = 0; u < MAXU; ++u) obs_chunk_minmax<P>(v[u], mn2, mx2);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        mn2 = min2_nan<P>(mn2, __shfl_xor_sync(0xffffffffu, mn2, d));
        mx2 = max2_nan<P>(mx2, __shfl_xor_sync(0xffffffffu, mx2, d));
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = mn2; red[1][threadIdx.x >> 5] = mx2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < NW; ++w) { mn2 = min2_nan<P>(mn2, red[0][w]); mx2 = max2_nan<P>(mx2, red[1][w]); }
        float lo, hi;
        obs_range2<P>(mn2, mx2, lo, hi);
        float zq;
        const float s = obs_scale_zp<P::DT>(lo, hi, ASYM, cm.qmin, cm.qmax, zq);
        reinterpret_cast<unsigned short*>(scale_out)[r] = (unsigned short)P::from_float1(s);
        zp_out[r] = (uint8_t)(int8_t)(int)zq;                          // int8 zero point, or the byte of an fp8 zero
        qp[0] = s; qp[1] = zq;
    }
    __syncthreads();
    RawQP q;
    q.s = P::from_float1(qp[0]);
    q.z = (int)qp[1];
    uint4* orow = out + r * units;
#pragma unroll
    for (int u = 0; u < MAXU; ++u) {
        const int i = u * NT + threadIdx.x;
        if (i >= units) continue;
        const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
        uint32_t o[4];
        FakeQuantOp<P, KIND, ZP>::apply(cm, q, w, o);
        stg_stream16(orow + i, make_uint4(o[0], o[1], o[2], o[3]));
    }
}

// ------------------------------------------------------------------------------------
// GROUP / TENSOR_GROUP: LPG lanes (8 elements each) per group; a warp covers GROUP_UNITS consecutive spans of 32 chunks
// ------------------------------------------------------------------------------------
// quantize + dequantize of one element as the generic kernel does it (generic.cuh: quant_at, then dequant_at), with the scale
// already divided by the global scale (s) and the zero point in x's dtype (zx) and in the effective scale dtype (zs)
__device__ __forceinline__ float fake_generic(float x, float s, float zx, float zs, const DynParams& p) {
    const float t = quant_scalar(x, s, true, zx, p.cd, p.qtype, p.cm.qmin, p.cm.qmax);
    float v = rnd_dt(t, p.se_dt);
    v = rnd_dt(hd_sub(v, zs), p.se_dt);
    return rnd_dt(hd_mul(v, s), p.se_dt);
}

template <class P, int LPG, int KIND, int ZP>
__global__ void __launch_bounds__(256) dyn_group_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, void* __restrict__ scale_out,
                                                        uint8_t* __restrict__ zp_out, int64_t n_chunks, const __grid_constant__ DynParams prm) {
    const int lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x * 8 + (threadIdx.x >> 5)) * (GROUP_UNITS * 32) + lane;
    uint4 v[GROUP_UNITS];
#pragma unroll
    for (int k = 0; k < GROUP_UNITS; ++k) {
        const int64_t c = base + k * 32;
        v[k] = (c < n_chunks) ? ldg_stream16(x + c) : make_uint4(0, 0, 0, 0);   // groups never straddle n_chunks: n_chunks % LPG == 0
    }
#pragma unroll
    for (int k = 0; k < GROUP_UNITS; ++k) {
        const int64_t c = base + k * 32;
        uint32_t mn2 = v[k].x, mx2 = v[k].x;
        obs_chunk_minmax<P>(v[k], mn2, mx2);
#pragma unroll
        for (int d = 1; d < LPG; d <<= 1) {
            mn2 = min2_nan<P>(mn2, __shfl_xor_sync(0xffffffffu, mn2, d));
            mx2 = max2_nan<P>(mx2, __shfl_xor_sync(0xffffffffu, mx2, d));
        }
        if (c >= n_chunks) continue;
        float lo, hi;
        obs_range2<P>(mn2, mx2, lo, hi);
        float s, zq = 0.f;
        if (prm.srule == SR_MX) {
            s = obs_mx_scale<P::DT>(fmax_nan(fabsf(lo), fabsf(hi)), prm.cm.bits);
        } else if (prm.srule == SR_FP8) {
            uint32_t byte;
            const float st = obs_sym_scale<P::DT>(lo, hi, prm.cm.qmin, prm.cm.qmax);
            s = obs_fp8_scale(prm.gs ? __fmul_rn(__ldg(prm.gs), st) : st, byte);   // global_scale * scales in float32
        } else {
            s = obs_scale_zp<P::DT>(lo, hi, prm.asym != 0, prm.cm.qmin, prm.cm.qmax, zq);
        }
        if ((lane & (LPG - 1)) == 0) {
            const int64_t g = c / LPG;
            if (prm.scale_f32) reinterpret_cast<float*>(scale_out)[g] = s;
            else reinterpret_cast<unsigned short*>(scale_out)[g] = (unsigned short)P::from_float1(s);
            zp_out[g] = (uint8_t)(int8_t)(int)zq;
        }
        const uint32_t w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
        uint32_t o[4];
        if constexpr (KIND == K_SCALAR) {
            // eff_scale (generic.cuh): the stored scale in the effective scale dtype, divided by the global scale there
            float se = rnd_dt(s, prm.se_dt);
            if (prm.gs) se = rnd_dt(hd_div(se, __ldg(prm.gs)), prm.se_dt);
            const float zv = prm.zp_i8 ? zq : 0.f;
            const float zx = rnd_dt(zv, prm.x_dt), zs = rnd_dt(zv, prm.se_dt);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                o[j] = P::from_float1(fake_generic(P::lo(w[j]), se, zx, zs, prm)) | (P::from_float1(fake_generic(P::hi(w[j]), se, zx, zs, prm)) << 16);
        } else {
            RawQP q;
            q.s = P::from_float1(s);
            q.z = (int)zq;
            FakeQuantOp<P, KIND, ZP>::apply(prm.cm, q, w, o);
        }
        stg_stream16(out + c, make_uint4(o[0], o[1], o[2], o[3]));
    }
}

// ------------------------------------------------------------------------------------
// launch selection
// ------------------------------------------------------------------------------------
template <class P, int KIND, int ZP, int ASYM>
static void launch_token(const uint4* x, uint4* out, void* s, uint8_t* z, int64_t rows, int units, const Common& cm, cudaStream_t st) {
    if (units <= 2 * 256) dyn_token_kernel<P, KIND, ZP, ASYM, 256, 2><<<(unsigned)rows, 256, 0, st>>>(x, out, s, z, units, cm);
    else if (units <= 8 * 256) dyn_token_kernel<P, KIND, ZP, ASYM, 256, 8><<<(unsigned)rows, 256, 0, st>>>(x, out, s, z, units, cm);
    else dyn_token_kernel<P, KIND, ZP, ASYM, 512, 8><<<(unsigned)rows, 512, 0, st>>>(x, out, s, z, units, cm);
}
template <class P>
static void launch_token_p(int kind, bool asym, const uint4* x, uint4* out, void* s, uint8_t* z, int64_t rows, int units, const Common& cm,
                           cudaStream_t st) {
    if (kind == QF8) launch_token<P, QF8, 2, 0>(x, out, s, z, rows, units, cm, st);
    else if (kind == QI_WIDE) { if (asym) launch_token<P, QI_WIDE, 1, 1>(x, out, s, z, rows, units, cm, st); else launch_token<P, QI_WIDE, 1, 0>(x, out, s, z, rows, units, cm, st); }
    else { if (asym) launch_token<P, QI_NARROW, 1, 1>(x, out, s, z, rows, units, cm, st); else launch_token<P, QI_NARROW, 1, 0>(x, out, s, z, rows, units, cm, st); }
}

template <class P, int KIND, int ZP>
static void launch_group(int lpg, const uint4* x, uint4* out, void* s, uint8_t* z, int64_t n_chunks, const DynParams& prm, cudaStream_t st) {
    const unsigned blocks = (unsigned)((n_chunks + 256 * GROUP_UNITS - 1) / (256 * GROUP_UNITS));
    switch (lpg) {
    case 2: dyn_group_kernel<P, 2, KIND, ZP><<<blocks, 256, 0, st>>>(x, out, s, z, n_chunks, prm); break;
    case 4: dyn_group_kernel<P, 4, KIND, ZP><<<blocks, 256, 0, st>>>(x, out, s, z, n_chunks, prm); break;
    case 8: dyn_group_kernel<P, 8, KIND, ZP><<<blocks, 256, 0, st>>>(x, out, s, z, n_chunks, prm); break;
    default: dyn_group_kernel<P, 16, KIND, ZP><<<blocks, 256, 0, st>>>(x, out, s, z, n_chunks, prm); break;
    }
}
template <class P>
static void launch_group_p(int kind, int lpg, const uint4* x, uint4* out, void* s, uint8_t* z, int64_t n_chunks, const DynParams& prm,
                           cudaStream_t st) {
    switch (kind) {
    case QF8: launch_group<P, QF8, 2>(lpg, x, out, s, z, n_chunks, prm, st); break;
    case QI_WIDE: launch_group<P, QI_WIDE, 1>(lpg, x, out, s, z, n_chunks, prm, st); break;
    case QI_NARROW: launch_group<P, QI_NARROW, 1>(lpg, x, out, s, z, n_chunks, prm, st); break;
    default: launch_group<P, K_SCALAR, 0>(lpg, x, out, s, z, n_chunks, prm, st); break;
    }
}

static int unsupported(const char* why) {
    set_error("dynamic_fake_quantize: %s; run the observer and fake_quantize separately", why);
    return CT_E_UNSUPPORTED;
}

static bool is_inf_div(int64_t v) { return v == CT_DIV_INF; }

}  // namespace ctb

using namespace ctb;

extern "C" int ct_dynamic_fake_quantize(const ct_quant_desc* d, int asymmetric, int scale_dtype_arg, const void* x, void* out, void* scale_out,
                                        void* zp_out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    if (device == CT_DEVICE_CPU) return unsupported("no host twin");
    const int xdt = d->x_dtype;
    if ((xdt != CT_BF16 && xdt != CT_F16) || d->out_dtype != xdt) return unsupported("x and out must be bf16 or fp16 of one dtype");
    const bool int_q = d->qtype == CT_Q_INT && d->num_bits >= 1 && d->num_bits <= 8;
    const bool fp8_q = d->qtype == CT_Q_FLOAT && d->num_bits == 8;
    const bool fp4_q = d->qtype == CT_Q_FP4 && d->num_bits == 4;
    if (!int_q && !fp8_q && !fp4_q) return unsupported("int 1..8, fp8 or fp4 quantization only");
    if (d->rows < 0 || d->cols <= 0 || d->cols % 8 != 0) return unsupported("rows of a multiple of 8 elements only");
    const int64_t n = d->rows * d->cols;
    if (n / 8 >= 0x7fffffffLL || d->rows >= 0x7fffffffLL) return unsupported("tensor too large");
    if (!aligned16(x) || !aligned16(out)) return unsupported("x and out must be 16-byte aligned");
    if (d->zp_dtype != CT_I8 && d->zp_dtype != CT_F8E4M3 && d->zp_dtype != CT_U8) return unsupported("zero point must be int8, float8_e4m3fn or uint8");
    const bool asym = asymmetric != 0;
    if (asym && !(int_q && d->zp_dtype == CT_I8)) return unsupported("asymmetric schemes need integer codes and an int8 zero point");
    const bool gs = d->global_scale != nullptr;
    int srule;
    if (scale_dtype_arg == CT_NONE) srule = SR_PLAIN;
    else if (scale_dtype_arg == CT_F8E4M3 && !asym) srule = SR_FP8;
    else if (scale_dtype_arg == CT_E8M0 && !asym && !int_q && !gs && d->cdiv == 32) srule = SR_MX;
    else return unsupported("scale_dtype must be none, float8_e4m3fn, or uint8 with MX group 32");
    if (gs && (srule != SR_FP8 || d->scale_dtype != CT_F32 || d->seff_dtype != CT_F32 || d->compute_dtype != CT_F32))
        return unsupported("a global scale is taken with scale_dtype float8_e4m3fn (NVFP4) only");
    if (!gs && d->scale_dtype != xdt) return unsupported("the scale is held in x's dtype without a global scale");
    if (n == 0) return CT_OK;
    if (!x || !out || !scale_out || !zp_out) { set_error("null tensor pointer"); return CT_E_ARG; }
    // the element rule ct_fake_quantize takes for the same tensors
    const bool fast = !gs && !fp4_q && d->compute_dtype == xdt && d->seff_dtype == xdt && (d->zp_dtype == CT_I8 || (d->zp_dtype == CT_F8E4M3 && fp8_q));
    const int kind = fast ? fake_kind(xdt, d->qtype, d->num_bits) : K_SCALAR;

    const bool tensor = is_inf_div(d->rdiv) && is_inf_div(d->cdiv);
    const bool token = d->rdiv == 1 && d->s_row_stride == 1 && is_inf_div(d->cdiv);
    const bool group = d->rdiv == 1 && !is_inf_div(d->cdiv) && (d->cdiv == 16 || d->cdiv == 32 || d->cdiv == 64 || d->cdiv == 128) &&
                       d->cols % d->cdiv == 0 && d->s_row_stride == d->cols / d->cdiv;
    if ((tensor || token) && (srule != SR_PLAIN || !fast)) return unsupported("per-token and per-tensor scales are int or fp8 in x's dtype");
    if (token && d->cols > TOKEN_MAX_COLS) return unsupported("per-token rows up to 32768 columns");
    if (!tensor && !token && !group) return unsupported("TOKEN, TENSOR, or GROUP with group size 16, 32, 64 or 128 dividing the row");

    int rc = check_device(device);
    if (rc) return rc;
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const uint4* xp = reinterpret_cast<const uint4*>(x);
    uint4* op = reinterpret_cast<uint4*>(out);
    uint8_t* zp = reinterpret_cast<uint8_t*>(zp_out);

    if (tensor) {
        // ct_observe_tensor (kind 0) writes the scale and an asymmetric zero point; a symmetric scheme's zero point is a zero byte
        ct_quant_desc q = *d;
        q.global_scale = nullptr;
        q.aux = nullptr;
        rc = ct_observe_tensor(&q, x, 0, scale_out, asym ? zp_out : nullptr, device, stream);
        if (rc) return rc;
        if (!asym) CT_CUDA_TRY(cudaMemsetAsync(zp_out, 0, 1, st));
        const void* ins[1] = {x};
        const void* scs[1] = {scale_out};
        const void* zps[1] = {zp_out};
        void* outs[1] = {out};
        return run_batched(CT_OP_FAKE_QUANTIZE, 1, &q, ins, scs, zps, nullptr, outs, device, st);
    }
    if (token) {
        const Common cm = make_common(xdt, d->qtype, d->num_bits);
        const int units = (int)(d->cols / 8);
        if (xdt == CT_BF16) launch_token_p<BF16>(kind, asym, xp, op, scale_out, zp, d->rows, units, cm, st);
        else launch_token_p<F16>(kind, asym, xp, op, scale_out, zp, d->rows, units, cm, st);
    } else {
        DynParams prm;
        memset(&prm, 0, sizeof(prm));
        prm.cm = make_common(xdt, d->qtype, d->num_bits);
        prm.srule = srule;
        prm.asym = asym ? 1 : 0;
        prm.scale_f32 = gs ? 1 : 0;
        prm.zp_i8 = d->zp_dtype == CT_I8 ? 1 : 0;
        prm.x_dt = xdt;
        prm.cd = d->compute_dtype;
        prm.se_dt = d->seff_dtype;
        prm.qtype = d->qtype;
        prm.gs = reinterpret_cast<const float*>(d->global_scale);
        const int lpg = (int)(d->cdiv / 8);
        if (xdt == CT_BF16) launch_group_p<BF16>(kind, lpg, xp, op, scale_out, zp, n / 8, prm, st);
        else launch_group_p<F16>(kind, lpg, xp, op, scale_out, zp, n / 8, prm, st);
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

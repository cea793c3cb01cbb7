// observe_tensor.cu -- per-TENSOR observers without a host round trip (SURVEY.md 8(f) rank 1, the TENSOR-strategy remainder):
//   kind 0: memoryless min-max observer + calculate_qparams (quantization/utils/helpers.py:50-137) for ONE scale (+ zero point) per tensor
//           -- the FP8 preset (BASELINE config 3), per-tensor INT8 / INT4
//   kind 1: generate_gparam (helpers.py:308-337), the float32 global scale of NVFP4
// A grid-wide reduction has to finish before anything can be scaled, so the flow is two phases in ONE ABI call:
//   phase 1  minmax kernel: 16-byte loads, packed min / max, one atomicMax pair per CTA on order-preserving integer keys; the LAST CTA
//            to finish (ticket counter) derives the qparams with the reference's per-op rounding and writes them to device memory
//   phase 2  the streaming quantize kernel (stream.cuh) reading that device-resident scale
// The reference reads the weight twice as well (observer pass, quantize pass) but goes through the host for the scalar and through a
// chain of torch ops; here phase 1 loads with an L2 evict_last hint when the tensor takes at most half of the device's L2 (25 MB on
// an H100), so that phase 2 is served from L2 (DRAM traffic ~ 2 + 1 B / element instead of 2 + 2 + 1) while the other half stays
// for everything else -- the 1024 x 4096 k / v projections of Llama-3-8B qualify, a 4096 x 4096 bf16 weight (32 MB) does not.
#include <cstring>

#include "engine.h"
#include "observe_core.cuh"
#include "ops.cuh"

namespace ctb {

__device__ __forceinline__ uint32_t enc_f32(float f) {          // order-preserving: larger float <=> larger key; every key > 0
    if (f != f) return 0xffffffffu;                               // a NaN of either sign wins the atomicMax and decodes to NaN
    const uint32_t u = __float_as_uint(f);
    return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float dec_f32(uint32_t e) { return __uint_as_float(e ^ ((e >> 31) ? 0x80000000u : 0xffffffffu)); }

__device__ __forceinline__ uint4 ldg16_hint(const void* p, uint64_t policy) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(policy));
    return r;
}
__device__ __forceinline__ uint64_t l2_policy(bool keep) {
    uint64_t p;
    if (keep) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    else asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}

struct ObsParams {
    float qmin, qmax;
    int kind;        // 0 calculate_qparams, 1 generate_gparam
    int asym;        // kind 0: int8 zero point wanted
    int keep_l2;     // the tensor takes at most half of the L2: load with evict_last
};

// slots[0] = max over enc(-min(x, 0)), slots[1] = max over enc(max(x, 0)), slots[2] = CTAs done; zeroed before the launch
template <class P>
__global__ void __launch_bounds__(256) minmax_qparams_kernel(const uint4* __restrict__ x, int64_t n_vec, uint32_t* __restrict__ slots,
                                                             void* __restrict__ scale_out, int8_t* __restrict__ zp_out, const __grid_constant__ ObsParams prm) {
    __shared__ float red[2][8];
    const uint64_t policy = l2_policy(prm.keep_l2 != 0);
    const int64_t stride = (int64_t)gridDim.x * 256;
    float lo = 0.f, hi = 0.f;                                    // the observer clamps min <= 0 <= max: 0 is neutral
    if constexpr (P::DT == CT_F32) {
        for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n_vec; i += 4 * stride) {
            uint4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = (i + u * stride < n_vec) ? ldg16_hint(x + i + u * stride, policy) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float a = __uint_as_float(v[u].x), b = __uint_as_float(v[u].y), c = __uint_as_float(v[u].z), d = __uint_as_float(v[u].w);
                lo = fmin_nan(lo, fmin_nan(fmin_nan(a, b), fmin_nan(c, d)));
                hi = fmax_nan(hi, fmax_nan(fmax_nan(a, b), fmax_nan(c, d)));
            }
        }
    } else {
        uint32_t mn2 = 0u, mx2 = 0u;                             // +0.0 | +0.0
        for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n_vec; i += 4 * stride) {
            uint4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) v[u] = (i + u * stride < n_vec) ? ldg16_hint(x + i + u * stride, policy) : make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int u = 0; u < 4; ++u) obs_chunk_minmax<P>(v[u], mn2, mx2);
        }
        obs_range2<P>(mn2, mx2, lo, hi);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        lo = fmin_nan(lo, __shfl_xor_sync(0xffffffffu, lo, d));
        hi = fmax_nan(hi, __shfl_xor_sync(0xffffffffu, hi, d));
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = lo; red[1][threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int w = 1; w < 8; ++w) { lo = fmin_nan(lo, red[0][w]); hi = fmax_nan(hi, red[1][w]); }
    atomicMax(slots + 0, enc_f32(-lo));
    atomicMax(slots + 1, enc_f32(hi));
    __threadfence();
    if (atomicAdd(slots + 2, 1u) != gridDim.x - 1) return;
    // ---- last CTA: every partial is in ----
    __threadfence();
    lo = -dec_f32(atomicMax(slots + 0, 0u));                     // min(min_vals, 0)
    hi = dec_f32(atomicMax(slots + 1, 0u));                      // max(max_vals, 0)
    if (prm.kind == 1) {
        // generate_gparam (helpers.py:308-337): 448 * 6 / clamp(max|x|, tiny) in x's dtype, NaN / inf -> 1, as float32.
        // `python_float / tensor` is Tensor.__rtruediv__ = tensor.reciprocal() * python_float: TWO roundings to x's dtype (1 / top, then
        // the product), not one division -- 2688 / 1.745 is 1541 in fp16 this way, 1540 by a correctly rounded quotient.
        float top = fmax_nan(fmax_nan(fabsf(lo), fabsf(hi)), obs_tiny<P::DT>());
        float g = obs_round<P::DT>(__fmul_rn(obs_round<P::DT>(__frcp_rn(top)), 2688.0f));
        if (g != g || fabsf(g) == __int_as_float(0x7f800000)) g = 1.0f;
        *reinterpret_cast<float*>(scale_out) = g;
        return;
    }
    // calculate_qparams, each op rounded to T (helpers.py:74-131)
    float zq;
    const float s = obs_scale_zp<P::DT>(lo, hi, prm.asym != 0, prm.qmin, prm.qmax, zq);
    if constexpr (P::DT == CT_F32) *reinterpret_cast<float*>(scale_out) = s;
    else *reinterpret_cast<unsigned short*>(scale_out) = (unsigned short)P::from_float1(s);
    if (prm.asym && zp_out) *zp_out = (int8_t)(int)zq;
}

static int observe_tensor(const ct_quant_desc* d, const void* x, int kind, void* scale_out, void* zp_out, int device, cudaStream_t st) {
    const int64_t n = d->rows * d->cols;
    const int es = dt_size(d->x_dtype);
    if (!is_float_dt(d->x_dtype) || n <= 0 || (n * es) % 16 != 0 || !aligned16(x)) {
        set_error("per-tensor observer supports contiguous bf16 / fp16 / fp32 tensors whose byte size is a multiple of 16, 16-byte aligned; "
                  "run the observer with torch reductions otherwise");
        return CT_E_UNSUPPORTED;
    }
    if (kind == 0 && (d->qtype == CT_Q_FP4 || (d->qtype == CT_Q_FLOAT && zp_out))) {
        set_error("per-tensor observer: fp8 is symmetric only, fp4 takes the NVFP4 observer");
        return CT_E_UNSUPPORTED;
    }
    ObsParams prm;
    if (d->qtype == CT_Q_INT) { const float r = (float)(1 << d->num_bits); prm.qmax = r / 2 - 1; prm.qmin = -r / 2; }
    else { prm.qmax = 448.f; prm.qmin = -448.f; }
    prm.kind = kind;
    prm.asym = (kind == 0 && zp_out) ? 1 : 0;
    prm.keep_l2 = (n * es <= l2_bytes(device) / 2) ? 1 : 0;
    uint32_t* slots = nullptr;
    int rc = scratch_alloc(reinterpret_cast<void**>(&slots), 16, device, st);
    if (rc) return rc;
    CT_CUDA_TRY(cudaMemsetAsync(slots, 0, 16, st));
    const int64_t n_vec = n * es / 16;
    int64_t blocks = (n_vec + 256 * 4 - 1) / (256 * 4);
    const int64_t cap = (int64_t)sm_count(device) * 8;
    if (blocks > cap) blocks = cap;
    const uint4* xp = reinterpret_cast<const uint4*>(x);
    int8_t* zp = reinterpret_cast<int8_t*>(zp_out);
    switch (d->x_dtype) {
    case CT_BF16: minmax_qparams_kernel<BF16><<<(unsigned)blocks, 256, 0, st>>>(xp, n_vec, slots, scale_out, zp, prm); break;
    case CT_F16: minmax_qparams_kernel<F16><<<(unsigned)blocks, 256, 0, st>>>(xp, n_vec, slots, scale_out, zp, prm); break;
    default: minmax_qparams_kernel<F32><<<(unsigned)blocks, 256, 0, st>>>(xp, n_vec, slots, scale_out, zp, prm); break;
    }
    count_launch();
    cudaFreeAsync(slots, st);
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

}  // namespace ctb

using namespace ctb;

extern "C" {

int ct_observe_tensor(const ct_quant_desc* d, const void* x, int kind, void* scale_out, void* zp_out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    if (kind != 0 && kind != 1) { set_error("kind must be 0 (calculate_qparams) or 1 (generate_gparam)"); return CT_E_ARG; }
    int rc = check_device(device);
    if (rc) return rc;
    if (!x || !scale_out) { set_error("null tensor pointer"); return CT_E_ARG; }
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    return observe_tensor(d, x, kind, scale_out, zp_out, device, reinterpret_cast<cudaStream_t>(stream));
}

int ct_observe_quantize_tensor(const ct_quant_desc* d, const void* x, void* scale_out, void* zp_out, void* q_out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    int rc = check_device(device);
    if (rc) return rc;
    if (!x || !scale_out || !q_out) { set_error("null tensor pointer"); return CT_E_ARG; }
    if (!(d->rdiv == CT_DIV_INF && d->cdiv == CT_DIV_INF) || d->scale_dtype != d->x_dtype) {
        set_error("ct_observe_quantize_tensor needs the TENSOR strategy (rdiv = cdiv = CT_DIV_INF) and the scale in x's dtype");
        return CT_E_UNSUPPORTED;
    }
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    rc = observe_tensor(d, x, 0, scale_out, zp_out, device, st);
    if (rc) return rc;
    // phase 2: the streaming kernels with the device-resident qparams (packed int32 when q_dtype == CT_I32, else 1-byte codes)
    ct_quant_desc q = *d;
    const int op = (d->q_dtype == CT_I32) ? CT_OP_QUANTIZE_PACK : CT_OP_QUANTIZE;
    if (op == CT_OP_QUANTIZE_PACK) q.q_dtype = CT_I8;
    q.zp_dtype = zp_out ? CT_I8 : CT_NONE;
    const void* ins[1] = {x};
    const void* scs[1] = {scale_out};
    const void* zps[1] = {zp_out};
    void* outs[1] = {q_out};
    return run_batched(op, 1, &q, ins, scs, zps, nullptr, outs, device, st);
}

}  // extern "C"

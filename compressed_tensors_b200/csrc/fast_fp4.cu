// fast_fp4.cu -- streaming instantiations of the FP4 functors (fp4_ops.cuh) and the device-side exhaustive check of the
// NVFP4 division shortcut.
#include <algorithm>

#include "engine.h"
#include "fp4_ops.cuh"

namespace ctb {

// quantize + pack.  Without a global scale: MX-style, scale and arithmetic in T, zero point absent, uint8 or int8.  With one: NVFP4,
// float32 arithmetic, scale in T or float32, zero point absent or float8_e4m3fn.
template <class P>
static StreamKernel fp4_quantpack_p(bool global_scale, int scale_dt, int zp_dt) {
    if (!global_scale) {
        if (scale_dt != P::DT) return {};
        if (zp_dt == CT_NONE) return stream_kernel<Fp4MxQuantPackOp<P, FZ_NONE>>();
        if (zp_dt == CT_U8) return stream_kernel<Fp4MxQuantPackOp<P, FZ_U8>>();
        if (zp_dt == CT_I8) return stream_kernel<Fp4MxQuantPackOp<P, FZ_I8>>();
    } else if (scale_dt == P::DT) {
        if (zp_dt == CT_NONE) return stream_kernel<Fp4NvQuantPackOp<P, FS_SAME, FZ_NONE>>();
        if (zp_dt == CT_F8E4M3) return stream_kernel<Fp4NvQuantPackOp<P, FS_SAME, FZ_F8>>();
    } else if (scale_dt == CT_F32) {
        if (zp_dt == CT_NONE) return stream_kernel<Fp4NvQuantPackOp<P, FS_F32, FZ_NONE>>();
        if (zp_dt == CT_F8E4M3) return stream_kernel<Fp4NvQuantPackOp<P, FS_F32, FZ_F8>>();
    }
    return {};
}
StreamKernel fp4_quantpack_kernel(int p_dt, bool global_scale, int scale_dt, int zp_dt) {
    if (p_dt == CT_BF16) return fp4_quantpack_p<BF16>(global_scale, scale_dt, zp_dt);
    if (p_dt == CT_F16) return fp4_quantpack_p<F16>(global_scale, scale_dt, zp_dt);
    return {};
}

// NVFP4 observe + quantize + pack: the float8_e4m3fn scale is an OUTPUT
StreamKernel fp4_observe_kernel(int p_dt, bool mse) {
    if (p_dt == CT_BF16) return mse ? stream_kernel<Fp4NvObserveQuantPackOp<BF16, true>>() : stream_kernel<Fp4NvObserveQuantPackOp<BF16>>();
    if (p_dt == CT_F16) return mse ? stream_kernel<Fp4NvObserveQuantPackOp<F16, true>>() : stream_kernel<Fp4NvObserveQuantPackOp<F16>>();
    return {};
}

// The NVFP4 MSE mode's second launch: the stop step from the call's `any` bits; a group of 16 whose mask has a bit above it is rewritten,
// by one thread, with its last improving step <= S: its fp8 scale byte and its 8 bytes of nibbles, with the generic kernels' per-element
// source (IEEE divisions, equal to the streaming shortcuts).  The global scale is an input and stays.
template <class P>
__global__ void __launch_bounds__(256) mse_fixup_nvfp4_kernel(const ct_mse_block* B, const void* x, const float* gsp, uint8_t* scale, uint8_t* packed,
                                                              int64_t n_groups) {
    const uint64_t keep = mse_keep(B);
    const float gs = *gsp;
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
        const uint64_t m = B->masks[g];
        if ((m & ~keep) == 0) continue;
        float amax = 0.f;   // a group that improved is finite
        for (int j = 0; j < 16; ++j) amax = fmaxf(amax, fabsf(load_as_f32(x, g * 16 + j, P::DT)));
        const float a = rnd_dt(amax * B->shrink[mse_last(m, keep)], P::DT);
        uint32_t byte;
        const float s = __fdiv_rn(obs_fp8_scale(__fmul_rn(gs, obs_round<P::DT>(__fdiv_rn(a, 6.0f))), byte), gs);
        scale[g] = (uint8_t)byte;
        for (int j = 0; j < 8; ++j) {
            const float v0 = quant_scalar(load_as_f32(x, g * 16 + 2 * j, P::DT), s, false, 0.f, CT_F32, CT_Q_FP4, -6.f, 6.f);
            const float v1 = quant_scalar(load_as_f32(x, g * 16 + 2 * j + 1, P::DT), s, false, 0.f, CT_F32, CT_Q_FP4, -6.f, 6.f);
            packed[g * 8 + j] = (uint8_t)(fp4_nibble(v0) | (fp4_nibble(v1) << 4));
        }
    }
}

int launch_mse_fixup_nvfp4(const ct_quant_desc& d, const void* x, void* scale, uint8_t* packed, cudaStream_t st) {
    const int64_t n_groups = d.rows * d.cols / 16;
    if (n_groups == 0) return CT_OK;
    const int64_t blocks = std::min<int64_t>((n_groups + 255) / 256, 4096);
    const ct_mse_block* B = reinterpret_cast<const ct_mse_block*>(d.aux);
    const float* gs = reinterpret_cast<const float*>(d.global_scale);
    uint8_t* sc = reinterpret_cast<uint8_t*>(scale);
    if (d.x_dtype == CT_BF16) mse_fixup_nvfp4_kernel<BF16><<<(unsigned)blocks, 256, 0, st>>>(B, x, gs, sc, packed, n_groups);
    else mse_fixup_nvfp4_kernel<F16><<<(unsigned)blocks, 256, 0, st>>>(B, x, gs, sc, packed, n_groups);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

// unpack + dequantize: the scale in the output dtype, or as stored (float8_e4m3fn / E8M0)
template <class P>
static StreamKernel fp4_unpackdeq_p(int scale_dt) {
    if (scale_dt == P::DT) return stream_kernel<Fp4UnpackDequantOp<P, FS_SAME>>();
    if (scale_dt == CT_F8E4M3) return stream_kernel<Fp4UnpackDequantOp<P, FS_F8>>();
    if (scale_dt == CT_E8M0) return stream_kernel<Fp4UnpackDequantOp<P, FS_E8M0>>();
    return {};
}
StreamKernel fp4_unpackdeq_kernel(int p_dt, int scale_dt) {
    if (p_dt == CT_BF16) return fp4_unpackdeq_p<BF16>(scale_dt);
    if (p_dt == CT_F16) return fp4_unpackdeq_p<F16>(scale_dt);
    return {};
}

// ---- selftest: the E2M1 code of quotient(x, s) (reciprocal + one residual step) must equal the code of div.rn(x, s) for
// ---- every 16-bit x and every float32 scale significand, at several scale exponents inside the fast range ------------------
// mode 0: E2M1 code of the quantization quotient (weights / effective scale).  mode 1: the float32 VALUE of scale / global_scale
// for every 16-bit scale with |scale| in [2^-40, 2^14] (what Fp4UnpackDequantOp uses recip_div for).
template <class P>
__global__ void __launch_bounds__(256) fp4_division_selftest_kernel(unsigned long long* mismatches, int exp_field, int mode) {
    using Op = Fp4NvQuantPackOp<P, FS_F32, FZ_NONE>;
    unsigned long long local = 0;
    for (uint32_t m = blockIdx.x; m < (1u << 23); m += gridDim.x) {
        const float s = __uint_as_float(((uint32_t)exp_field << 23) | m);
        const float rc = __frcp_rn(s);
        for (uint32_t xp = threadIdx.x; xp < 65536u; xp += blockDim.x) {
            const float x = P::lo(xp);
            if (mode == 1) {
                const float a = fabsf(x);
                if (!(a >= 9.094947017729282e-13f && a <= 16384.0f)) continue;
                if (__float_as_uint(recip_div(x, s, rc)) != __float_as_uint(__fdiv_rn(x, s))) ++local;
                continue;
            }
            const float fast = Op::quotient(P::lo(Op::clamp_x(xp)), s, rc);   // exactly what chunk_fast does; nothing is added without a zero point
            const float ref = __fadd_rn(__fdiv_rn(x, s), 0.0f);
            if (x != x) continue;   // NaN weights are outside the bit-exact contract
            if (f32x2_to_e2m1x2(fast, 0.f) != f32x2_to_e2m1x2(ref, 0.f)) ++local;
        }
    }
    for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(mismatches, local);
}

}  // namespace ctb

extern "C" int ct_selftest_fp4_division(int dtype, int scale_exponent, int mode, uint64_t* mismatches, int device) {
    using namespace ctb;
    if (!mismatches) { set_error("null output"); return CT_E_ARG; }
    if (mode == 0 && (scale_exponent < -100 || scale_exponent > 9)) { set_error("scale exponent outside the fast range [-100, 9] (|scale| in [2^-100, 2^10))"); return CT_E_ARG; }
    if (mode == 1 && (scale_exponent < -60 || scale_exponent > 59)) { set_error("global-scale exponent outside the fast range [-60, 59]"); return CT_E_ARG; }
    if (mode != 0 && mode != 1) { set_error("mode must be 0 or 1"); return CT_E_ARG; }
    int rc = check_device(device);
    if (rc) return rc;
    DeviceGuard guard(device);
    unsigned long long* d = nullptr;
    CT_CUDA_TRY(cudaMalloc(&d, sizeof(unsigned long long)));
    CT_CUDA_TRY(cudaMemset(d, 0, sizeof(unsigned long long)));
    const int ef = scale_exponent + 127;
    if (dtype == CT_BF16) fp4_division_selftest_kernel<BF16><<<GRID_SMS * 16, 256>>>(d, ef, mode);
    else if (dtype == CT_F16) fp4_division_selftest_kernel<F16><<<GRID_SMS * 16, 256>>>(d, ef, mode);
    else { cudaFree(d); set_error("selftest supports bf16 / f16"); return CT_E_DTYPE; }
    count_launch();
    unsigned long long h = 0;
    cudaError_t e = cudaMemcpy(&h, d, sizeof(h), cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (e != cudaSuccess) return cuda_fail(e, "fp4 selftest");
    *mismatches = h;
    return CT_OK;
}

// fp4.cu -- FP4 (E2M1) and MX (E8M0 scale) pieces, generic kernels: cast_to_fp4, nibble pack / unpack,
// fused quantize+pack / unpack+dequantize for any strategy / dtype mix (the streaming fast path for the
// NVFP4 / MXFP4 layouts is fast_fp4.cu), E8M0 scale encode / decode.
// Reference: quantization/utils/fp4_utils.py:77-98, compressors/nvfp4/helpers.py:108-193,
// compressors/nvfp4/base.py:73-128, compressors/mx_utils.py:18-44.
#include "generic.cuh"
#include "observe_core.cuh"

namespace ctb {

__global__ void __launch_bounds__(256) cast_to_fp4_kernel(const void* __restrict__ x, int dt, void* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        store_from_f32(out, i, dt, fp4_round(load_as_f32(x, i, dt)));
}

// one thread per output byte = two consecutive elements (cols is even, so pairs never straddle rows)
__global__ void __launch_bounds__(256) pack_fp4_kernel(const void* __restrict__ x, int dt, uint8_t* __restrict__ out, int64_t n_bytes) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_bytes; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (uint8_t)(fp4_nibble(load_as_f32(x, 2 * i, dt)) | (fp4_nibble(load_as_f32(x, 2 * i + 1, dt)) << 4));
}

__global__ void __launch_bounds__(256) unpack_fp4_kernel(const uint8_t* __restrict__ in, void* __restrict__ out, int out_dt, int64_t n_bytes) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_bytes; i += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t b = in[i];
        store_from_f32(out, 2 * i, out_dt, fp4_value(b & 15u));
        store_from_f32(out, 2 * i + 1, out_dt, fp4_value(b >> 4));
    }
}

__global__ void __launch_bounds__(256) fp4_quantpack_generic_kernel(const __grid_constant__ GParams p) {
    const int64_t half = p.cols / 2, n_bytes = p.rows * half;
    uint8_t* out = reinterpret_cast<uint8_t*>(p.out);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_bytes; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / half, c = (i - r * half) * 2;
        out[i] = (uint8_t)(fp4_nibble(quant_at(p, r, c)) | (fp4_nibble(quant_at(p, r, c + 1)) << 4));
    }
}

__global__ void __launch_bounds__(256) fp4_unpackdeq_generic_kernel(const __grid_constant__ GParams p) {
    const int64_t half = p.cols / 2, n_bytes = p.rows * half;
    const uint8_t* in = reinterpret_cast<const uint8_t*>(p.in);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_bytes; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / half, c = (i - r * half) * 2;
        const uint32_t b = in[i];
        store_from_f32(p.out, r * p.cols + c, p.out_dt, dequant_at(p, fp4_value(b & 15u), r, c));
        store_from_f32(p.out, r * p.cols + c + 1, p.out_dt, dequant_at(p, fp4_value(b >> 4), r, c + 1));
    }
}

// 127 + floor(log2(scale)) with log2 and floor in the scale's dtype, -> int32 -> uint8 (wraps); mx_utils.py:30-31 (observe_core.cuh)
__global__ void __launch_bounds__(256) mx_scale_compress_kernel(const void* __restrict__ s, int dt, uint8_t* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = (uint8_t)mx_scale_code(load_as_f32(s, i, dt), dt);
}

// 2.0 ** (e - 127).to(bfloat16) -> bfloat16; mx_utils.py:43-44
__global__ void __launch_bounds__(256) mx_scale_decompress_kernel(const uint8_t* __restrict__ in, __nv_bfloat16* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = __float2bfloat16_rn(load_as_f32(in, i, CT_E8M0));
}

// ---- launchers ---------------------------------------------------------------------------------
int launch_cast_to_fp4(const void* x, int dt, void* out, int64_t n, cudaStream_t st) {
    if (n == 0) return CT_OK;
    cast_to_fp4_kernel<<<grid_for(n), 256, 0, st>>>(x, dt, out, n);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
int launch_pack_fp4(const void* x, int dt, uint8_t* out, int64_t rows, int64_t cols, cudaStream_t st) {
    const int64_t nb = rows * cols / 2;
    if (nb == 0) return CT_OK;
    pack_fp4_kernel<<<grid_for(nb), 256, 0, st>>>(x, dt, out, nb);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
int launch_unpack_fp4(const uint8_t* in, void* out, int out_dt, int64_t rows, int64_t cols, cudaStream_t st) {
    const int64_t nb = rows * cols / 2;
    if (nb == 0) return CT_OK;
    unpack_fp4_kernel<<<grid_for(nb), 256, 0, st>>>(in, out, out_dt, nb);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
int launch_generic_quantpack_fp4(const ct_quant_desc& d, const void* x, const void* scale, const void* zp,
                                 const int32_t* g_idx, uint8_t* packed, cudaStream_t st) {
    if (d.rows * d.cols == 0) return CT_OK;
    GParams p = make_params(d, x, scale, zp, g_idx, packed);
    fp4_quantpack_generic_kernel<<<grid_for(d.rows * d.cols / 2), 256, 0, st>>>(p);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
int launch_generic_unpackdeq_fp4(const ct_quant_desc& d, const uint8_t* packed, const void* scale, const void* zp,
                                 const int32_t* g_idx, void* out, cudaStream_t st) {
    if (d.rows * d.cols == 0) return CT_OK;
    GParams p = make_params(d, packed, scale, zp, g_idx, out);
    fp4_unpackdeq_generic_kernel<<<grid_for(d.rows * d.cols / 2), 256, 0, st>>>(p);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
int launch_mx_scale_compress(const void* s, int dt, uint8_t* out, int64_t n, cudaStream_t st) {
    if (n == 0) return CT_OK;
    mx_scale_compress_kernel<<<grid_for(n), 256, 0, st>>>(s, dt, out, n);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
int launch_mx_scale_decompress(const uint8_t* in, void* out, int64_t n, cudaStream_t st) {
    if (n == 0) return CT_OK;
    mx_scale_decompress_kernel<<<grid_for(n), 256, 0, st>>>(in, reinterpret_cast<__nv_bfloat16*>(out), n);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

}  // namespace ctb

// engine.h -- internal interfaces between the translation units of libct_b200.so
#pragma once

#include "common.cuh"
#include "stream.cuh"

namespace ctb {

// ---- fast (flat, streaming) path: one selector per kernel family, defined in the file that instantiates it -----------------
// Each returns the kernel for its arguments, or one with a null `launch` when no instantiation exists.  p_dt: CT_BF16 / CT_F16 / CT_F32;
// zp_kind: 0 none, 1 int8, 2 float8_e4m3fn; max_unit: the largest thread unit (chunks; 4, 2 or 1) the tensor's layout admits.
StreamKernel quantpack_kernel(int p_dt, int bits, int zp_kind, int max_unit);   // fast_pack.cu
StreamKernel unpackdeq_kernel(int p_dt, int bits, int zp_kind);
StreamKernel bits_kernel(bool pack, int bits);                                  // standalone int8 <-> int32 packing
StreamKernel quant_kernel(int p_dt, bool fp8, int zp_kind, int max_unit);       // fast_quant.cu
StreamKernel dequant_kernel(int p_dt, bool fp8, int zp_kind, bool f32_scale);   // f32_scale: fp8 codes, float32 scale, 16-bit output
StreamKernel fake_kernel(int p_dt, int qtype, int bits, int zp_kind);           // fast_fake.cu
StreamKernel observe_kernel(int p_dt, int bits, bool asym, int lanes_per_group, bool mse); // fast_observe.cu; mse: Job::aux = ct_mse_block
// the MSE mode's stop-step fix-up after observe_kernel(..., mse = true) over the whole tensor of d (d.aux = ct_mse_block)
int launch_mse_fixup_pack(const ct_quant_desc& d, const void* x, void* scale, void* zp, int32_t* packed, cudaStream_t st);
int launch_mse_fixup_nvfp4(const ct_quant_desc& d, const void* x, void* scale, uint8_t* packed, cudaStream_t st);   // fast_fp4.cu
StreamKernel fp4_quantpack_kernel(int p_dt, bool global_scale, int scale_dt, int zp_dt);   // fast_fp4.cu; zp_dt CT_NONE: no zero point
StreamKernel fp4_observe_kernel(int p_dt, bool mse);   // mse: Job::zp = ct_mse_block
StreamKernel fp4_unpackdeq_kernel(int p_dt, int scale_dt);
StreamKernel sparse24q_kernel(bool compress, int p_dt, int zp_kind);            // fast_sparse24q.cu: fused 2:4 select + int4

// ---- generic path (any strategy, g_idx, ragged shapes, mixed dtypes) -----------------------
enum GenericMode { G_QUANTIZE = 0, G_DEQUANTIZE = 1, G_FAKE = 2 };
int launch_generic_quant(int mode, const ct_quant_desc& d, const void* in, const void* scale, const void* zp,
                         const int32_t* g_idx, void* out, cudaStream_t stream);
int launch_generic_quantpack(const ct_quant_desc& d, const void* x, const void* scale, const void* zp,
                             const int32_t* g_idx, int32_t* packed, cudaStream_t stream);
int launch_generic_unpackdeq(const ct_quant_desc& d, const int32_t* packed, const void* scale, const void* zp,
                             const int32_t* g_idx, void* out, cudaStream_t stream);
int launch_generic_pack(const int8_t* in, int32_t* out, int64_t rows, int64_t cols, int bits, int packed_dim, cudaStream_t stream);
int launch_generic_unpack(const int32_t* in, int8_t* out, int64_t rows, int64_t cols, int bits, int packed_dim, cudaStream_t stream);

// ---- FP4 / MX (fp4.cu) ----------------------------------------------------------------------------
int launch_cast_to_fp4(const void* x, int dt, void* out, int64_t n, cudaStream_t st);
int launch_pack_fp4(const void* x, int dt, uint8_t* out, int64_t rows, int64_t cols, cudaStream_t st);
int launch_unpack_fp4(const uint8_t* in, void* out, int out_dt, int64_t rows, int64_t cols, cudaStream_t st);
int launch_generic_quantpack_fp4(const ct_quant_desc& d, const void* x, const void* scale, const void* zp,
                                 const int32_t* g_idx, uint8_t* packed, cudaStream_t st);
int launch_generic_unpackdeq_fp4(const ct_quant_desc& d, const uint8_t* packed, const void* scale, const void* zp,
                                 const int32_t* g_idx, void* out, cudaStream_t st);
int launch_mx_scale_compress(const void* s, int dt, uint8_t* out, int64_t n, cudaStream_t st);
int launch_mx_scale_decompress(const uint8_t* in, void* out_bf16, int64_t n, cudaStream_t st);

// ---- dispatch (dispatch.cu): one tensor or a table of tensors ---------------------------------
int run_batched(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale,
                const void* const* zp, const int32_t* const* g_idx, void* const* out, int device, cudaStream_t stream);

int check_device(int device);
// the fused BLOCK / MX observers (observe_block_mx.cu): ct_batched ops CT_OP_OBSERVE_QUANTIZE_BLOCK / _MX; scale[i] are OUTPUTS
int run_observe_block_mx(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale, void* const* out,
                         int device, cudaStream_t stream);
Common make_common(int p_dt, int qtype, int bits);   // clamp bounds of a (qtype, bits) in the compute dtype p_dt (dispatch.cu)

// ---- CPU twins (cpu_twin.cu): host code behind device = CT_DEVICE_CPU, same per-element source as the generic kernels ----
int cpu_run_bits(bool pack, const void* in, void* out, int64_t rows, int64_t cols, int bits, int packed_dim);
int cpu_run_one(int op, const ct_quant_desc& d, const void* in, const void* scale, const void* zp, const int32_t* g_idx, void* out);
void cpu_hadamard(const ct_hadamard_job& j);   // ct_hadamard_transform on host pointers (job already validated)

// ---- unstructured bitmask in one pass (bitmask_onepass.cu): decoupled look-back over per-tile counts ----------------
bool bitmask_lookback_ok(int dtype, int64_t rows, int64_t cols, const void* dense, const void* mask, const void* values);
template <bool COMPRESS>
int launch_bitmask_lookback(const void* src, uint8_t* bitmask, void* dst, int64_t* row_offsets, int64_t* nnz_out, int64_t rows, int64_t cols,
                            int device, cudaStream_t st);

}  // namespace ctb

// engine.h -- internal interfaces between the translation units of libct_b200.so
#pragma once

#include "common.cuh"
#include "stream.cuh"

namespace ctb {

// ---- fast (flat, streaming) path -------------------------------------------------------
enum FastOp { F_QUANTPACK = 0, F_UNPACKDEQ = 1, F_QUANT = 2, F_DEQUANT = 3, F_FAKE = 4, F_PACK = 5, F_UNPACK = 6, F_OBSERVE_QP = 7,
              F_FP4_QUANTPACK = 8, F_FP4_UNPACKDEQ = 9, F_S24_QUANTPACK = 10, F_S24_UNPACKDEQ = 11 };

struct FastSig {
    int op;      // FastOp
    int p_dt;    // CT_BF16 / CT_F16 / CT_F32 (unused for F_PACK / F_UNPACK)
    int sel;     // QUANTPACK/UNPACKDEQ/PACK/UNPACK: bits (4 | 8); QUANT/DEQUANT/FAKE: QKind
    int zp;      // 0 none, 1 int8, 2 float8_e4m3fn (fp8 quantize / dequantize / fake_quantize only)
    int group;   // chunks per thread unit (1, 2 or 4): stream.cuh
    bool operator==(const FastSig& o) const { return op == o.op && p_dt == o.p_dt && sel == o.sel && zp == o.zp && group == o.group; }
};

// chunks per tile of the kernel a signature selects (stream.cuh: TileOf<Op>): the 16-bit quantize+pack, unpack+dequantize, quantize and
// dequantize functors run on the big tile
static inline int sig_tile_chunks(const FastSig& s) {
    const bool p16 = (s.p_dt == CT_BF16 || s.p_dt == CT_F16);
    return (p16 && (s.op == F_QUANTPACK || s.op == F_UNPACKDEQ || s.op == F_QUANT || s.op == F_DEQUANT)) ? BIG_TILE_CHUNKS : TILE_CHUNKS;
}

// defined in fast_pack.cu / fast_quant.cu / fast_fake.cu
int launch_fast_quantpack(const FastSig&, const LaunchPlan&, int device, cudaStream_t);
int launch_fast_unpackdeq(const FastSig&, const LaunchPlan&, int device, cudaStream_t);
int launch_fast_quant(const FastSig&, const LaunchPlan&, int device, cudaStream_t);
int launch_fast_dequant(const FastSig&, const LaunchPlan&, int device, cudaStream_t);
int launch_fast_fake(const FastSig&, const LaunchPlan&, int device, cudaStream_t);
int launch_fast_bits(const FastSig&, const LaunchPlan&, int device, cudaStream_t);
int fast_group_quantpack(int p_dt, int bits);   // preferred unit size of the instantiated kernels
int fast_group_quant(int p_dt);
int launch_fast_fp4(const FastSig&, const LaunchPlan&, int device, cudaStream_t);       // fast_fp4.cu; sig.sel / sig.zp: see there
int launch_fast_observe(const FastSig&, const LaunchPlan&, int device, cudaStream_t);   // fast_observe.cu; sig.group = lanes per quantization group
int launch_fast_sparse24q(const FastSig&, const LaunchPlan&, int device, cudaStream_t); // fast_sparse24q.cu: fused 2:4 select + int4 (BASELINE config 4)

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

/*
 * ct_b200.h -- C ABI of the H100-native compress/decompress + quantize/dequantize engine.
 *
 * This is the drop-in boundary for the per-tensor hot path of
 * vllm-project/compressed-tensors.  The reference has no native layer (it is
 * 100% Python/torch eager), so each entry point names the reference Python
 * function whose body it replaces (paths under src/compressed_tensors of the
 * reference).  INTEGRATION.md shows the ctypes stub a maintainer of the
 * reference would add to bind them.
 *
 * Conventions
 *   - plain C types only; every function returns a ct_status_t (0 = ok, <0 = error);
 *     ct_last_error() gives a thread-local message.  Nothing throws across the boundary.
 *   - the caller owns every buffer.  `device` >= 0: all pointers are device pointers on
 *     that CUDA device and the work is ENQUEUED on `stream` (a cudaStream_t passed as
 *     void*; NULL = legacy default stream); no synchronisation happens inside.
 *     Functions named ct_host_* take HOST pointers, stage through the device in
 *     pipelined chunks and return when the outputs are complete in host memory.
 *   - reentrant, no global mutable state besides per-device lazily created scratch
 *     guarded by a mutex (the reference's convert_checkpoint calls decompress from a
 *     thread pool: entrypoints/convert/convert_checkpoint.py:110-134).
 *   - NO SILENT CPU FALLBACK: `device` >= 0 without a usable H100 fails with CT_E_NODEV, always.  The seven per-tensor
 *     entry points of the hot path (ct_pack_int32, ct_unpack_int32, ct_quantize, ct_dequantize, ct_fake_quantize,
 *     ct_quantize_pack_int32, ct_unpack_dequantize_int32, and ct_batched over them) and ct_hadamard_transform have an EXPLICIT CPU twin: pass
 *     device = CT_DEVICE_CPU (-1) with HOST pointers and the call runs synchronously in host code of this library
 *     (csrc/cpu_twin.cu; same per-element source as the generic CUDA kernels), `stream` ignored.  That is the body the reference
 *     calls "eager" (utils/impl_backend.py:98-123): what a GPU-less host and CT_ENFORCE_EAGER=1 get.  Every other entry point
 *     answers CT_E_NODEV / CT_E_UNSUPPORTED for device = -1.
 */
#ifndef CT_B200_H
#define CT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum ct_status_t {
    CT_OK = 0,
    CT_E_DTYPE = -1,       /* unsupported / inconsistent dtype */
    CT_E_BITS = -2,        /* num_bits outside [1, 8] */
    CT_E_SHAPE = -3,       /* inconsistent shapes (e.g. cols % group_size != 0) */
    CT_E_ALIGN = -4,       /* pointer alignment not supported */
    CT_E_CUDA = -5,        /* CUDA runtime error (message in ct_last_error) */
    CT_E_ARG = -6,         /* NULL pointer / bad enum */
    CT_E_NODEV = -7,       /* no usable CUDA device: this library has no CPU path */
    CT_E_UNSUPPORTED = -8
} ct_status_t;

typedef enum ct_dtype_t {
    CT_NONE = -1,
    CT_F32 = 0,
    CT_F16 = 1,
    CT_BF16 = 2,
    CT_I8 = 3,
    CT_F8E4M3 = 4,         /* torch.float8_e4m3fn */
    CT_I32 = 5,
    CT_U8 = 6,             /* also torch.bool */
    CT_I64 = 7,
    CT_E8M0 = 8,           /* uint8 biased power-of-two exponent: an MX scale as STORED (compressors/mx_utils.py:18-44) */
    CT_F64 = 9             /* float64: only as the compute precision of ct_hadamard_transform */
} ct_dtype_t;

/* CT_Q_FLOAT = fp8 e4m3 (num_bits 8); CT_Q_FP4 = fp4 e2m1 (num_bits 4: values 0, .5, 1, 1.5, 2, 3, 4, 6 and negatives) */
typedef enum ct_qtype_t { CT_Q_INT = 0, CT_Q_FLOAT = 1, CT_Q_FP4 = 2 } ct_qtype_t;

#define CT_DIV_INF INT64_MAX
#define CT_DEVICE_CPU (-1)   /* explicit CPU twin of the per-tensor entry points (see the conventions above) */

/*
 * One 2-D quantization problem: x is [rows, cols] row-major contiguous.
 * Scale / zero-point element used for x[r, c]:
 *     sidx = (r / rdiv) * s_row_stride + (g_idx ? g_idx[c] : c / cdiv)
 * which covers every strategy of quantization/lifecycle/forward.py:184-241:
 *     TENSOR  rdiv = cdiv = CT_DIV_INF, s_row_stride = 0
 *     CHANNEL/TOKEN  rdiv = 1, s_row_stride = 1, cdiv = CT_DIV_INF
 *     GROUP   rdiv = 1, s_row_stride = n_groups (0 for a one-row scale), cdiv = group_size
 *     BLOCK   rdiv = block_h, s_row_stride = ceil(cols / block_w), cdiv = block_w
 * compute_dtype is the torch promotion of `x / scale` (forward_helpers.py:538): every
 * reference op rounds to it, and the kernels reproduce those roundings bit for bit.
 */
typedef struct ct_quant_desc {
    int64_t rows, cols;
    int64_t rdiv, cdiv, s_row_stride;
    int32_t x_dtype;        /* float tensor: input of quantize / fake_quantize */
    int32_t scale_dtype;
    int32_t zp_dtype;       /* CT_NONE when there is no zero point */
    int32_t compute_dtype;
    int32_t q_dtype;        /* quantized tensor: CT_I8 / CT_F8E4M3, or a float dtype ("dtype=None") */
    int32_t out_dtype;      /* float output of dequantize / fake_quantize */
    int32_t qtype;          /* ct_qtype_t */
    int32_t num_bits;
    /* NVFP4-style two-level scaling (forward_helpers.py:535-536, 559-560, 196-197): when global_scale != NULL
     * (DEVICE pointer to one float32) every op first forms  scale = scale / global_scale  in
     * seff_dtype = result_type(scale, global_scale), and "scale dtype" below means seff_dtype. */
    const void* global_scale;
    int32_t seff_dtype;
    int32_t _reserved;
    /* second tensor of the ops that have two streamed outputs / inputs (CT_OP_SPARSE24_*: the uint8 bitmask [rows, cols/8]);
     * NULL otherwise.  A DEVICE pointer, like global_scale. */
    void* aux;
} ct_quant_desc;

/* ---- library / device ---------------------------------------------------- */
const char* ct_version(void);
const char* ct_last_error(void);
int ct_device_count(void);                 /* 0 when no CUDA device / driver */
int ct_device_ok(int device);              /* 1 if `device` is sm_90 (H100) */
/* number of kernels this library has launched in the calling process */
int64_t ct_launch_count(void);

/* ---- int32 bit packing ---------------------------------------------------
 * replaces compressors/pack_quantized/helpers.py:20-101 (pack_to_int32) and
 * :104-180 (unpack_from_int32) for one 2-D slice.
 *   in  int8 [rows, cols]
 *   packed_dim = 1: out int32 [rows, ceil(cols*bits/32)]
 *   packed_dim = 0: out int32 [ceil(rows*bits/32), cols]  (the .contiguous() of the
 *                   transposed view the reference returns, pack_quantized/base.py:109-110) */
int ct_pack_int32(const int8_t* in, int32_t* out, int64_t rows, int64_t cols, int bits, int packed_dim,
                  int device, void* stream);
int ct_unpack_int32(const int32_t* in, int8_t* out, int64_t rows, int64_t cols, int bits, int packed_dim,
                    int device, void* stream);

/* ---- quantize / dequantize / fake_quantize ---------------------------------
 * replace quantization/lifecycle/forward_helpers.py:523-546 (_quantize), :549-572
 * (_dequantize), :180-215 (_quantize_dequantize) together with the strategy reshapes of
 * :62-177 (_process_block, _process_group) and quant_args.py:460-496. */
int ct_quantize(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, const int32_t* g_idx,
                void* q_out, int device, void* stream);
int ct_dequantize(const ct_quant_desc* d, const void* q, const void* scale, const void* zp, const int32_t* g_idx,
                  void* out, int device, void* stream);
int ct_fake_quantize(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, const int32_t* g_idx,
                     void* out, int device, void* stream);

/* ---- attention K / V / Q fake quantization in place of their strided layout ----------------
 * replaces the forward_quantize calls of modeling/kvcache.py (QuantizedKVCache.forward: key and value states) and
 * modeling/attention.py (QuantizedAttentionImpl.forward: query states).  transformers hands those tensors over as the
 * transposed views [B, H, S, D] of [B, S, H, D] projections, which are not contiguous; one launch fake-quantizes every job
 * where it lies, with ct_fake_quantize's per-element arithmetic (bit-identical), and writes `out` with the same strides.
 *   scale / zp: per_head = 0 -> one element (TENSOR); per_head = 1 -> H elements (ATTN_HEAD, scale [H, 1, 1]); zp may be NULL
 * Supported: x_dtype == scale_dtype in {F32, F16, BF16}; CT_Q_INT with 1..8 bits or CT_Q_FLOAT (fp8 e4m3, 8 bits); zp_dtype
 * CT_I8 (or CT_F8E4M3 for CT_Q_FLOAT); stride[3] == 1, D % 8 == 0, x / out 16-byte aligned and the other strides a multiple
 * of 16 bytes; fewer than 2^31 / 8 elements per job; all jobs of a call share dtypes, qtype, bits and the zero-point kind.
 * Anything else returns CT_E_UNSUPPORTED (the caller then runs ct_fake_quantize on contiguous copies).  n is 1 or 2.
 * Enqueue-only, no host synchronisation. */
typedef struct ct_head_job {
    const void* x;
    void* out;
    const void* scale;
    const void* zp;
    int64_t shape[4];       /* B, H, S, D */
    int64_t stride[4];      /* element strides of x and out */
    int32_t per_head;
    int32_t x_dtype, scale_dtype, zp_dtype;   /* zp_dtype CT_NONE without a zero point */
    int32_t qtype, num_bits;
} ct_head_job;
int ct_fake_quantize_heads(int n, const ct_head_job* jobs, int device, void* stream);

/* ---- Walsh-Hadamard transforms of the transform factories ------------------------------------------------
 * replaces HadamardTransform.forward (transform/factory/hadamard.py) -- apply_transform_weight / _multihead_matmul with a dense n x n
 * matrix, then `/ sqrt(n)` and `.to(dtype)` -- for the structured matrices the `hadamard` and `random-hadamard` factories build:
 *     y = x . M / sqrt(n) on every block of n consecutive elements of the last dimension (n = 2^log2_n, 1 <= log2_n <= 15, n | D)
 *     M = H, H[perm][:, perm], diag(sign) . H or (diag(sign) . H)[perm][:, perm]  (H: Sylvester), M^T when `inverse`
 * as an O(n log n) butterfly in `precision` (CT_F32, or CT_F64 for the fused weights), IEEE division by sqrt(n) in that precision,
 * one conversion to `dtype` (fp64 reaches 16-bit dtypes through fp32, as torch's CPU conversion does).  x and out are [B, H, S, D]
 * views with the same element strides (stride[3] == 1; anything else returns CT_E_UNSUPPORTED: run it on a contiguous copy); sign is
 * int8 +-1 [n] or NULL, perm int64 [n] or NULL, both on the device of x.  device = CT_DEVICE_CPU runs the host twin (same butterfly
 * order, same bits) on host pointers.  Enqueue-only on a device.
 * With core_order = K >= 1, n = K . 2^log2_n (0 <= log2_n, n <= 2^15) and H above is (C (x) H_{2^log2_n})^T, C = `core` (K x K, +-1):
 * the matrices the reference's random_hadamard_matrix builds from its table of known Hadamard matrices.  The butterflies run on each
 * 2^log2_n slice, then the K slices are mixed with C (C^T under `inverse`), summing sequentially over the K rows; K additions per
 * element.  CT_E_SHAPE for K outside 1 .. 256 or n above 2^15, CT_E_ARG for a NULL core with K > 1 (K = 1 and NULL: C = [1]).
 * Zero-initialised core fields (core_order 0) leave the forms above unchanged. */
typedef struct ct_hadamard_job {
    const void* x;
    void* out;
    int64_t shape[4];       /* B, H, S, D */
    int64_t stride[4];      /* element strides of x and out */
    const int8_t* sign;
    const int64_t* perm;
    int32_t dtype;          /* x and out: CT_F32 / CT_F16 / CT_BF16 */
    int32_t precision;      /* CT_F32 / CT_F64 */
    int32_t log2_n;
    int32_t inverse;
    const int8_t* core;     /* K x K +-1, row-major, on the device of x; NULL with core_order 0 or 1 */
    int32_t core_order;     /* K: 0 = no core (the forms above) */
} ct_hadamard_job;
int ct_hadamard_transform(const ct_hadamard_job* job, int device, void* stream);

/* ---- fused compressor bodies ------------------------------------------------
 * quantize(dtype=int8) -> pack_to_int32 in one pass (pack_quantized/base.py:96-104) and
 * unpack_from_int32 -> dequantize (pack_quantized/base.py:159-166); the int8
 * intermediate never touches HBM.  packed is int32 [rows, ceil(cols*bits/32)]. */
int ct_quantize_pack_int32(const ct_quant_desc* d, const void* x, const void* scale, const void* zp,
                           const int32_t* g_idx, int32_t* packed, int device, void* stream);
int ct_unpack_dequantize_int32(const ct_quant_desc* d, const int32_t* packed, const void* scale, const void* zp,
                               const int32_t* g_idx, void* out, int device, void* stream);

/* one-pass min-max observer + quantize + pack for GROUP-quantized integer weights (bf16 / fp16, 4- or 8-bit,
 * group_size in {32, 64, 128, 256}): computes scale (x dtype, [rows, cols/group]) and, when zp_out != NULL
 * (asymmetric, d->zp_dtype = CT_I8), the int8 zero point with the reference's observer rule calculate_qparams
 * (quantization/utils/helpers.py:50-137) on the per-group min / max, then quantizes and packs with them in the same
 * pass.  Replaces observer + quantize + pack_to_int32 (SURVEY.md 8(f) rank 1).  Returns CT_E_UNSUPPORTED for
 * anything else: run the observer and ct_quantize_pack_int32 separately. */
int ct_observe_quantize_pack_int32(const ct_quant_desc* d, const void* x, void* scale_out, void* zp_out, int32_t* packed,
                                   int device, void* stream);

/* MSE observer mode of ct_observe_quantize_pack_int32 (and of the NVFP4 and channel observers, below): d->aux != NULL points to this block, in DEVICE memory.  Every group's
 * min / max is shrunk by each p_i, i < steps (lo = T(min * p_i), hi = T(max * p_i) in x's dtype T), calculate_qparams gives the
 * candidate's scale / zero point, and the group's error e(i) = sum |fake_quantize(x) - x|^norm is formed in float32 (d * d for
 * norm == 2, exp2(norm * log2|d|) otherwise).  Step i improves a group when e(i) < min(FLT_MAX, e(0 .. i-1)); the search stops at
 * the first step S ending `patience` steps in which no group of the call improved (steps - 1 if none), and every group is written
 * with the qparams of its last improving step <= S (step 0, the min-max qparams, if none).
 *   shrink[i]  p_i = float32(1 - i / grid), computed on the host
 *   any        bit i set when some group improved at step i; the entry point zeroes it
 *   masks      uint64 [rows * cols / group] scratch: each group's improvement bits (written)
 *   errors     float32 [rows * cols / group, steps] or NULL: every e(i) (written when given)
 * The kernel writes each group's best improving step over all steps; a second launch computes S on the device and rewrites only
 * the groups whose mask has a bit above S.  No host synchronisation.  Same shapes and limits as the min-max mode; anything else
 * (and device = CT_DEVICE_CPU) returns CT_E_UNSUPPORTED.  The block is read on the device and not checked: it must hold a valid
 * `steps` and `masks`.
 * ct_observe_quantize_pack_nvfp4 and ct_observe_quantize_channel take the same block: NVFP4 searches each group of 16's max |x| with
 * the global scale fixed (masks / errors per group of 16); CHANNEL searches each row (masks / errors per row) on rows up to 16384
 * columns.  ct_observe_quantize_block, ct_observe_quantize_mx, ct_observe_tensor / _quantize_tensor and ct_batched's observer ops
 * return CT_E_UNSUPPORTED when d->aux is set. */
#define CT_MSE_MAX_STEPS 64
typedef struct ct_mse_block {
    float shrink[CT_MSE_MAX_STEPS];
    int32_t steps;          /* 1 .. CT_MSE_MAX_STEPS */
    int32_t patience;       /* >= 1 */
    float norm;             /* finite, > 0 */
    int32_t _reserved;
    uint64_t any;
    uint64_t* masks;
    float* errors;
} ct_mse_block;

/* ---- FP4 (E2M1) and MX formats (SURVEY.md 8(f) rank 2) -------------------------
 * cast_to_fp4: quantization/utils/fp4_utils.py:77-98 (x and out share a float dtype).
 * pack_fp4 / unpack_fp4: compressors/nvfp4/helpers.py:108-158 / :162-193 -- x [rows, cols] of VALID fp4 values
 *   <-> uint8 [rows, cols/2], element 2j in the low nibble, bit 3 of a nibble = sign (so -0.0 survives).
 * quantize_pack_fp4 / unpack_dequantize_fp4: the bodies of NVFP4PackedCompressor / MXFP4PackedCompressor
 *   .compress / .decompress (compressors/nvfp4/base.py:73-93, 111-128) in one pass: quantize (d->qtype =
 *   CT_Q_FP4, group 16 with d->global_scale for NVFP4, group 32 for MXFP4) -> nibbles, and nibbles -> dequantize.
 *   For the decompress direction the scale may be given AS STORED: CT_F8E4M3 (NVFP4) or CT_E8M0 (MXFP4).
 * mx_scale_compress / decompress: compressors/mx_utils.py:18-31 / :34-44 (E8M0 encode of float scales; decode to bf16). */
int ct_cast_to_fp4(const void* x, int dtype, void* out, int64_t n, int device, void* stream);
int ct_pack_fp4(const void* x, int dtype, uint8_t* packed, int64_t rows, int64_t cols, int device, void* stream);
int ct_unpack_fp4(const uint8_t* packed, void* out, int out_dtype, int64_t rows, int64_t cols, int device, void* stream);
int ct_quantize_pack_fp4(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, const int32_t* g_idx,
                         uint8_t* packed, int device, void* stream);
/* NVFP4 with the per-group observer fused in: given the tensor's global scale (d->global_scale, from generate_gparam,
 * quantization/utils/helpers.py:308-337) computes every group-of-16 scale with calculate_qparams' rule (helpers.py:74-131: max|x| / 6
 * in x's dtype, x global_scale in float32, clamp, .to(float8_e4m3fn), 0 -> 0.125), stores it AS float8_e4m3fn in scale_out
 * [rows, cols / 16] and quantizes + packs with it in the same pass.  bf16 / fp16, cols % 32 == 0; CT_E_UNSUPPORTED otherwise. */
int ct_observe_quantize_pack_nvfp4(const ct_quant_desc* d, const void* x, void* scale_out_fp8, uint8_t* packed, int device, void* stream);
int ct_unpack_dequantize_fp4(const ct_quant_desc* d, const uint8_t* packed, const void* scale, const void* zp,
                             const int32_t* g_idx, void* out, int device, void* stream);
int ct_mx_scale_compress(const void* scale, int dtype, uint8_t* out, int64_t n, int device, void* stream);
int ct_mx_scale_decompress(const uint8_t* in, void* out_bf16, int64_t n, int device, void* stream);

/* ---- checkpoint-format conversions (SURVEY.md 8(f) rank 3) ----------------------
 * AutoAWQ GEMM -> pack-quantized: entrypoints/convert/converters/autoawq.py:120-128 with :179-262 (unpack_awq, reverse_awq_order,
 * & 15, - 8, .T.contiguous(), pack_to_int32) in one pass.
 *   qweight int32 [K, N/8] (AutoAWQ nibble order)  ->  weight_packed int32 [N, ceil(K/8)]
 *   qzeros  int32 [G, N/8]                         ->  weight_zero_point int32 [N/8, G]  (packed along dim 0, contiguous)
 * FP8 block checkpoints (fp8block_dequantizer.py:111-158) go through ct_dequantize with scale_dtype = CT_F32, BLOCK addressing and
 * out_dtype = CT_BF16 / CT_F16. */
int ct_awq_repack_int4(const int32_t* qweight, int32_t* weight_packed, int64_t K, int64_t N, int device, void* stream);
int ct_awq_repack_zeros_int4(const int32_t* qzeros, int32_t* zero_point_packed, int64_t G, int64_t N, int device, void* stream);

/* one-pass min-max observer + quantize for CHANNEL-wise weight quantization (one scale per row): the same observer rule as
 * above on the row's min / max, then quantize (forward_helpers.py:523-546) and, for d->q_dtype == CT_I32, pack_to_int32.
 *   d->q_dtype = CT_I8 (num_bits 8)      -> int8 codes  [rows, cols]        (W8A8 / INT8 presets)
 *   d->q_dtype = CT_F8E4M3 (CT_Q_FLOAT)  -> fp8 codes   [rows, cols]        (FP8_DYNAMIC preset; symmetric only)
 *   d->q_dtype = CT_I32 (num_bits 4 | 8) -> packed int32 [rows, cols*bits/32] (W4A16 / W8A16 channel-wise)
 * scale_out: x dtype [rows]; zp_out: int8 [rows] or NULL (symmetric).  bf16 / fp16, cols % 8 == 0, cols <= 16384; anything else
 * returns CT_E_UNSUPPORTED. */
int ct_observe_quantize_channel(const ct_quant_desc* d, const void* x, void* scale_out, void* zp_out, void* out, int device, void* stream);

/* ---- per-TENSOR observers without a host round trip (SURVEY.md 8(f) rank 1, TENSOR strategy) -------------
 * ct_observe_tensor: grid-wide min / max of x [rows, cols] (bf16 / fp16 / fp32, byte size % 16 == 0) and, on the device,
 *   kind 0: calculate_qparams (quantization/utils/helpers.py:50-137) for ONE scale per tensor: scale_out = x dtype [1];
 *           zp_out = int8 [1] for asymmetric integer schemes, NULL for symmetric ones (d->qtype / d->num_bits give the range)
 *   kind 1: generate_gparam (helpers.py:308-337): scale_out = float32 [1], the NVFP4 global scale (448 * 6 / max|x|)
 * ct_observe_quantize_tensor: kind 0 followed, in the same call, by ct_quantize (d->q_dtype = CT_I8 / CT_F8E4M3) or
 *   ct_quantize_pack_int32 (d->q_dtype = CT_I32) with the fresh device-resident qparams: what
 *   observer -> calculate_qparams -> quantize(dtype=args.pytorch_dtype()) [-> pack_to_int32] does for the FP8 preset / per-tensor INT
 *   schemes (BASELINE config 3), with no host synchronisation and, for tensors that fit the L2, the second pass served from it.
 * Anything else returns CT_E_UNSUPPORTED. */
int ct_observe_tensor(const ct_quant_desc* d, const void* x, int kind, void* scale_out, void* zp_out, int device, void* stream);
int ct_observe_quantize_tensor(const ct_quant_desc* d, const void* x, void* scale_out, void* zp_out, void* q_out, int device, void* stream);

/* ---- one-pass observe + compress for the BLOCK and MX weight formats ------------------------------------------
 * The memoryless min-max observer and calculate_qparams (quantization/utils/helpers.py:50-137) fused with the compressor body, so the
 * weight x [rows, cols] (bf16 / fp16, contiguous, cols % 8 == 0, x and q_out 16-byte aligned) is read once.
 * ct_observe_quantize_block: FP8_BLOCK.  d: rdiv = block rows, cdiv = block columns (cdiv % 8 == 0), s_row_stride = ceil(cols / cdiv),
 *   qtype CT_Q_FLOAT, q_dtype CT_F8E4M3, scale_dtype = compute_dtype = x_dtype, zp_dtype CT_NONE.  Per block (edge blocks of a ragged shape
 *   over the elements that exist): max(|min|, |max|) / 448 in x's dtype (0 -> eps), then quantize (forward_helpers.py:523-546) with it.
 *     scale_out  x dtype [ceil(rows / rdiv), ceil(cols / cdiv)];  q_out  float8_e4m3fn [rows, cols]
 * ct_observe_quantize_mx: MXFP4 / MXFP8.  d: rdiv = 1, cdiv = 32, s_row_stride = cols / 32 (cols % 32 == 0), scale_dtype CT_E8M0,
 *   compute_dtype = x_dtype, zp_dtype CT_NONE; qtype CT_Q_FP4 (num_bits 4) or CT_Q_FLOAT (num_bits 8, q_dtype CT_F8E4M3).  Per group:
 *   generate_mx_scales / maybe_convert_from_mx_exp of max |x| (quantization/utils/mxfp_utils.py:47-139), quantize, and the layouts of
 *   MXFP4PackedCompressor / MXFP8QuantizationCompressor.compress (compressors/mxfp4/base.py, compressors/mxfp8/base.py):
 *     scale_out  uint8 [rows, cols / 32] (compress_mx_scale, compressors/mx_utils.py:18-31)
 *     q_out      uint8 [rows, cols / 2] (E2M1, element 2j in the low nibble) or float8_e4m3fn [rows, cols]
 * A NaN in a block gives a NaN block scale (and NaN-derived codes).  Anything else -- fp32 x, cols % 8 != 0, a zero point or a global
 * scale, device = CT_DEVICE_CPU -- returns CT_E_UNSUPPORTED: run the observer and ct_quantize / ct_quantize_pack_fp4 separately.
 * Enqueue-only.  ct_batched ops CT_OP_OBSERVE_QUANTIZE_BLOCK / _MX run many weights in one launch. */
int ct_observe_quantize_block(const ct_quant_desc* d, const void* x, void* scale_out, void* q_out, int device, void* stream);
int ct_observe_quantize_mx(const ct_quant_desc* d, const void* x, void* scale_out_e8m0, void* q_out, int device, void* stream);

/* ---- dynamic activation quantization in one pass ---------------------------------------------------
 * replaces compute_dynamic_scales_and_zp (quantization/utils/helpers.py:140-195) followed by fake_quantize (forward.py:148-181), the
 * dynamic branch of forward_quantize (forward.py:292-329): the memoryless min-max observer and calculate_qparams (helpers.py:50-137)
 * fused with quantize-dequantize, so x [rows, cols] (bf16 / fp16, contiguous, cols % 8 == 0, 16-byte aligned) is read once.
 *   out        x's shape and dtype: the fake-quantized values, bit-identical to ct_fake_quantize with the qparams below
 *   scale_out  x's dtype, or float32 when d->global_scale is given (NVFP4: global_scale * scales promotes); zp_out d->zp_dtype
 *              (CT_I8, CT_F8E4M3 or CT_U8, zeros for a symmetric scheme); one element per row / group / tensor
 * The strategy is read from the scale addressing of d:
 *   TOKEN   rdiv = 1, s_row_stride = 1, cdiv = CT_DIV_INF: one scale per row (the caller folds every dim after the first two into cols),
 *           cols <= 32768; int (asymmetric: int8 zero point) or fp8
 *   GROUP   rdiv = 1, cdiv = group size in {16, 32, 64, 128} dividing cols, s_row_stride = cols / cdiv (also TENSOR_GROUP)
 *   TENSOR  rdiv = cdiv = CT_DIV_INF: ct_observe_tensor (kind 0), then ct_fake_quantize on the device-resident scale
 * asymmetric: args.symmetric is False.  scale_dtype_arg: args.scale_dtype as CT_NONE, CT_F8E4M3 (clamp to +-448 and round through
 * float8_e4m3fn, optionally after d->global_scale, a DEVICE pointer to one float32) or CT_E8M0 (uint8: the MX exponent scales of
 * generate_mx_scales / maybe_convert_from_mx_exp, quantization/utils/mxfp_utils.py:47-139, group 32).  d->compute_dtype / d->seff_dtype
 * are those ct_fake_quantize would get for the returned scale.  Anything else, and device = CT_DEVICE_CPU, returns CT_E_UNSUPPORTED:
 * run the observer and ct_fake_quantize separately.  Enqueue-only, no host synchronisation (capturable into a CUDA graph). */
int ct_dynamic_fake_quantize(const ct_quant_desc* d, int asymmetric, int scale_dtype_arg, const void* x, void* out, void* scale_out,
                             void* zp_out, int device, void* stream);

/* ---- multi-tensor (whole-model) launches -------------------------------------
 * One persistent launch over `n` independent tensors: the body of the module loop of
 * ModelCompressor.compress_model / decompress_model
 * (compressors/model_compressors/model_compressor.py:153-172, :183-207).
 * descs / pointer tables are HOST arrays of length n; tensor i uses descs[i], x[i], ...
 * Enqueue-only like every device entry point, and capturable into a CUDA graph: when `stream` is being captured the job table of
 * a multi-tensor launch travels as kernel parameters (one small upload kernel per 32 tensors) instead of a host-to-device copy from
 * pageable memory, so a whole-model call can be captured once and replayed on the same buffers (tests/test_gpu_robust.py). */
typedef enum ct_batch_op_t {
    CT_OP_QUANTIZE_PACK = 0,      /* in x        -> out packed int32 */
    CT_OP_UNPACK_DEQUANTIZE = 1,  /* in packed   -> out float */
    CT_OP_QUANTIZE = 2,           /* in x        -> out q (int8 / fp8) */
    CT_OP_DEQUANTIZE = 3,         /* in q        -> out float */
    CT_OP_FAKE_QUANTIZE = 4,      /* in x        -> out float */
    CT_OP_PACK_INT32 = 5,         /* in int8 codes -> out packed int32 (packed_dim 1; desc: rows, cols, num_bits; no scale) */
    CT_OP_UNPACK_INT32 = 6,       /* in packed   -> out int8 codes */
    CT_OP_OBSERVE_QUANTIZE_PACK = 7, /* in x     -> out packed int32; scale[i] / zp[i] are OUTPUTS (see ct_observe_quantize_pack_int32) */
    CT_OP_QUANTIZE_PACK_FP4 = 8,  /* in x        -> out uint8 nibbles (ct_quantize_pack_fp4) */
    CT_OP_UNPACK_DEQUANTIZE_FP4 = 9, /* in nibbles -> out float (ct_unpack_dequantize_fp4) */
    CT_OP_OBSERVE_QUANTIZE_PACK_FP4 = 10, /* in x -> out nibbles; scale[i] (float8_e4m3fn) is an OUTPUT (ct_observe_quantize_pack_nvfp4) */
    CT_OP_SPARSE24_QUANTIZE_PACK = 11,    /* in x       -> out packed int32 [rows, cols/16] + descs[i].aux = bitmask OUT (ct_sparse24_quantize_pack_int4) */
    CT_OP_SPARSE24_UNPACK_DEQUANTIZE = 12, /* in packed  -> out float; descs[i].aux = bitmask IN (ct_sparse24_unpack_dequantize_int4) */
    CT_OP_OBSERVE_QUANTIZE_BLOCK = 13,     /* in x -> out fp8 codes; scale[i] (x dtype, one per block) is an OUTPUT (ct_observe_quantize_block) */
    CT_OP_OBSERVE_QUANTIZE_MX = 14         /* in x -> out nibbles / fp8 codes; scale[i] (E8M0 uint8) is an OUTPUT (ct_observe_quantize_mx) */
} ct_batch_op_t;
int ct_batched(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale,
               const void* const* zp, void* const* out, int device, void* stream);

/* ---- bitmasks and sparse formats ----------------------------------------------
 * pack_bitmasks / unpack_bitmasks: utils/helpers.py:306-343 (numpy.packbits little).
 * sparse24 / bitmask compress+decompress: the Sparse24BitMask / Bitmask compressors named
 * by CompressionFormat.sparse_24_bitmask / sparse_bitmask (config/base.py:17-18); they are
 * absent from the reference snapshot, so these follow the restated format of
 * oracle/ct_oracle.c ("parity unpinned"). */
int ct_pack_bitmasks(const uint8_t* bytemask, uint8_t* packed, int64_t rows, int64_t cols, int device, void* stream);
int ct_unpack_bitmasks(const uint8_t* packed, uint8_t* bytemask, int64_t rows, int64_t cols, int device, void* stream);
int ct_sparse24_compress(const void* x, int dtype, void* values, uint8_t* bitmask, int64_t rows, int64_t cols,
                         int device, void* stream);
int ct_sparse24_decompress(const void* values, int dtype, const uint8_t* bitmask, void* out, int64_t rows,
                           int64_t cols, int device, void* stream);
/* unstructured: two-phase.  count writes row_offsets[rows] (exclusive scan of per-row nnz) and
 * *nnz_out (device int64); compress then scatters values.  workspace from ct_bitmask_workspace_bytes. */
int64_t ct_bitmask_workspace_bytes(int64_t rows, int64_t cols);
int ct_bitmask_count(const void* x, int dtype, uint8_t* bitmask, int64_t* row_offsets, int64_t* nnz_out,
                     void* workspace, int64_t rows, int64_t cols, int device, void* stream);
int ct_bitmask_compress(const void* x, int dtype, const uint8_t* bitmask, const int64_t* row_offsets, void* values,
                        int64_t rows, int64_t cols, int device, void* stream);
int ct_bitmask_decompress(const void* values, int dtype, const uint8_t* bitmask, const int64_t* row_offsets,
                          void* out, int64_t rows, int64_t cols, int device, void* stream);
/* The same compression in ONE call without a host round trip (BitmaskCompressor of CompressionFormat.sparse_bitmask, config/base.py:17;
 * mask bit order of utils/helpers.py:306-317): `values` is a caller buffer of CAPACITY rows * cols elements of which the first *nnz_out
 * (device int64) are written, row_offsets [rows] and bitmask [rows, ceil(cols/8)] as above.  bf16 / fp16 tensors with cols % 8 == 0
 * are read exactly once (per-tile counts combined by a decoupled look-back scan inside the kernel); other dtypes / shapes run the
 * two-phase kernels above on a stream-ordered workspace.  Enqueue-only.
 * (ct_bitmask_decompress is one pass either way: with row_offsets every row knows where its values start; row_offsets = NULL is
 * accepted for bf16 / fp16, cols % 8 == 0: the scan is then recomputed from the mask popcounts with the same look-back.) */
int ct_bitmask_compress_onepass(const void* x, int dtype, void* values, uint8_t* bitmask, int64_t* row_offsets, int64_t* nnz_out,
                                int64_t rows, int64_t cols, int device, void* stream);

/* BASELINE config 4, "Sparse24BitMask + int4": the composition of the 2:4 bitmask format above with pack-quantized, fused.
 *   compress  : per quad of x keep the 2 of largest |x| (ties: lower column), quantize the KEPT values with the scale / zero point of
 *               their original column (forward_helpers.py:523-546), pack the 4-bit codes [rows, cols/2] with pack_to_int32's bitstream
 *               (pack_quantized/helpers.py:20-101) -> packed int32 [rows, cols/16]; bitmask = pack_bitmasks(mask) (utils/helpers.py:306-317)
 *   decompress: codes back to their columns, dequantized (forward_helpers.py:549-572) to d->out_dtype; dropped columns are +0
 * d as for ct_quantize_pack_int32 / ct_unpack_dequantize_int32 (num_bits = 4, CT_Q_INT).  The selection rule and the composition are
 * restated ("parity unpinned": the compressor pair is absent from the reference snapshot).  Fast kernels: bf16 / fp16, cols % 32 == 0,
 * scales in the weight dtype with full rows (group % 32 == 0, channel, tensor), zero point absent or int8, 16-byte aligned tensors;
 * anything else returns CT_E_UNSUPPORTED (the Python layer then composes the unfused kernels). */
int ct_sparse24_quantize_pack_int4(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, int32_t* packed,
                                   uint8_t* bitmask, int device, void* stream);
int ct_sparse24_unpack_dequantize_int4(const ct_quant_desc* d, const int32_t* packed, const uint8_t* bitmask, const void* scale,
                                       const void* zp, void* out, int device, void* stream);

/* 2:4 "semi-structured" values + metadata in the CUTLASS / marlin-24 layout: replaces
 * utils/semi_structured_conversions.py:66-197 (sparse_semi_structured_from_dense_cutlass) and
 * :204-298 (sparse_semi_structured_to_dense_cutlass).  dense [m, k] -> sparse [m, k/2] + meta
 * (int16 [m, k/16] for 2-byte data, int32 [m, k/32] for int8 data, int16 [m, k/8] for fp32 1:2),
 * meta reordered for ColumnMajorInterleaved<2> (:33-60).  m % 64 == 0.  to_dense takes the number
 * of SPARSE columns k and writes dense [m, 2k]. */
int ct_semi_structured_from_dense(const void* dense, int dtype, void* sparse, void* meta, int64_t m, int64_t k,
                                  int device, void* stream);
int ct_semi_structured_to_dense(const void* sparse, int dtype, const void* meta, void* dense, int64_t m, int64_t k,
                                int device, void* stream);

/* ---- host-buffer entry point (what a CPU-resident caller of the reference API hits) ----
 * Same semantics as ct_batched, but every pointer is a HOST pointer (pinned memory gives full PCIe rate; pageable works),
 * d->global_scale of the FP4 ops included.  n == 1 for one large CPU tensor; a CPU-resident model (the body of
 * ModelCompressor.compress_model / decompress_model for state dicts that live in host memory) passes all its tensors.
 * Rows are streamed through the device in chunks, and the chunks of all tensors form one queue through 4 staging slots
 * (H2D copy / kernel / D2H copy on a stream each), so the PCIe copy engines do not drain between tensors.  Blocking, on
 * error too: no copy from or into the caller's buffers is left in flight.  Serialises per device on its staging buffers. */
int ct_host_run_many(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale,
                     const void* const* zp, void* const* out, int device);

/* ---- self tests (device-side exhaustive checks used by tests/) ----------------- */
/* compares the fast reciprocal-based quotient rounding used by the kernels with IEEE
 * division for every (x, s) pair of 16-bit patterns of `dtype` (CT_BF16 or CT_F16) with
 * s restricted to the fast-path range; writes the mismatch count to *mismatches (host). */
int ct_selftest_division(int dtype, uint64_t* mismatches, int device);
/* NVFP4 fast path: the E2M1 code obtained through the reciprocal + one-residual-step quotient must equal the code of the
 * IEEE quotient for every 16-bit x of `dtype` and every float32 scale significand at binary exponent `scale_exponent`
 * (within [-100, 9]: the kernels use the shortcut for |scale / global_scale| in [2^-100, 2^10]).
 * mode 1: the float32 value of  scale / global_scale  for every 16-bit scale with |scale| in [2^-40, 2^14] and every global-scale
 * significand at exponent `scale_exponent` (within [-60, 59]) must equal div.rn bit for bit (used by the decompress kernel). */
int ct_selftest_fp4_division(int dtype, int scale_exponent, int mode, uint64_t* mismatches, int device);

#ifdef __cplusplus
}
#endif
#endif /* CT_B200_H */

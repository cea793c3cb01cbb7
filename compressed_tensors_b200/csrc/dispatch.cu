// dispatch.cu -- decides, per tensor, between the streaming fast path and the generic kernels,
// builds the job tables for multi-tensor launches, and implements the C ABI compute entry points.
#include <cstring>
#include <vector>

#include "engine.h"

namespace ctb {

static bool is_inf(int64_t v) { return v == CT_DIV_INF; }

// flat scale divisor D (elements per scale element) if scale index == flat_index / D
static bool flat_divisor(const ct_quant_desc& d, int64_t& D) {
    if (is_inf(d.rdiv) && is_inf(d.cdiv)) { D = CT_DIV_INF; return true; }          // TENSOR
    if (d.rdiv == 1 && d.s_row_stride == 1 && (is_inf(d.cdiv) || d.cdiv >= d.cols)) {  // CHANNEL / one group per row
        D = d.cols;
        return true;
    }
    if (d.rdiv == 1 && !is_inf(d.cdiv) && d.cdiv > 0 && d.cols % d.cdiv == 0 && d.s_row_stride == d.cols / d.cdiv) {
        D = d.cdiv;                                                                  // GROUP, full rows of scales
        return true;
    }
    return false;
}

static int validate_desc(const ct_quant_desc* d) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    if (d->rows < 0 || d->cols < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    if (d->qtype == CT_Q_INT && (d->num_bits < 1 || d->num_bits > 8)) {
        set_error("num_bits %d outside [1, 8]", d->num_bits);
        return CT_E_BITS;
    }
    if (d->qtype == CT_Q_FLOAT && d->num_bits != 8) { set_error("fp8 quantization needs num_bits == 8"); return CT_E_BITS; }
    if (d->qtype == CT_Q_FP4 && d->num_bits != 4) { set_error("fp4 quantization needs num_bits == 4"); return CT_E_BITS; }
    if (d->qtype != CT_Q_INT && d->qtype != CT_Q_FLOAT && d->qtype != CT_Q_FP4) { set_error("bad qtype %d", d->qtype); return CT_E_ARG; }
    if (d->global_scale && !is_float_dt(d->seff_dtype)) { set_error("seff_dtype must be a float dtype when a global scale is given"); return CT_E_DTYPE; }
    if (d->rdiv <= 0 || d->cdiv <= 0) { set_error("rdiv/cdiv must be positive"); return CT_E_SHAPE; }
    return CT_OK;
}

struct Plan {
    StreamKernel k;   // k.launch == nullptr: the tensor takes the generic kernels
    Job job;          // tile_begin/end filled by the caller
    Common cm;
};

// The streaming plan of kernel k (none: the generic plan) over n elements in chunks of `chunk`, D elements per scale element;
// `two_d`: the 2-D scale addressing of d (BLOCK strategy, one-row group scales).
static Plan fast_plan(StreamKernel k, const Common& cm, const void* in, const void* scale, const void* zp, void* out, const void* aux,
                      int64_t n, int64_t chunk, int64_t D, const ct_quant_desc* two_d = nullptr) {
    Plan p{};
    if (!k.launch) return p;
    p.k = k;
    p.cm = cm;
    p.job.in = reinterpret_cast<const uint8_t*>(in);
    p.job.scale = scale;
    p.job.zp = zp;
    p.job.out = reinterpret_cast<uint8_t*>(out);
    p.job.aux = aux;
    p.job.n_chunks = (uint32_t)(n / chunk);
    p.job.dc = make_fastdiv(is_inf(D) ? (uint64_t)0x7FFFFFFFull : (uint64_t)(D / chunk));
    if (two_d) {
        p.job.cpr = make_fastdiv((uint64_t)(two_d->cols / chunk));
        p.job.rd = make_fastdiv(is_inf(two_d->rdiv) ? (uint64_t)0x7FFFFFFFull : (uint64_t)two_d->rdiv);
        p.job.srs = (uint32_t)two_d->s_row_stride;
    }
    return p;
}

static uint32_t bits_of(int dt, float v) {
    // v as a 16-bit float pattern duplicated in both halves (host-side conversion, RNE; v is exact)
    if (dt == CT_BF16) {
        uint32_t u; memcpy(&u, &v, 4);
        uint32_t h = u >> 16;
        return h | (h << 16);
    }
    if (dt == CT_F16) {
        __half hv = __float2half_rn(v);
        uint16_t h; memcpy(&h, &hv, 2);
        return (uint32_t)h | ((uint32_t)h << 16);
    }
    return 0;
}

Common make_common(int p_dt, int qtype, int bits) {
    Common cm;
    if (qtype == CT_Q_INT) {
        const float r = (float)(1 << bits);
        cm.qmax = r / 2 - 1;
        cm.qmin = -r / 2;
    } else if (qtype == CT_Q_FP4) {
        cm.qmax = 6.f;
        cm.qmin = -6.f;
    } else {
        cm.qmax = 448.f;
        cm.qmin = -448.f;
    }
    cm.qmin2 = bits_of(p_dt, cm.qmin);
    cm.qmax2 = bits_of(p_dt, cm.qmax);
    cm.bits = bits;
    return cm;
}

// Try to express (op, desc) as a streaming job.  in/out are the streamed tensors of the op.
static Plan plan_one(int op, const ct_quant_desc& d, const void* in, const void* scale, const void* zp,
                     const int32_t* g_idx, void* out) {
    const int64_t n = d.rows * d.cols;
    if (g_idx || n == 0 || n % 8 != 0 || (n / 8) >= 0x7fffffffLL) return {};
    if (!aligned16(in) || !aligned16(out)) return {};
    if (d.global_scale || d.qtype == CT_Q_FP4) return {};   // two-level scales / FP4 rounding: fp4 ops have their own plans (below), the rest is generic
    int64_t D;
    bool two_d = false;
    if (!flat_divisor(d, D)) {
        // 2-D scale addressing (BLOCK strategy, one-row group scales): chunks must not straddle rows or column blocks
        if (op == CT_OP_OBSERVE_QUANTIZE_PACK || d.cols % 8 != 0 || (d.cols / 8) >= 0x7fffffffLL) return {};
        if (!is_inf(d.cdiv) && d.cdiv % 8 != 0) return {};
        if (d.s_row_stride < 0 || d.s_row_stride >= 0x7fffffffLL) return {};
        two_d = true;
        D = d.cdiv;
    }
    if (!is_inf(D) && D % 8 != 0) return {};
    // zero point: int8 everywhere; float8_e4m3fn (what the FP8 presets register) on the fp8 quantize / dequantize / fake_quantize kernels
    const bool fp8_op = (op == CT_OP_QUANTIZE && d.qtype == CT_Q_FLOAT) || (op == CT_OP_FAKE_QUANTIZE && d.qtype == CT_Q_FLOAT) ||
                        (op == CT_OP_DEQUANTIZE && d.q_dtype == CT_F8E4M3 && d.out_dtype == d.scale_dtype);
    if (zp && d.zp_dtype != CT_I8 && !(d.zp_dtype == CT_F8E4M3 && fp8_op)) return {};
    const int zpk = zp ? (d.zp_dtype == CT_I8 ? 1 : 2) : 0;
    // the largest thread unit (chunks) the layout admits: a unit must see one scale and must not straddle a row or the end of the tensor
    int max_unit = 4;
    while (max_unit > 1 && !((is_inf(D) || (D / 8) % max_unit == 0) && (!two_d || (d.cols / 8) % max_unit == 0) && (n / 8) % max_unit == 0))
        max_unit /= 2;

    int p_dt, in_bytes_per_chunk;
    StreamKernel k;
    switch (op) {
    case CT_OP_QUANTIZE_PACK:
        if (d.qtype != CT_Q_INT || (d.num_bits != 4 && d.num_bits != 8)) return {};
        if ((d.cols * d.num_bits) % 32 != 0) return {};
        if (d.x_dtype != d.scale_dtype || d.x_dtype != d.compute_dtype || !is_float_dt(d.x_dtype)) return {};
        p_dt = d.x_dtype; in_bytes_per_chunk = 8 * dt_size(p_dt);
        k = quantpack_kernel(p_dt, d.num_bits, zpk, max_unit);
        break;
    case CT_OP_OBSERVE_QUANTIZE_PACK: {
        // fused observer: `scale` / `zp` are OUTPUTS; group strategy only, a group = 32 * {1,2,4,8} elements
        if (d.qtype != CT_Q_INT || (d.num_bits != 4 && d.num_bits != 8)) return {};
        if ((d.cols * d.num_bits) % 32 != 0 || n % 32 != 0) return {};
        if (d.x_dtype != d.scale_dtype || d.x_dtype != d.compute_dtype || (d.x_dtype != CT_BF16 && d.x_dtype != CT_F16)) return {};
        if (is_inf(D) || D != d.cdiv || D % 32 != 0) return {};
        p_dt = d.x_dtype; in_bytes_per_chunk = 16;
        k = observe_kernel(p_dt, d.num_bits, zp != nullptr, (int)(D / 32), d.aux != nullptr);
        break;
    }
    case CT_OP_UNPACK_DEQUANTIZE:
        if (d.num_bits != 4 && d.num_bits != 8) return {};
        if ((d.cols * d.num_bits) % 32 != 0) return {};
        if (d.out_dtype != d.scale_dtype || !is_float_dt(d.out_dtype)) return {};
        p_dt = d.scale_dtype; in_bytes_per_chunk = d.num_bits;
        k = unpackdeq_kernel(p_dt, d.num_bits, zpk);
        break;
    case CT_OP_QUANTIZE:
        if (d.x_dtype != d.scale_dtype || d.x_dtype != d.compute_dtype || !is_float_dt(d.x_dtype)) return {};
        if (d.qtype == CT_Q_INT && d.q_dtype != CT_I8) return {};
        if (d.qtype == CT_Q_FLOAT && d.q_dtype != CT_F8E4M3) return {};
        p_dt = d.x_dtype; in_bytes_per_chunk = 8 * dt_size(p_dt);
        k = quant_kernel(p_dt, d.qtype == CT_Q_FLOAT, zpk, max_unit);
        break;
    case CT_OP_DEQUANTIZE:
        if (d.scale_dtype == CT_F32 && (d.out_dtype == CT_BF16 || d.out_dtype == CT_F16) && d.q_dtype == CT_F8E4M3 && !zp) {
            // (q.to(float32) * scale).to(T): fp8 block checkpoints
            p_dt = d.out_dtype; in_bytes_per_chunk = 8;
            k = dequant_kernel(p_dt, true, 0, true);
            break;
        }
        if (d.out_dtype != d.scale_dtype || !is_float_dt(d.out_dtype)) return {};
        if (d.q_dtype != CT_I8 && d.q_dtype != CT_F8E4M3) return {};
        p_dt = d.scale_dtype; in_bytes_per_chunk = 8;
        k = dequant_kernel(p_dt, d.q_dtype == CT_F8E4M3, zpk, false);
        break;
    case CT_OP_FAKE_QUANTIZE:
        if (d.x_dtype != d.scale_dtype || d.x_dtype != d.compute_dtype || d.out_dtype != d.x_dtype || !is_float_dt(d.x_dtype)) return {};
        p_dt = d.x_dtype; in_bytes_per_chunk = 8 * dt_size(p_dt);
        k = fake_kernel(p_dt, d.qtype, d.num_bits, zpk);
        break;
    default:
        return {};
    }
    // a partial last tile must still be a multiple of 16 bytes for the bulk copy
    if (((n / 8) * in_bytes_per_chunk) % 16 != 0) return {};
    return fast_plan(k, make_common(p_dt, d.qtype, d.num_bits), in, scale, zp, out, op == CT_OP_OBSERVE_QUANTIZE_PACK ? d.aux : nullptr, n, 8, D,
                     two_d ? &d : nullptr);
}

// FP4 fused ops as streaming jobs (fast_fp4.cu).  Both need GROUP strategy with full rows of scales and no g_idx.
//   quantize+pack: x bf16 / fp16, units of 32 elements inside a row;  NVFP4 = group 16 + global scale (fp32 arithmetic, scale in
//                  x's dtype or float32, zero point absent or fp8), MX-style = group % 32 == 0, scale and arithmetic in x's dtype
//   unpack+dequantize: out bf16 / fp16, units of 16 elements; scale in the out dtype or as stored (fp8 / E8M0)
static Plan plan_fp4(int op, const ct_quant_desc& d, const void* in, const void* scale, const void* zp,
                     const int32_t* g_idx, void* out) {
    const int64_t n = d.rows * d.cols;
    int64_t D;
    if (g_idx || n == 0 || (n / 8) >= 0x7fffffffLL || !aligned16(in) || !aligned16(out)) return {};
    if (!flat_divisor(d, D) || is_inf(D) || d.qtype != CT_Q_FP4) return {};
    StreamKernel k;
    int p_dt;
    if (op == CT_OP_OBSERVE_QUANTIZE_PACK_FP4) {
        // scale (float8_e4m3fn [rows, cols / 16]) is an OUTPUT; NVFP4 only: group 16, float32 global scale given, no zero point
        if ((d.x_dtype != CT_BF16 && d.x_dtype != CT_F16) || d.cols % 32 != 0 || D != 16 || !d.global_scale || zp) return {};
        if ((reinterpret_cast<uintptr_t>(scale) & 1u) != 0) return {};
        p_dt = d.x_dtype;
        k = fp4_observe_kernel(p_dt, d.aux != nullptr);
        zp = d.aux;   // the MSE mode's ct_mse_block (or none): this op has no zero point
    } else if (op == CT_OP_QUANTIZE_PACK_FP4) {
        if (d.x_dtype != CT_BF16 && d.x_dtype != CT_F16) return {};
        if (d.cols % 32 != 0 || !aligned16(scale) ) return {};
        if (d.global_scale ? (D != 16 || d.seff_dtype != CT_F32 || d.compute_dtype != CT_F32) : (D % 32 != 0 || d.compute_dtype != d.x_dtype)) return {};
        p_dt = d.x_dtype;
        k = fp4_quantpack_kernel(p_dt, d.global_scale != nullptr, d.scale_dtype, zp ? d.zp_dtype : CT_NONE);
    } else {
        if (d.out_dtype != CT_BF16 && d.out_dtype != CT_F16) return {};
        if (zp || d.cols % 8 != 0 || D % 8 != 0) return {};
        if (d.global_scale ? d.seff_dtype != CT_F32 : (d.seff_dtype != d.out_dtype && d.scale_dtype != d.out_dtype)) return {};
        if (((n / 8) * 4) % 16 != 0) return {};   // a partial last tile must still be a multiple of 16 bytes for the bulk copy
        p_dt = d.out_dtype;
        k = fp4_unpackdeq_kernel(p_dt, d.scale_dtype);
    }
    return fast_plan(k, make_common(p_dt, CT_Q_FP4, 4), in, scale, zp, out, d.global_scale, n, 8, D);
}

// fused 2:4 select + int4 (fast_sparse24q.cu).  compress: chunk = 8 dense elements, unit = 4 chunks; decompress: chunk = 16 dense
// elements (4 bytes of nibbles) = one unit.  Full rows of scales only (flat scale index), cols % 32 == 0.
static Plan plan_s24(int op, const ct_quant_desc& d, const void* in, const void* scale, const void* zp, const int32_t* g_idx, void* out) {
    const int64_t n = d.rows * d.cols;
    int64_t D;
    if (g_idx || n == 0 || n % 64 != 0 || d.cols % 32 != 0 || (n / 8) >= 0x7fffffffLL || !aligned16(in) || !aligned16(out)) return {};
    if (!d.aux || (reinterpret_cast<uintptr_t>(d.aux) & 3u) != 0 || d.global_scale || d.qtype != CT_Q_INT || d.num_bits != 4) return {};
    if (!flat_divisor(d, D) || (!is_inf(D) && D % 32 != 0)) return {};
    if (zp && d.zp_dtype != CT_I8) return {};
    const bool comp = (op == CT_OP_SPARSE24_QUANTIZE_PACK);
    if (!comp && (reinterpret_cast<uintptr_t>(out) & 31u) != 0) return {};   // the expansion writes with 256-bit stores
    const int p_dt = comp ? d.x_dtype : d.out_dtype;
    if (p_dt != CT_BF16 && p_dt != CT_F16) return {};
    if (d.scale_dtype != p_dt || (comp && d.compute_dtype != p_dt)) return {};
    return fast_plan(sparse24q_kernel(comp, p_dt, zp ? 1 : 0), make_common(p_dt, CT_Q_INT, 4), in, scale, zp, out, d.aux, n, comp ? 8 : 16, D);
}

// standalone pack / unpack (packed_dim 1) as a streaming job; for these ops a chunk is 16 codes
static Plan plan_bits(bool pack, int64_t rows, int64_t cols, int bits, const void* in, void* out) {
    const int64_t n = rows * cols;
    const int in_bytes = pack ? 16 : 2 * bits;
    const int unit = (pack && bits == 4) ? 32 : 16;   // 4-bit packing works on units of 2 chunks
    if (!(bits == 4 || bits == 8) || (cols * bits) % 32 != 0 || n == 0 || n % unit != 0 || (n / 16) >= 0x7fffffffLL) return {};
    if (!aligned16(in) || !aligned16(out) || ((n / 16) * in_bytes) % 16 != 0) return {};
    return fast_plan(bits_kernel(pack, bits), make_common(CT_F32, CT_Q_INT, bits), in, nullptr, nullptr, out, nullptr, n, 16, CT_DIV_INF);
}

static int run_generic(int op, const ct_quant_desc& d, const void* in, const void* scale, const void* zp,
                       const int32_t* g_idx, void* out, cudaStream_t st) {
    switch (op) {
    case CT_OP_QUANTIZE_PACK:
        if (d.qtype != CT_Q_INT) { set_error("quantize_pack needs integer quantization"); return CT_E_DTYPE; }
        return launch_generic_quantpack(d, in, scale, zp, g_idx, reinterpret_cast<int32_t*>(out), st);
    case CT_OP_UNPACK_DEQUANTIZE:
        return launch_generic_unpackdeq(d, reinterpret_cast<const int32_t*>(in), scale, zp, g_idx, out, st);
    case CT_OP_QUANTIZE: return launch_generic_quant(G_QUANTIZE, d, in, scale, zp, g_idx, out, st);
    case CT_OP_DEQUANTIZE: return launch_generic_quant(G_DEQUANTIZE, d, in, scale, zp, g_idx, out, st);
    case CT_OP_FAKE_QUANTIZE: return launch_generic_quant(G_FAKE, d, in, scale, zp, g_idx, out, st);
    case CT_OP_QUANTIZE_PACK_FP4:
        return launch_generic_quantpack_fp4(d, in, scale, zp, g_idx, reinterpret_cast<uint8_t*>(out), st);
    case CT_OP_UNPACK_DEQUANTIZE_FP4:
        return launch_generic_unpackdeq_fp4(d, reinterpret_cast<const uint8_t*>(in), scale, zp, g_idx, out, st);
    case CT_OP_OBSERVE_QUANTIZE_PACK_FP4:
        set_error("fused NVFP4 observe+quantize+pack supports bf16 / fp16 weights, group_size 16 with full rows of scales, cols %% 32 == 0, "
                  "a float32 global scale, 16-byte aligned contiguous tensors; run the observer and quantize_pack_fp4 separately otherwise");
        return CT_E_UNSUPPORTED;
    case CT_OP_SPARSE24_QUANTIZE_PACK:
    case CT_OP_SPARSE24_UNPACK_DEQUANTIZE:
        set_error("fused 2:4 + int4 supports bf16 / fp16 weights, 4-bit integer codes, cols %% 32 == 0, rows * cols %% 64 == 0, scales in the weight dtype "
                  "with full rows (group %% 32 == 0, channel, tensor), zero point absent or int8, 16-byte aligned contiguous tensors and a "
                  "4-byte aligned bitmask; compose sparse24 + quantize + pack separately otherwise");
        return CT_E_UNSUPPORTED;
    case CT_OP_OBSERVE_QUANTIZE_PACK:
        set_error("fused observe+quantize+pack supports bf16/fp16 group quantization with group_size in {32,64,128,256}, "
                  "4- or 8-bit codes, 16-byte aligned contiguous tensors; run the observer and quantize_pack separately otherwise");
        return CT_E_UNSUPPORTED;
    }
    set_error("unknown op %d", op);
    return CT_E_ARG;
}

static int check_dtypes(int op, const ct_quant_desc& d, bool has_zp) {
    const bool quantizing = (op == CT_OP_QUANTIZE_PACK || op == CT_OP_QUANTIZE || op == CT_OP_FAKE_QUANTIZE || op == CT_OP_OBSERVE_QUANTIZE_PACK ||
                             op == CT_OP_QUANTIZE_PACK_FP4 || op == CT_OP_OBSERVE_QUANTIZE_PACK_FP4 || op == CT_OP_SPARSE24_QUANTIZE_PACK);
    const bool fp4_op = (op == CT_OP_QUANTIZE_PACK_FP4 || op == CT_OP_UNPACK_DEQUANTIZE_FP4 || op == CT_OP_OBSERVE_QUANTIZE_PACK_FP4);
    if (op == CT_OP_OBSERVE_QUANTIZE_PACK_FP4) {   // the scale is produced, as float8_e4m3fn
        if (d.qtype != CT_Q_FP4 || d.cols % 2 != 0) { set_error("fp4 ops need qtype fp4 and an even number of columns"); return CT_E_DTYPE; }
        if (!is_float_dt(d.x_dtype)) { set_error("x dtype must be float"); return CT_E_DTYPE; }
        return CT_OK;
    }
    if (fp4_op && (d.qtype != CT_Q_FP4 || d.cols % 2 != 0)) { set_error("fp4 ops need qtype fp4 and an even number of columns"); return d.cols % 2 ? CT_E_SHAPE : CT_E_DTYPE; }
    const bool stored_scale = (op == CT_OP_UNPACK_DEQUANTIZE_FP4 && (d.scale_dtype == CT_F8E4M3 || d.scale_dtype == CT_E8M0));
    if (stored_scale && !is_float_dt(d.seff_dtype)) { set_error("stored (fp8 / E8M0) scales need seff_dtype = the float dtype they decode to"); return CT_E_DTYPE; }
    if (!is_float_dt(d.scale_dtype) && !stored_scale) { set_error("scale dtype %d is not a float dtype", d.scale_dtype); return CT_E_DTYPE; }
    if (quantizing && (!is_float_dt(d.x_dtype) || !is_float_dt(d.compute_dtype))) {
        set_error("x / compute dtype must be float (got %d / %d)", d.x_dtype, d.compute_dtype);
        return CT_E_DTYPE;
    }
    if (has_zp && dt_size(d.zp_dtype) == 0) { set_error("bad zero-point dtype %d", d.zp_dtype); return CT_E_DTYPE; }
    if ((op == CT_OP_DEQUANTIZE || op == CT_OP_UNPACK_DEQUANTIZE || op == CT_OP_FAKE_QUANTIZE || op == CT_OP_UNPACK_DEQUANTIZE_FP4 ||
         op == CT_OP_SPARSE24_UNPACK_DEQUANTIZE) && !is_float_dt(d.out_dtype)) {
        set_error("output dtype %d is not a float dtype", d.out_dtype);
        return CT_E_DTYPE;
    }
    if (op == CT_OP_QUANTIZE && dt_size(d.q_dtype) == 0) { set_error("bad q dtype"); return CT_E_DTYPE; }
    if (op == CT_OP_DEQUANTIZE && dt_size(d.q_dtype) == 0) { set_error("bad q dtype"); return CT_E_DTYPE; }
    return CT_OK;
}

int run_batched(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale,
                const void* const* zp, const int32_t* const* g_idx, void* const* out, int device, cudaStream_t stream) {
    if (op == CT_OP_OBSERVE_QUANTIZE_BLOCK || op == CT_OP_OBSERVE_QUANTIZE_MX) return run_observe_block_mx(op, n, descs, in, scale, out, device, stream);
    const bool bits_op = (op == CT_OP_PACK_INT32 || op == CT_OP_UNPACK_INT32);
    if (n < 0 || (n > 0 && (!descs || !in || (!scale && !bits_op) || !out))) { set_error("null table"); return CT_E_ARG; }
    if (device == CT_DEVICE_CPU) {
        // explicit CPU twins (cpu_twin.cu): host pointers, synchronous, tensor by tensor
        for (int i = 0; i < n; ++i) {
            int rc;
            if (bits_op) {
                rc = cpu_run_bits(op == CT_OP_PACK_INT32, in[i], out[i], descs[i].rows, descs[i].cols, descs[i].num_bits, 1);
            } else {
                rc = validate_desc(&descs[i]);
                if (!rc) rc = check_dtypes(op, descs[i], zp && zp[i]);
                if (!rc) rc = cpu_run_one(op, descs[i], in[i], scale[i], zp ? zp[i] : nullptr, g_idx ? g_idx[i] : nullptr, out[i]);
            }
            if (rc) return rc;
        }
        return CT_OK;
    }
    int rc = check_device(device);
    if (rc) return rc;
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");

    std::vector<Plan> plans((size_t)n);
    for (int i = 0; i < n; ++i) {
        if (bits_op) {
            const ct_quant_desc& d = descs[i];
            if (d.num_bits < 1 || d.num_bits > 8) { set_error("num_bits %d outside [1, 8]", d.num_bits); return CT_E_BITS; }
            if (d.rows < 0 || d.cols < 0) { set_error("negative shape"); return CT_E_SHAPE; }
            if (d.rows * d.cols > 0 && (!in[i] || !out[i])) { set_error("null tensor pointer (tensor %d)", i); return CT_E_ARG; }
            plans[i] = plan_bits(op == CT_OP_PACK_INT32, d.rows, d.cols, d.num_bits, in[i], out[i]);
            continue;
        }
        rc = validate_desc(&descs[i]);
        if (rc) return rc;
        const void* z = zp ? zp[i] : nullptr;
        rc = check_dtypes(op, descs[i], z != nullptr);
        if (rc) return rc;
        if (descs[i].rows * descs[i].cols > 0 && (!in[i] || !scale[i] || !out[i])) { set_error("null tensor pointer (tensor %d)", i); return CT_E_ARG; }
        if (op == CT_OP_QUANTIZE_PACK_FP4 || op == CT_OP_UNPACK_DEQUANTIZE_FP4 || op == CT_OP_OBSERVE_QUANTIZE_PACK_FP4) plans[i] = plan_fp4(op, descs[i], in[i], scale[i], z, g_idx ? g_idx[i] : nullptr, out[i]);
        else if (op == CT_OP_SPARSE24_QUANTIZE_PACK || op == CT_OP_SPARSE24_UNPACK_DEQUANTIZE) plans[i] = plan_s24(op, descs[i], in[i], scale[i], z, g_idx ? g_idx[i] : nullptr, out[i]);
        else plans[i] = plan_one(op, descs[i], in[i], scale[i], z, g_idx ? g_idx[i] : nullptr, out[i]);
    }
    // group fast jobs by kernel (and clamp constants), one launch per group
    std::vector<char> done((size_t)n, 0);
    for (int i = 0; i < n; ++i) {
        if (done[i]) continue;
        if (!plans[i].k.launch) {
            // an empty tensor has nothing to compute, whatever op it is in (the fused-only ops would otherwise refuse it)
            if (descs[i].rows * descs[i].cols == 0) { done[i] = 1; continue; }
            if (bits_op) {
                rc = (op == CT_OP_PACK_INT32)
                         ? launch_generic_pack(reinterpret_cast<const int8_t*>(in[i]), reinterpret_cast<int32_t*>(out[i]), descs[i].rows, descs[i].cols, descs[i].num_bits, 1, stream)
                         : launch_generic_unpack(reinterpret_cast<const int32_t*>(in[i]), reinterpret_cast<int8_t*>(out[i]), descs[i].rows, descs[i].cols, descs[i].num_bits, 1, stream);
                if (rc) return rc;
                done[i] = 1;
                continue;
            }
            rc = run_generic(op, descs[i], in[i], scale ? scale[i] : nullptr, zp ? zp[i] : nullptr, g_idx ? g_idx[i] : nullptr, out[i], stream);
            if (rc) return rc;
            done[i] = 1;
            continue;
        }
        std::vector<Job> jobs;
        uint32_t tiles = 0;
        const StreamKernel kern = plans[i].k;
        const uint32_t tc = (uint32_t)kern.tile_chunks;
        for (int k = i; k < n; ++k) {
            if (done[k] || plans[k].k.launch != kern.launch || plans[k].cm.bits != plans[i].cm.bits) continue;
            const uint32_t nt = (plans[k].job.n_chunks + tc - 1) / tc;
            if ((uint64_t)tiles + nt >= 0xffffffffull) break;
            Job j = plans[k].job;
            j.tile_begin = tiles;
            j.tile_end = tiles + nt;
            tiles += nt;
            jobs.push_back(j);
            done[k] = 1;
        }
        LaunchPlan lp;
        lp.cm = plans[i].cm;
        lp.total_tiles = tiles;
        lp.tbl.n = (int)jobs.size();
        lp.tbl.jobs = nullptr;
        lp.tbl.one = jobs[0];
        // Device scratch of the launch (stream-ordered allocation, so concurrent callers never share it):
        // [16 bytes: tile counter of the dynamic schedule, zero] [job table when there is more than one job].
        // Launches with few tiles per CTA keep the static deal and need no scratch at all.
        uint8_t* scratch = nullptr;
        const bool many = jobs.size() > 1;
        const bool dynamic = (uint64_t)tiles * tc >= (uint64_t)DYNAMIC_MIN_TILES_PER_SM * TILE_CHUNKS * sm_count(device);
        if (many || dynamic) {
            const size_t tbl_bytes = many ? jobs.size() * sizeof(Job) : 0;
            rc = scratch_alloc(reinterpret_cast<void**>(&scratch), 16 + tbl_bytes, device, stream);
            if (rc) return rc;
            if (many) {
                rc = upload_jobs<Job, 32>(scratch, 16, jobs.data(), jobs.size(), stream);   // 32 jobs = 3.3 KB of kernel parameters
                if (rc) return rc;
                lp.tbl.jobs = reinterpret_cast<const Job*>(scratch + 16);
            } else {
                CT_CUDA_TRY(cudaMemsetAsync(scratch, 0, 16, stream));
            }
            if (dynamic) lp.sched = reinterpret_cast<uint32_t*>(scratch);
        }
        rc = kern.launch(lp, device, stream);
        if (scratch) cudaFreeAsync(scratch, stream);
        if (rc) return rc;
    }
    return CT_OK;
}

// the checks of an MSE-mode call (d->aux = ct_mse_block) of the fused observer `op`, and the zeroed `any`: 1 when the streaming pass
// should run, else the return code (CT_OK for an empty tensor; CT_E_UNSUPPORTED where only the generic path would take it)
static int mse_prologue(int op, const ct_quant_desc* d, const void* x, void* scale_out, void* zp_out, void* out, int device, void* stream) {
    if (device == CT_DEVICE_CPU || (reinterpret_cast<uintptr_t>(d->aux) & 7u) != 0) {
        set_error("the MSE observer mode runs on a CUDA device with an 8-byte aligned ct_mse_block");
        return CT_E_UNSUPPORTED;
    }
    int rc = validate_desc(d);
    if (rc) return rc;
    rc = check_dtypes(op, *d, zp_out != nullptr);
    if (rc) return rc;
    if (d->rows * d->cols == 0) return CT_OK;
    if (!x || !scale_out || !out) { set_error("null tensor pointer"); return CT_E_ARG; }
    const Plan p = op == CT_OP_OBSERVE_QUANTIZE_PACK ? plan_one(op, *d, x, scale_out, zp_out, nullptr, out) : plan_fp4(op, *d, x, scale_out, zp_out, nullptr, out);
    if (!p.k.launch) return run_generic(op, *d, x, scale_out, zp_out, nullptr, out, nullptr);
    rc = check_device(device);
    if (rc) return rc;
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    CT_CUDA_TRY(cudaMemsetAsync(reinterpret_cast<uint8_t*>(d->aux) + offsetof(ct_mse_block, any), 0, sizeof(uint64_t), reinterpret_cast<cudaStream_t>(stream)));
    return 1;
}

static int run_one(int op, const ct_quant_desc* d, const void* in, const void* scale, const void* zp,
                   const int32_t* g_idx, void* out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    const void* ins[1] = {in};
    const void* scales[1] = {scale};
    const void* zps[1] = {zp};
    const int32_t* gis[1] = {g_idx};
    void* outs[1] = {out};
    return run_batched(op, 1, d, ins, scales, zps, gis, outs, device, reinterpret_cast<cudaStream_t>(stream));
}

// standalone pack / unpack
static int run_bits(bool pack, const void* in, void* out, int64_t rows, int64_t cols, int bits, int packed_dim,
                    int device, cudaStream_t stream) {
    if (bits < 1 || bits > 8) { set_error("num_bits %d outside [1, 8]", bits); return CT_E_BITS; }
    if (packed_dim != 0 && packed_dim != 1) { set_error("packed_dim must be 0 or 1"); return CT_E_ARG; }
    if (rows < 0 || cols < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    if (device == CT_DEVICE_CPU) return cpu_run_bits(pack, in, out, rows, cols, bits, packed_dim);
    if (packed_dim == 1) {   // as one tensor of ct_batched: the streaming kernel where the layout admits it, the generic one otherwise
        ct_quant_desc d;
        memset(&d, 0, sizeof(d));
        d.rows = rows;
        d.cols = cols;
        d.num_bits = bits;
        const void* ins[1] = {in};
        void* outs[1] = {out};
        return run_batched(pack ? CT_OP_PACK_INT32 : CT_OP_UNPACK_INT32, 1, &d, ins, nullptr, nullptr, nullptr, outs, device, stream);
    }
    int rc = check_device(device);
    if (rc) return rc;
    if (rows * cols == 0) return CT_OK;
    if (!in || !out) { set_error("null tensor pointer"); return CT_E_ARG; }
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    if (pack) return launch_generic_pack(reinterpret_cast<const int8_t*>(in), reinterpret_cast<int32_t*>(out), rows, cols, bits, packed_dim, stream);
    return launch_generic_unpack(reinterpret_cast<const int32_t*>(in), reinterpret_cast<int8_t*>(out), rows, cols, bits, packed_dim, stream);
}

// small elementwise FP4 / MX entry points: device checks + one generic launch
template <class F>
static int run_simple(int device, int64_t rows, int64_t cols, const void* in, const void* out, F launch) {
    if (rows < 0 || cols < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    int rc = check_device(device);
    if (rc) return rc;
    if (rows * cols == 0) return CT_OK;
    if (!in || !out) { set_error("null tensor pointer"); return CT_E_ARG; }
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    return launch();
}

}  // namespace ctb

using namespace ctb;

extern "C" {

int ct_cast_to_fp4(const void* x, int dtype, void* out, int64_t n, int device, void* stream) {
    if (!is_float_dt(dtype)) { set_error("cast_to_fp4 needs a float dtype"); return CT_E_DTYPE; }
    return run_simple(device, 1, n, x, out, [&] { return launch_cast_to_fp4(x, dtype, out, n, reinterpret_cast<cudaStream_t>(stream)); });
}
int ct_pack_fp4(const void* x, int dtype, uint8_t* packed, int64_t rows, int64_t cols, int device, void* stream) {
    if (!is_float_dt(dtype)) { set_error("pack_fp4 needs a float dtype"); return CT_E_DTYPE; }
    if (cols % 2 != 0) { set_error("tensor must have an even number of columns for nvfp4 compression"); return CT_E_SHAPE; }
    return run_simple(device, rows, cols, x, packed, [&] { return launch_pack_fp4(x, dtype, packed, rows, cols, reinterpret_cast<cudaStream_t>(stream)); });
}
int ct_unpack_fp4(const uint8_t* packed, void* out, int out_dtype, int64_t rows, int64_t cols, int device, void* stream) {
    if (!is_float_dt(out_dtype)) { set_error("unpack_fp4 needs a float output dtype"); return CT_E_DTYPE; }
    if (cols % 2 != 0) { set_error("unpack_fp4 needs an even number of columns"); return CT_E_SHAPE; }
    return run_simple(device, rows, cols, packed, out, [&] { return launch_unpack_fp4(packed, out, out_dtype, rows, cols, reinterpret_cast<cudaStream_t>(stream)); });
}
int ct_quantize_pack_fp4(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, const int32_t* g_idx, uint8_t* packed, int device, void* stream) {
    return run_one(CT_OP_QUANTIZE_PACK_FP4, d, x, scale, zp, g_idx, packed, device, stream);
}
int ct_observe_quantize_pack_nvfp4(const ct_quant_desc* d, const void* x, void* scale_out_fp8, uint8_t* packed, int device, void* stream) {
    if (!d || !d->aux) return run_one(CT_OP_OBSERVE_QUANTIZE_PACK_FP4, d, x, scale_out_fp8, nullptr, nullptr, packed, device, stream);
    // MSE mode: the streaming pass with the search (local scales only; the global scale is an input), then the stop-step fix-up
    int rc = mse_prologue(CT_OP_OBSERVE_QUANTIZE_PACK_FP4, d, x, scale_out_fp8, nullptr, packed, device, stream);
    if (rc != 1) return rc;
    rc = run_one(CT_OP_OBSERVE_QUANTIZE_PACK_FP4, d, x, scale_out_fp8, nullptr, nullptr, packed, device, stream);
    if (rc) return rc;
    return launch_mse_fixup_nvfp4(*d, x, scale_out_fp8, packed, reinterpret_cast<cudaStream_t>(stream));
}
int ct_unpack_dequantize_fp4(const ct_quant_desc* d, const uint8_t* packed, const void* scale, const void* zp, const int32_t* g_idx, void* out, int device, void* stream) {
    return run_one(CT_OP_UNPACK_DEQUANTIZE_FP4, d, packed, scale, zp, g_idx, out, device, stream);
}
int ct_mx_scale_compress(const void* scale, int dtype, uint8_t* out, int64_t n, int device, void* stream) {
    if (!is_float_dt(dtype)) { set_error("mx_scale_compress needs a float dtype"); return CT_E_DTYPE; }
    return run_simple(device, 1, n, scale, out, [&] { return launch_mx_scale_compress(scale, dtype, out, n, reinterpret_cast<cudaStream_t>(stream)); });
}
int ct_mx_scale_decompress(const uint8_t* in, void* out_bf16, int64_t n, int device, void* stream) {
    return run_simple(device, 1, n, in, out_bf16, [&] { return launch_mx_scale_decompress(in, out_bf16, n, reinterpret_cast<cudaStream_t>(stream)); });
}

int ct_pack_int32(const int8_t* in, int32_t* out, int64_t rows, int64_t cols, int bits, int packed_dim, int device, void* stream) {
    return run_bits(true, in, out, rows, cols, bits, packed_dim, device, reinterpret_cast<cudaStream_t>(stream));
}
int ct_unpack_int32(const int32_t* in, int8_t* out, int64_t rows, int64_t cols, int bits, int packed_dim, int device, void* stream) {
    return run_bits(false, in, out, rows, cols, bits, packed_dim, device, reinterpret_cast<cudaStream_t>(stream));
}
int ct_quantize(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, const int32_t* g_idx, void* q_out, int device, void* stream) {
    return run_one(CT_OP_QUANTIZE, d, x, scale, zp, g_idx, q_out, device, stream);
}
int ct_dequantize(const ct_quant_desc* d, const void* q, const void* scale, const void* zp, const int32_t* g_idx, void* out, int device, void* stream) {
    return run_one(CT_OP_DEQUANTIZE, d, q, scale, zp, g_idx, out, device, stream);
}
int ct_fake_quantize(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, const int32_t* g_idx, void* out, int device, void* stream) {
    return run_one(CT_OP_FAKE_QUANTIZE, d, x, scale, zp, g_idx, out, device, stream);
}
int ct_quantize_pack_int32(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, const int32_t* g_idx, int32_t* packed, int device, void* stream) {
    return run_one(CT_OP_QUANTIZE_PACK, d, x, scale, zp, g_idx, packed, device, stream);
}
int ct_unpack_dequantize_int32(const ct_quant_desc* d, const int32_t* packed, const void* scale, const void* zp, const int32_t* g_idx, void* out, int device, void* stream) {
    return run_one(CT_OP_UNPACK_DEQUANTIZE, d, packed, scale, zp, g_idx, out, device, stream);
}
int ct_sparse24_quantize_pack_int4(const ct_quant_desc* d, const void* x, const void* scale, const void* zp, int32_t* packed,
                                   uint8_t* bitmask, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    ct_quant_desc t = *d;
    t.aux = bitmask;
    return run_one(CT_OP_SPARSE24_QUANTIZE_PACK, &t, x, scale, zp, nullptr, packed, device, stream);
}
int ct_sparse24_unpack_dequantize_int4(const ct_quant_desc* d, const int32_t* packed, const uint8_t* bitmask, const void* scale,
                                       const void* zp, void* out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    ct_quant_desc t = *d;
    t.aux = const_cast<uint8_t*>(bitmask);
    return run_one(CT_OP_SPARSE24_UNPACK_DEQUANTIZE, &t, packed, scale, zp, nullptr, out, device, stream);
}
int ct_observe_quantize_pack_int32(const ct_quant_desc* d, const void* x, void* scale_out, void* zp_out, int32_t* packed, int device, void* stream) {
    if (!d || !d->aux) return run_one(CT_OP_OBSERVE_QUANTIZE_PACK, d, x, scale_out, zp_out, nullptr, packed, device, stream);
    // MSE mode: the streaming pass with the search, then the stop-step fix-up; only the streaming kernel has the search
    int rc = mse_prologue(CT_OP_OBSERVE_QUANTIZE_PACK, d, x, scale_out, zp_out, packed, device, stream);
    if (rc != 1) return rc;
    rc = run_one(CT_OP_OBSERVE_QUANTIZE_PACK, d, x, scale_out, zp_out, nullptr, packed, device, stream);
    if (rc) return rc;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return launch_mse_fixup_pack(*d, x, scale_out, zp_out, packed, st);
}
int ct_batched(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale,
               const void* const* zp, void* const* out, int device, void* stream) {
    if (op == CT_OP_OBSERVE_QUANTIZE_PACK || op == CT_OP_OBSERVE_QUANTIZE_PACK_FP4 || op == CT_OP_OBSERVE_QUANTIZE_BLOCK || op == CT_OP_OBSERVE_QUANTIZE_MX)
        for (int i = 0; i < n && descs; ++i)
            if (descs[i].aux) {   // an MSE observer block: the whole-model observers run min-max only
                set_error("ct_batched: tensor %d asks for the MSE observer (aux set); run it through its per-tensor entry point", i);
                return CT_E_UNSUPPORTED;
            }
    return run_batched(op, n, descs, in, scale, zp, nullptr, out, device, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"

// observe_block_mx.cu -- one-pass "observe + compress" of weights for the formats whose scales come from a BLOCK or an MX reduction:
//   BLOCK  (FP8_BLOCK: block_structure [bh, bw], fp8 codes)    x [R, C] -> float8_e4m3fn [R, C] + scale in x's dtype [ceil(R/bh), ceil(C/bw)]
//   MX     (MXFP4 / MXFP8: groups of 32 along C, E8M0 scales)  x [R, C] -> E2M1 nibbles [R, C/2] or float8_e4m3fn [R, C] + uint8 [R, C/32]
// i.e. the memoryless min-max observer, calculate_qparams (quantization/utils/helpers.py:50-137, observe_core.cuh) and the compressor
// body (quantize, forward_helpers.py:523-546, then pack_fp4_to_uint8 / compress_mx_scale) in one pass: the weight crosses HBM once and
// neither the min / max tensors nor the float scales nor the unpacked codes exist in memory.  The per-element arithmetic is the one
// ct_quantize / ct_quantize_pack_fp4 run on the same scale (QuantizeOp with QF8, Fp4MxQuantPackOp), so the result equals the unfused
// path bit for bit.
//   BLOCK  one CTA of 256 threads per block.  A block of up to 2048 chunks of 8 elements (128 x 128) is held in registers, 8 chunks per
//          thread, between the reduction and the quantize; larger blocks read the block twice (the second read mostly from L2).  Edge
//          blocks of a ragged shape reduce over the elements that exist.
//   MX     4 lanes of one chunk each per group of 32 (min / max combined by two shuffles), 4 chunks per lane, 8 warps per CTA.
// Many tensors run in ONE launch: every CTA finds its tensor in a job table by a binary search on the first CTA of each job.
#include <cstring>
#include <vector>

#include "engine.h"
#include "fp4_ops.cuh"
#include "observe_core.cuh"
#include "ops.cuh"

namespace ctb {

constexpr int BM_THREADS = 256;
constexpr int BM_MAXU = 8;       // chunks per thread a block keeps in registers: blocks up to 256 * 8 * 8 = 16384 elements
constexpr int MX_UNITS = 4;      // chunks per lane of the MX kernel (one per warp-wide span of 32 chunks)
constexpr int64_t MX_CTA_CHUNKS = (int64_t)(BM_THREADS / 32) * MX_UNITS * 32;

struct BmJob {
    const uint8_t* x;
    uint8_t* out;
    void* scale;
    int64_t rows, cols;
    int64_t bh, bw, nbc;     // BLOCK: block rows, block columns, blocks per row of blocks
    int64_t cta_begin;       // first CTA of this job in the launch
    Common cm;
    int32_t dt;              // CT_BF16 / CT_F16
    int32_t fp4;             // MX: E2M1 nibbles (else fp8 codes)
};

// the job of this CTA and the CTA's index inside it
__device__ __forceinline__ const BmJob& find_job(const BmJob* jobs, int n, const BmJob& one, int64_t& local) {
    if (n == 1) { local = blockIdx.x; return one; }
    __shared__ int sj;
    if (threadIdx.x == 0) {
        int lo = 0, hi = n - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (jobs[mid].cta_begin <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
        }
        sj = lo;
    }
    __syncthreads();
    const BmJob& J = jobs[sj];
    local = (int64_t)blockIdx.x - J.cta_begin;
    return J;
}

// ------------------------------------------------------------------------------------
// BLOCK
// ------------------------------------------------------------------------------------
template <class P>
__device__ __forceinline__ void quant_block_chunk(const uint4& v, const ScaleCtx& sc, const Common& cm, uint8_t* dst) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t o[2];
    using QZ = QuantizeOp<P, QF8, 0, 1>;
    if (sc.slow) QZ::template chunk<true>(w, sc, 0u, cm, o);
    else QZ::template chunk<false>(w, sc, 0u, cm, o);
    stg_stream8(dst, make_uint2(o[0], o[1]));
}

template <class P>
__device__ __forceinline__ void block_body(const BmJob& J, int64_t blk) {
    __shared__ uint32_t red[2][BM_THREADS / 32];
    __shared__ float qs;
    const int64_t br = blk / J.nbc, bc = blk - br * J.nbc;
    const int64_t r0 = br * J.bh, c0 = bc * J.bw;
    const int64_t h = min(J.bh, J.rows - r0);
    const int wch = (int)(min(J.bw, J.cols - c0) / 8);   // chunks per row inside this block
    const int64_t nch = h * wch;
    const int64_t ucols = J.cols / 8;
    const uint4* xb = reinterpret_cast<const uint4*>(J.x) + r0 * ucols + c0 / 8;
    uint8_t* ob = J.out + r0 * J.cols + c0;
    const bool resident = nch <= (int64_t)BM_THREADS * BM_MAXU;

    uint4 v[BM_MAXU];
    uint32_t mn2 = 0u, mx2 = 0u;                          // +0.0 | +0.0: neutral, the observer clamps min <= 0 <= max
    if (resident) {
#pragma unroll
        for (int u = 0; u < BM_MAXU; ++u) {
            const int i = u * BM_THREADS + threadIdx.x;
            v[u] = make_uint4(0, 0, 0, 0);
            if (i < nch) { const int rr = i / wch; v[u] = ldg_stream16(xb + rr * ucols + (i - rr * wch)); }
        }
#pragma unroll
        for (int u = 0; u < BM_MAXU; ++u) obs_chunk_minmax<P>(v[u], mn2, mx2);
    } else {
        for (int64_t i = threadIdx.x; i < nch; i += BM_THREADS) {
            const int64_t rr = i / wch;
            obs_chunk_minmax<P>(__ldg(xb + rr * ucols + (i - rr * wch)), mn2, mx2);
        }
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        mn2 = min2_nan<P>(mn2, __shfl_xor_sync(0xffffffffu, mn2, d));
        mx2 = max2_nan<P>(mx2, __shfl_xor_sync(0xffffffffu, mx2, d));
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = mn2; red[1][threadIdx.x >> 5] = mx2; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < BM_THREADS / 32; ++w) { mn2 = min2_nan<P>(mn2, red[0][w]); mx2 = max2_nan<P>(mx2, red[1][w]); }
        float lo, hi, zq;
        obs_range2<P>(mn2, mx2, lo, hi);
        const float s = obs_scale_zp<P::DT>(lo, hi, false, J.cm.qmin, J.cm.qmax, zq);   // symmetric fp8: max|x| / 448 in T, 0 -> eps
        reinterpret_cast<unsigned short*>(J.scale)[blk] = (unsigned short)P::from_float1(s);
        qs = s;
    }
    __syncthreads();
    const ScaleCtx sc = make_scale_ctx(qs);
    if (resident) {
#pragma unroll
        for (int u = 0; u < BM_MAXU; ++u) {
            const int i = u * BM_THREADS + threadIdx.x;
            if (i >= nch) continue;
            const int rr = i / wch;
            quant_block_chunk<P>(v[u], sc, J.cm, ob + rr * J.cols + (int64_t)(i - rr * wch) * 8);
        }
    } else {
        for (int64_t i = threadIdx.x; i < nch; i += BM_THREADS) {
            const int64_t rr = i / wch;
            quant_block_chunk<P>(ldg_stream16(xb + rr * ucols + (i - rr * wch)), sc, J.cm, ob + rr * J.cols + (i - rr * wch) * 8);
        }
    }
}

__global__ void __launch_bounds__(BM_THREADS) observe_quantize_block_kernel(const BmJob* __restrict__ jobs, int n, const __grid_constant__ BmJob one) {
    int64_t blk;
    const BmJob& J = find_job(jobs, n, one, blk);
    if (J.dt == CT_BF16) block_body<BF16>(J, blk);
    else block_body<F16>(J, blk);
}

// ------------------------------------------------------------------------------------
// MX
// ------------------------------------------------------------------------------------
template <class P>
__device__ __forceinline__ void mx_body(const BmJob& J, int64_t cta) {
    const int lane = threadIdx.x & 31;
    const int64_t n_chunks = J.rows * J.cols / 8;
    const int64_t base = cta * MX_CTA_CHUNKS + (int64_t)(threadIdx.x >> 5) * (MX_UNITS * 32) + lane;
    const uint4* x = reinterpret_cast<const uint4*>(J.x);
    uint4 v[MX_UNITS];
#pragma unroll
    for (int k = 0; k < MX_UNITS; ++k) {
        const int64_t c = base + k * 32;
        v[k] = (c < n_chunks) ? ldg_stream16(x + c) : make_uint4(0, 0, 0, 0);   // groups never straddle n_chunks: cols % 32 == 0
    }
#pragma unroll
    for (int k = 0; k < MX_UNITS; ++k) {
        const int64_t c = base + k * 32;
        uint32_t mn2 = v[k].x, mx2 = v[k].x;
        obs_chunk_minmax<P>(v[k], mn2, mx2);
#pragma unroll
        for (int d = 1; d < 4; d <<= 1) {
            mn2 = min2_nan<P>(mn2, __shfl_xor_sync(0xffffffffu, mn2, d));
            mx2 = max2_nan<P>(mx2, __shfl_xor_sync(0xffffffffu, mx2, d));
        }
        if (c >= n_chunks) continue;
        float lo, hi;
        obs_range2<P>(mn2, mx2, lo, hi);
        const float s = obs_mx_scale<P::DT>(fmax_nan(fabsf(lo), fabsf(hi)), J.fp4 ? 4 : 8);   // power of two in T
        if ((lane & 3) == 0) reinterpret_cast<uint8_t*>(J.scale)[c >> 2] = (uint8_t)mx_scale_code(s, P::DT);   // as compress_mx_scale stores it
        const ScaleCtx sc = make_scale_ctx(s);
        const uint32_t w[4] = {v[k].x, v[k].y, v[k].z, v[k].w};
        if (J.fp4) {
            using QP = Fp4MxQuantPackOp<P, FZ_NONE>;
            stg_stream4(J.out + c * 4, sc.slow ? QP::template chunk<true>(w, sc, 0u, J.cm) : QP::template chunk<false>(w, sc, 0u, J.cm));
        } else {
            uint32_t o[2];
            using QZ = QuantizeOp<P, QF8, 0, 1>;
            if (sc.slow) QZ::template chunk<true>(w, sc, 0u, J.cm, o);
            else QZ::template chunk<false>(w, sc, 0u, J.cm, o);
            stg_stream8(J.out + c * 8, make_uint2(o[0], o[1]));
        }
    }
}

__global__ void __launch_bounds__(BM_THREADS) observe_quantize_mx_kernel(const BmJob* __restrict__ jobs, int n, const __grid_constant__ BmJob one) {
    int64_t cta;
    const BmJob& J = find_job(jobs, n, one, cta);
    if (J.dt == CT_BF16) mx_body<BF16>(J, cta);
    else mx_body<F16>(J, cta);
}

// ------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------
constexpr int UPLOAD_JOBS = 24;   // jobs per kernel-parameter block of a captured table upload (upload_jobs, common.cuh)

static bool is_inf_div(int64_t v) { return v == CT_DIV_INF; }

// the job of one descriptor, or CT_E_UNSUPPORTED with the reason
static int plan_job(bool block, const ct_quant_desc& d, const void* x, void* scale, void* out, BmJob& j) {
    memset(&j, 0, sizeof(j));
    const int xdt = d.x_dtype;
    if ((xdt != CT_BF16 && xdt != CT_F16) || d.compute_dtype != xdt) {
        set_error("fused BLOCK / MX observer: x must be bf16 or fp16 (compute dtype the same)");
        return CT_E_UNSUPPORTED;
    }
    if (d.zp_dtype != CT_NONE || d.global_scale) {
        set_error("fused BLOCK / MX observer: symmetric scales without a global scale only");
        return CT_E_UNSUPPORTED;
    }
    if (d.rows < 0 || d.cols < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    if (d.cols % 8 != 0 || !aligned16(x) || !aligned16(out)) {
        set_error("fused BLOCK / MX observer: rows of a multiple of 8 elements, 16-byte aligned x and codes");
        return CT_E_UNSUPPORTED;
    }
    if (block) {
        if (d.qtype != CT_Q_FLOAT || d.num_bits != 8 || d.q_dtype != CT_F8E4M3 || d.scale_dtype != xdt) {
            set_error("fused BLOCK observer: fp8 (e4m3) codes with the scale in x's dtype only");
            return CT_E_UNSUPPORTED;
        }
        if (is_inf_div(d.rdiv) || is_inf_div(d.cdiv) || d.rdiv <= 0 || d.cdiv <= 0 || d.cdiv % 8 != 0 || d.rdiv >= 0x7fffffffLL ||
            d.cdiv >= 0x7fffffffLL || d.rdiv * (d.cdiv / 8) >= 0x7fffffffLL || d.s_row_stride != (d.cols + d.cdiv - 1) / d.cdiv) {
            set_error("fused BLOCK observer: block [rdiv, cdiv] with cdiv %% 8 == 0 and s_row_stride = ceil(cols / cdiv)");
            return CT_E_UNSUPPORTED;
        }
        j.bh = d.rdiv; j.bw = d.cdiv; j.nbc = d.s_row_stride;
        j.cm = make_common(xdt, CT_Q_FLOAT, 8);
    } else {
        const bool fp4 = d.qtype == CT_Q_FP4 && d.num_bits == 4;
        const bool fp8 = d.qtype == CT_Q_FLOAT && d.num_bits == 8 && d.q_dtype == CT_F8E4M3;
        if ((!fp4 && !fp8) || d.scale_dtype != CT_E8M0 || d.rdiv != 1 || d.cdiv != 32 || d.cols % 32 != 0 || d.s_row_stride != d.cols / 32) {
            set_error("fused MX observer: E2M1 or fp8 (e4m3) codes, group 32 along the row with cols %% 32 == 0, E8M0 scales");
            return CT_E_UNSUPPORTED;
        }
        j.fp4 = fp4 ? 1 : 0;
        j.cm = make_common(xdt, fp4 ? CT_Q_FP4 : CT_Q_FLOAT, fp4 ? 4 : 8);
    }
    j.x = reinterpret_cast<const uint8_t*>(x);
    j.out = reinterpret_cast<uint8_t*>(out);
    j.scale = scale;
    j.rows = d.rows;
    j.cols = d.cols;
    j.dt = xdt;
    return CT_OK;
}

int run_observe_block_mx(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale, void* const* out,
                         int device, cudaStream_t st) {
    const bool block = op == CT_OP_OBSERVE_QUANTIZE_BLOCK;
    if (n < 0 || (n > 0 && (!descs || !in || !scale || !out))) { set_error("null table"); return CT_E_ARG; }
    for (int i = 0; i < n; ++i)
        if (descs[i].aux) { set_error("the fused BLOCK / MX observers have no MSE mode (aux set, tensor %d)", i); return CT_E_UNSUPPORTED; }
    if (device == CT_DEVICE_CPU) {
        set_error("the fused BLOCK / MX observers have no host twin; run the observer and the quantize separately");
        return CT_E_UNSUPPORTED;
    }
    int rc = check_device(device);
    if (rc) return rc;
    std::vector<BmJob> jobs;
    int64_t ctas = 0;
    for (int i = 0; i < n; ++i) {
        const ct_quant_desc& d = descs[i];
        if (d.rows * d.cols > 0 && (!in[i] || !scale[i] || !out[i])) { set_error("null tensor pointer (tensor %d)", i); return CT_E_ARG; }
        BmJob j;
        rc = plan_job(block, d, in[i], const_cast<void*>(scale[i]), out[i], j);
        if (rc) return rc;
        if (d.rows * d.cols == 0) continue;
        const int64_t c = block ? ((d.rows + d.rdiv - 1) / d.rdiv) * d.s_row_stride : (d.rows * d.cols / 8 + MX_CTA_CHUNKS - 1) / MX_CTA_CHUNKS;
        j.cta_begin = ctas;
        ctas += c;
        if (ctas >= 0x7fffffffLL) { set_error("fused BLOCK / MX observer: more than 2^31 CTAs in one launch"); return CT_E_UNSUPPORTED; }
        jobs.push_back(j);
    }
    if (jobs.empty()) return CT_OK;
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    BmJob* table = nullptr;
    if (jobs.size() > 1) {
        rc = scratch_alloc(reinterpret_cast<void**>(&table), jobs.size() * sizeof(BmJob), device, st);
        if (rc) return rc;
        rc = upload_jobs<BmJob, UPLOAD_JOBS>(reinterpret_cast<uint8_t*>(table), 0, jobs.data(), jobs.size(), st);
        if (rc) return rc;
    }
    if (block) observe_quantize_block_kernel<<<(unsigned)ctas, BM_THREADS, 0, st>>>(table, (int)jobs.size(), jobs[0]);
    else observe_quantize_mx_kernel<<<(unsigned)ctas, BM_THREADS, 0, st>>>(table, (int)jobs.size(), jobs[0]);
    count_launch();
    if (table) cudaFreeAsync(table, st);
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

}  // namespace ctb

using namespace ctb;

extern "C" {

int ct_observe_quantize_block(const ct_quant_desc* d, const void* x, void* scale_out, void* q_out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    const void* ins[1] = {x};
    const void* scs[1] = {scale_out};
    void* outs[1] = {q_out};
    return run_observe_block_mx(CT_OP_OBSERVE_QUANTIZE_BLOCK, 1, d, ins, scs, outs, device, reinterpret_cast<cudaStream_t>(stream));
}

int ct_observe_quantize_mx(const ct_quant_desc* d, const void* x, void* scale_out_e8m0, void* q_out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    const void* ins[1] = {x};
    const void* scs[1] = {scale_out_e8m0};
    void* outs[1] = {q_out};
    return run_observe_block_mx(CT_OP_OBSERVE_QUANTIZE_MX, 1, d, ins, scs, outs, device, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"

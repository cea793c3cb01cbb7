// observe_channel.cu -- one-pass "observe + quantize" for CHANNEL-wise (per output row) weight quantization:
//   x (bf16 / fp16) [rows, cols]  ->  codes + scale [rows, 1] (+ int8 zero point [rows, 1])
// The memoryless min-max observer, calculate_qparams (quantization/utils/helpers.py:50-137) and quantize
// (forward_helpers.py:523-546) [+ pack_to_int32] for the presets that quantize weights per channel (W8A8 / INT8: int8 codes,
// FP8_DYNAMIC: float8_e4m3fn codes, W8A16 / W4A16 channel: packed int32), SURVEY.md section 8 row (f)1.
// The reference reads the weight twice (observer, then quantize); here one CTA owns a row, keeps it in registers (up to
// 8 x 16 bytes per thread = 16384 columns), reduces min / max with packed min/max + shuffles, derives the qparams with the
// reference's per-op rounding and quantizes from the registers: the weight crosses HBM once.
// Wider rows (up to CH_MAXC x 16384 columns) are split over the CTAs of one thread-block cluster: each CTA keeps its slice in
// registers, the partial min / max meet in distributed shared memory, cluster rank 0 derives the qparams once and writes them into
// every CTA's shared memory, and each CTA quantizes its own slice -- still one HBM read of the weight.
#include <cooperative_groups.h>
#include <algorithm>
#include <cstring>

#include "engine.h"
#include "observe_core.cuh"
#include "ops.cuh"

namespace ctb {

enum ChanOut { CO_PACK4 = 0, CO_PACK8 = 1, CO_I8 = 2, CO_F8 = 3 };
constexpr int CH_MAXU = 8;   // most units (of 8 elements) per thread: rows up to 16384 columns.  The kernel is instantiated for 2, 4 and
                             // 8 units so that short rows do not pay for registers they do not use (more CTAs resident per SM)
constexpr int CH_MAXC = 8;   // most CTAs per cluster (the portable cluster size): rows up to 8 x 16384 = 131072 columns

template <class P, int OUT, int ASYM, int MAXU>
__global__ void __launch_bounds__(256) observe_channel_kernel(const uint4* __restrict__ x, void* __restrict__ scale_out, int8_t* __restrict__ zp_out,
                                                              uint8_t* __restrict__ out, int64_t rows, int units /* cols / 8 */, const __grid_constant__ Common cm) {
    __shared__ uint32_t red[2][8];
    __shared__ float qp[2];
    const int64_t r = blockIdx.x;
    const uint4* row = x + r * units;
    uint4 v[MAXU];
#pragma unroll
    for (int u = 0; u < MAXU; ++u) {
        const int i = u * 256 + threadIdx.x;
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
        for (int w = 1; w < 8; ++w) { mn2 = min2_nan<P>(mn2, red[0][w]); mx2 = max2_nan<P>(mx2, red[1][w]); }
        float lo, hi;
        obs_range2<P>(mn2, mx2, lo, hi);
        // calculate_qparams, each op rounded to T (helpers.py:74-131)
        float zq;
        const float s = obs_scale_zp<P::DT>(lo, hi, ASYM, cm.qmin, cm.qmax, zq);
        reinterpret_cast<unsigned short*>(scale_out)[r] = (unsigned short)P::from_float1(s);
        if (ASYM) zp_out[r] = (int8_t)(int)zq;
        qp[0] = s; qp[1] = zq;
    }
    __syncthreads();
    const ScaleCtx sc = make_scale_ctx(qp[0]);
    const uint32_t zp2 = ASYM ? dup2<P>(qp[1]) : 0u;
    constexpr int OW = (OUT == CO_PACK4) ? 1 : 2;   // output words per unit
    uint8_t* orow = out + (size_t)r * units * (4 * OW);
#pragma unroll
    for (int u = 0; u < MAXU; ++u) {
        const int i = u * 256 + threadIdx.x;
        if (i >= units) continue;
        const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
        uint32_t o[2];
        if constexpr (OUT == CO_PACK4 || OUT == CO_PACK8) {
            using QP = QuantPackOp<P, (OUT == CO_PACK4) ? 4 : 8, ASYM, 1>;
            if (sc.slow) QP::template chunk<true>(w, sc, zp2, cm, o);
            else QP::template chunk<false>(w, sc, zp2, cm, o);
        } else {
            using QZ = QuantizeOp<P, (OUT == CO_F8) ? QF8 : QI_WIDE, ASYM, 1>;
            if (sc.slow) QZ::template chunk<true>(w, sc, zp2, cm, o);
            else QZ::template chunk<false>(w, sc, zp2, cm, o);
        }
        if constexpr (OW == 1) stg_stream4(orow + (size_t)i * 4, o[0]);
        else stg_stream8(orow + (size_t)i * 8, make_uint2(o[0], o[1]));
    }
}

// Rows of one cluster of `csize` CTAs each, grid-strided over the resident clusters; CTA `rank` owns units
// [rank * slice, min(units, (rank + 1) * slice)) of every row.  The next row's slice is loaded while the current one is exchanged and
// quantized, so the two cluster barriers per row overlap HBM reads.  Same element rules as observe_channel_kernel: zero-filled lanes
// are neutral, min / max propagate NaN, so the split does not change any bit.
template <class P, int OUT, int ASYM, int MAXU>
__global__ void __launch_bounds__(256) observe_channel_cluster_kernel(const uint4* __restrict__ x, void* __restrict__ scale_out, int8_t* __restrict__ zp_out,
                                                                      uint8_t* __restrict__ out, int64_t rows, int units, int slice,
                                                                      const __grid_constant__ Common cm) {
    namespace cg = cooperative_groups;
    __shared__ uint32_t red[2][8];
    __shared__ uint32_t part[2];
    __shared__ float qp[2];
    cg::cluster_group cluster = cg::this_cluster();
    const unsigned rank = cluster.block_rank(), csize = cluster.num_blocks();
    const int64_t stride = gridDim.x / csize;
    const int beg = (int)rank * slice, end = min(units, beg + slice);
    auto load = [&](int64_t r, uint4 (&v)[MAXU]) {
        const uint4* row = x + r * units;
#pragma unroll
        for (int u = 0; u < MAXU; ++u) {
            const int i = beg + u * 256 + threadIdx.x;
            v[u] = (r < rows && i < end) ? ldg_stream16(row + i) : make_uint4(0, 0, 0, 0);
        }
    };
    uint4 v[MAXU], vn[MAXU];
    load(blockIdx.x / csize, v);
    for (int64_t r = blockIdx.x / csize; r < rows; r += stride) {
        uint32_t mn2 = v[0].x, mx2 = v[0].x;
#pragma unroll
        for (int u = 0; u < MAXU; ++u) obs_chunk_minmax<P>(v[u], mn2, mx2);
        load(r + stride, vn);   // in flight across the exchange and the quantize of row r
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            mn2 = min2_nan<P>(mn2, __shfl_xor_sync(0xffffffffu, mn2, d));
            mx2 = max2_nan<P>(mx2, __shfl_xor_sync(0xffffffffu, mx2, d));
        }
        if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = mn2; red[1][threadIdx.x >> 5] = mx2; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < 8; ++w) { mn2 = min2_nan<P>(mn2, red[0][w]); mx2 = max2_nan<P>(mx2, red[1][w]); }
            part[0] = mn2; part[1] = mx2;
        }
        cluster.sync();   // every CTA's partial is in its shared memory (and the previous row's qp has been read by all)
        if (rank == 0 && threadIdx.x == 0) {
            for (unsigned c = 1; c < csize; ++c) {
                const uint32_t* pc = cluster.map_shared_rank(part, c);
                mn2 = min2_nan<P>(mn2, pc[0]); mx2 = max2_nan<P>(mx2, pc[1]);
            }
            float lo, hi;
            obs_range2<P>(mn2, mx2, lo, hi);
            float zq;
            const float s = obs_scale_zp<P::DT>(lo, hi, ASYM, cm.qmin, cm.qmax, zq);
            reinterpret_cast<unsigned short*>(scale_out)[r] = (unsigned short)P::from_float1(s);
            if (ASYM) zp_out[r] = (int8_t)(int)zq;
            for (unsigned c = 0; c < csize; ++c) {
                float* qc = cluster.map_shared_rank(qp, c);
                qc[0] = s; qc[1] = zq;
            }
        }
        cluster.sync();   // qparams delivered; part[] may be rewritten from here on, and no CTA touches another's memory until
                          // the next row's first barrier, so the last row may exit
        const ScaleCtx sc = make_scale_ctx(qp[0]);
        const uint32_t zp2 = ASYM ? dup2<P>(qp[1]) : 0u;
        constexpr int OW = (OUT == CO_PACK4) ? 1 : 2;
        uint8_t* orow = out + (size_t)r * units * (4 * OW);
#pragma unroll
        for (int u = 0; u < MAXU; ++u) {
            const int i = beg + u * 256 + threadIdx.x;
            if (i >= end) continue;
            const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
            uint32_t o[2];
            if constexpr (OUT == CO_PACK4 || OUT == CO_PACK8) {
                using QP = QuantPackOp<P, (OUT == CO_PACK4) ? 4 : 8, ASYM, 1>;
                if (sc.slow) QP::template chunk<true>(w, sc, zp2, cm, o);
                else QP::template chunk<false>(w, sc, zp2, cm, o);
            } else {
                using QZ = QuantizeOp<P, (OUT == CO_F8) ? QF8 : QI_WIDE, ASYM, 1>;
                if (sc.slow) QZ::template chunk<true>(w, sc, zp2, cm, o);
                else QZ::template chunk<false>(w, sc, zp2, cm, o);
            }
            if constexpr (OW == 1) stg_stream4(orow + (size_t)i * 4, o[0]);
            else stg_stream8(orow + (size_t)i * 8, make_uint2(o[0], o[1]));
        }
#pragma unroll
        for (int u = 0; u < MAXU; ++u) v[u] = vn[u];
    }
}

template <class P, int OUT, int ASYM, int MAXU>
static cudaError_t launch_chan_cluster(int csize, const uint4* x, void* s, int8_t* z, uint8_t* out, int64_t rows, int units, const Common& cm, cudaStream_t st) {
    auto kern = observe_channel_cluster_kernel<P, OUT, ASYM, MAXU>;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(256);
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)csize; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    cfg.gridDim = dim3((unsigned)csize);
    int resident = 0;   // clusters the device holds at once: the grid, so every cluster loops over rows with its next row in flight
    cudaError_t e = cudaOccupancyMaxActiveClusters(&resident, kern, &cfg);
    if (e != cudaSuccess) return e;
    if (resident < 1) return cudaErrorInvalidConfiguration;
    cfg.gridDim = dim3((unsigned)(std::min<int64_t>(rows, resident) * csize));
    const int slice = (units + csize - 1) / csize;
    return cudaLaunchKernelEx(&cfg, kern, x, s, z, out, rows, units, slice, cm);
}

// cluster shape of a row of `units` 8-element units: the fewest CTAs of at most 4 units per thread (8192 columns), else of at most 8;
// 0 when the row is wider than CH_MAXC CTAs hold
static int chan_cluster_shape(int units, int& maxu) {
    for (int mu : {4, CH_MAXU}) {
        const int c = (units + 256 * mu - 1) / (256 * mu);
        if (c <= CH_MAXC) { maxu = mu; return c; }
    }
    return 0;
}

template <class P, int OUT>
static int launch_chan(bool asym, const uint4* x, void* s, int8_t* z, uint8_t* out, int64_t rows, int units, const Common& cm, cudaStream_t st) {
    if (units > 256 * CH_MAXU) {
        int maxu = 0;
        const int csize = chan_cluster_shape(units, maxu);
        cudaError_t e;
        if (maxu == 4) e = asym ? launch_chan_cluster<P, OUT, 1, 4>(csize, x, s, z, out, rows, units, cm, st) : launch_chan_cluster<P, OUT, 0, 4>(csize, x, s, z, out, rows, units, cm, st);
        else e = asym ? launch_chan_cluster<P, OUT, 1, CH_MAXU>(csize, x, s, z, out, rows, units, cm, st) : launch_chan_cluster<P, OUT, 0, CH_MAXU>(csize, x, s, z, out, rows, units, cm, st);
        count_launch();
        CT_CUDA_TRY(e);
        return CT_OK;
    }
    const int per_thread = (units + 255) / 256;
#define CT_CHAN_LAUNCH(A, U) observe_channel_kernel<P, OUT, A, U><<<(unsigned)rows, 256, 0, st>>>(x, s, z, out, rows, units, cm)
    if (asym) { if (per_thread <= 2) CT_CHAN_LAUNCH(1, 2); else if (per_thread <= 4) CT_CHAN_LAUNCH(1, 4); else CT_CHAN_LAUNCH(1, 8); }
    else { if (per_thread <= 2) CT_CHAN_LAUNCH(0, 2); else if (per_thread <= 4) CT_CHAN_LAUNCH(0, 4); else CT_CHAN_LAUNCH(0, 8); }
#undef CT_CHAN_LAUNCH
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
template <class P>
static int launch_chan_p(int outk, bool asym, const uint4* x, void* s, int8_t* z, uint8_t* out, int64_t rows, int units, const Common& cm, cudaStream_t st) {
    switch (outk) {
    case CO_PACK4: return launch_chan<P, CO_PACK4>(asym, x, s, z, out, rows, units, cm, st);
    case CO_PACK8: return launch_chan<P, CO_PACK8>(asym, x, s, z, out, rows, units, cm, st);
    case CO_I8: return launch_chan<P, CO_I8>(asym, x, s, z, out, rows, units, cm, st);
    default: return launch_chan<P, CO_F8>(false, x, s, z, out, rows, units, cm, st);
    }
}

}  // namespace ctb

using namespace ctb;

extern "C" int ct_observe_quantize_channel(const ct_quant_desc* d, const void* x, void* scale_out, void* zp_out, void* out, int device, void* stream) {
    if (!d) { set_error("null descriptor"); return CT_E_ARG; }
    int rc = check_device(device);
    if (rc) return rc;
    const bool asym = zp_out != nullptr;
    const bool dt_ok = (d->x_dtype == CT_BF16 || d->x_dtype == CT_F16) && d->scale_dtype == d->x_dtype && d->compute_dtype == d->x_dtype;
    int outk = -1;
    if (d->qtype == CT_Q_INT && d->q_dtype == CT_I32 && d->num_bits == 4) outk = CO_PACK4;
    else if (d->qtype == CT_Q_INT && d->q_dtype == CT_I32 && d->num_bits == 8) outk = CO_PACK8;
    else if (d->qtype == CT_Q_INT && d->q_dtype == CT_I8 && d->num_bits == 8) outk = CO_I8;
    else if (d->qtype == CT_Q_FLOAT && d->q_dtype == CT_F8E4M3 && d->num_bits == 8 && !asym) outk = CO_F8;
    const bool chan = d->rdiv == 1 && d->s_row_stride == 1 && (d->cdiv == CT_DIV_INF || d->cdiv >= d->cols);
    const bool width_ok = d->cols <= 8LL * 256 * CH_MAXU * CH_MAXC;
    if (!dt_ok || outk < 0 || !chan || d->cols % 8 != 0 || !width_ok || d->rows > 0x7fffffffLL ||
        (asym && d->zp_dtype != CT_I8) || !aligned16(x) || !aligned16(out)) {
        set_error("fused channel observer supports bf16 / fp16 weights, cols %% 8 == 0, cols <= %d, int8 / fp8 codes or 4- / 8-bit packed int32, "
                  "int8 zero points; run the observer and quantize separately otherwise", 8 * 256 * CH_MAXU * CH_MAXC);
        return CT_E_UNSUPPORTED;
    }
    if (d->rows * d->cols == 0) return CT_OK;
    if (!x || !scale_out || !out) { set_error("null tensor pointer"); return CT_E_ARG; }
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    Common cm;
    if (d->qtype == CT_Q_INT) { const float rr = (float)(1 << d->num_bits); cm.qmax = rr / 2 - 1; cm.qmin = -rr / 2; }
    else { cm.qmax = 448.f; cm.qmin = -448.f; }
    auto bits16 = [&](float v) -> uint32_t {   // host-side conversion; the bounds are exact in both dtypes
        uint16_t h;
        if (d->x_dtype == CT_BF16) { uint32_t u; memcpy(&u, &v, 4); h = (uint16_t)(u >> 16); }
        else { __half hv = __float2half_rn(v); memcpy(&h, &hv, 2); }
        return (uint32_t)h | ((uint32_t)h << 16);
    };
    cm.qmin2 = bits16(cm.qmin); cm.qmax2 = bits16(cm.qmax); cm.bits = d->num_bits;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const uint4* xp = reinterpret_cast<const uint4*>(x);
    if (d->x_dtype == CT_BF16) return launch_chan_p<BF16>(outk, asym, xp, scale_out, reinterpret_cast<int8_t*>(zp_out), reinterpret_cast<uint8_t*>(out), d->rows, (int)(d->cols / 8), cm, st);
    return launch_chan_p<F16>(outk, asym, xp, scale_out, reinterpret_cast<int8_t*>(zp_out), reinterpret_cast<uint8_t*>(out), d->rows, (int)(d->cols / 8), cm, st);
}

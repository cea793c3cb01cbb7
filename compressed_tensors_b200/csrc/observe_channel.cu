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
// MSE mode (d->aux = ct_mse_block, per-row kernel only): between the row's min / max and its qparams the CTA runs the shrink-grid
// search from the registers (observe_mse.cuh; the row's error is summed over the CTA with the warp shuffles and shared memory of the
// min / max), writes the row with its best improving step, and mse_fixup_channel_kernel then applies the call's stop step.
#include <cooperative_groups.h>
#include <algorithm>
#include <cstring>

#include "engine.h"
#include "generic.cuh"
#include "observe_core.cuh"
#include "observe_mse.cuh"
#include "ops.cuh"

namespace ctb {

enum ChanOut { CO_PACK4 = 0, CO_PACK8 = 1, CO_I8 = 2, CO_F8 = 3 };
constexpr int CH_MAXU = 8;   // most units (of 8 elements) per thread: rows up to 16384 columns.  The kernel is instantiated for 2, 4 and
                             // 8 units so that short rows do not pay for registers they do not use (more CTAs resident per SM)
constexpr int CH_MAXC = 8;   // most CTAs per cluster (the portable cluster size): rows up to 8 x 16384 = 131072 columns

template <class P, int OUT, int ASYM, int MAXU, bool MSE = false>
__global__ void __launch_bounds__(256) observe_channel_kernel(const uint4* __restrict__ x, void* __restrict__ scale_out, int8_t* __restrict__ zp_out,
                                                              uint8_t* __restrict__ out, int64_t rows, int units /* cols / 8 */, const __grid_constant__ Common cm,
                                                              ct_mse_block* B = nullptr) {
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
    if constexpr (MSE) {
        __shared__ float lh[2];
        __shared__ float esum[2][8];
        if (threadIdx.x == 0) {
            for (int w = 1; w < 8; ++w) { mn2 = min2_nan<P>(mn2, red[0][w]); mx2 = max2_nan<P>(mx2, red[1][w]); }
            obs_range2<P>(mn2, mx2, lh[0], lh[1]);
        }
        __syncthreads();
        const float lo = lh[0], hi = lh[1], norm = B->norm;
        const bool square = norm == 2.0f;
        const int steps = B->steps;
        float best = FLT_MAX;
        int best_i = 0;
        uint64_t mask = 0;
        for (int i = 0; i < steps; ++i) {   // one barrier per step: the partial sums alternate between two rows of esum
            const float p = __ldg(&B->shrink[i]);
            float czq;
            const float cs = obs_scale_zp<P::DT>(rnd_dt(lo * p, P::DT), rnd_dt(hi * p, P::DT), ASYM, cm.qmin, cm.qmax, czq);
            const ScaleCtx c = make_scale_ctx(cs);
            float e = 0.f;
#pragma unroll
            for (int u = 0; u < MAXU; ++u) {
                if (u * 256 + (int)threadIdx.x >= units) continue;
                const uint32_t w4[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    e += mse_elem<P, ASYM, OUT == CO_F8>(P::lo(w4[k]), cs, czq, c, cm.qmin, cm.qmax, norm, square) +
                         mse_elem<P, ASYM, OUT == CO_F8>(P::hi(w4[k]), cs, czq, c, cm.qmin, cm.qmax, norm, square);
            }
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) e += __shfl_xor_sync(0xffffffffu, e, d);
            if ((threadIdx.x & 31) == 0) esum[i & 1][threadIdx.x >> 5] = e;
            __syncthreads();
            if (threadIdx.x == 0) {
                float t = esum[i & 1][0];
                for (int w = 1; w < 8; ++w) t += esum[i & 1][w];
                if (B->errors) B->errors[(size_t)r * steps + i] = t;
                if (t < best) { best = t; best_i = i; mask |= 1ull << i; }   // NaN / inf never improve
            }
        }
        if (threadIdx.x == 0) {
            mse_publish(B, (uint64_t)r, mask);
            const float p = __ldg(&B->shrink[best_i]);
            float zq;
            const float s = obs_scale_zp<P::DT>(rnd_dt(lo * p, P::DT), rnd_dt(hi * p, P::DT), ASYM, cm.qmin, cm.qmax, zq);
            reinterpret_cast<unsigned short*>(scale_out)[r] = (unsigned short)P::from_float1(s);
            if (ASYM) zp_out[r] = (int8_t)(int)zq;
            qp[0] = s; qp[1] = zq;
        }
    } else if (threadIdx.x == 0) {
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

// The MSE mode's second launch, one CTA per row: the stop step from the call's `any` bits; a row whose mask has a bit above it is
// rewritten with its last improving step <= S (min / max, calculate_qparams and codes with the generic kernels' per-element source,
// equal to the streaming arithmetic); every other row only reads its mask.
template <class P, int OUT, int ASYM>
__global__ void __launch_bounds__(256) mse_fixup_channel_kernel(const ct_mse_block* B, const void* x, void* scale_out, int8_t* zp_out, uint8_t* out,
                                                                int64_t cols, float qmin, float qmax) {
    __shared__ float red[2][8];
    __shared__ float qp[2];
    const int64_t r = blockIdx.x;
    const uint64_t keep = mse_keep(B), m = B->masks[r];
    if ((m & ~keep) == 0) return;
    const int best = mse_last(m, keep);
    float mn = 0.f, mx = 0.f;   // min(min_vals, 0), max(max_vals, 0); a row that improved is finite
    for (int64_t j = threadIdx.x; j < cols; j += 256) {
        const float v = load_as_f32(x, r * cols + j, P::DT);
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, d));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = mn; red[1][threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) { mn = fminf(mn, red[0][w]); mx = fmaxf(mx, red[1][w]); }
        const float p = B->shrink[best];
        float zq;
        const float s = obs_scale_zp<P::DT>(rnd_dt(mn * p, P::DT), rnd_dt(mx * p, P::DT), ASYM, qmin, qmax, zq);
        reinterpret_cast<unsigned short*>(scale_out)[r] = (unsigned short)P::from_float1(s);
        if (ASYM) zp_out[r] = (int8_t)(int)zq;
        qp[0] = s; qp[1] = zq;
    }
    __syncthreads();
    const float s = qp[0], zq = qp[1];
    constexpr int QT = OUT == CO_F8 ? CT_Q_FLOAT : CT_Q_INT;
    auto code = [&](int64_t j) { return quant_scalar(load_as_f32(x, r * cols + j, P::DT), s, ASYM, zq, P::DT, QT, qmin, qmax); };
    if constexpr (OUT == CO_I8) {
        for (int64_t j = threadIdx.x; j < cols; j += 256) reinterpret_cast<int8_t*>(out)[r * cols + j] = (int8_t)(int)code(j);
    } else if constexpr (OUT == CO_F8) {
        for (int64_t j = threadIdx.x; j < cols; j += 256) out[r * cols + j] = hd_f32_to_e4m3(code(j));
    } else {
        constexpr int BITS = OUT == CO_PACK4 ? 4 : 8;
        uint32_t* words_out = reinterpret_cast<uint32_t*>(out) + r * cols * BITS / 32;
        for (int64_t u = threadIdx.x * 32; u < cols; u += 256 * 32) {
            const int nvalid = cols - u < 32 ? (int)(cols - u) : 32;
            uint32_t words[BITS];
            pack_group<BITS>(words, nvalid, [&](int j) { return (int32_t)code(u + j); });
            for (int w = 0; w < (nvalid * BITS + 31) / 32; ++w) words_out[u * BITS / 32 + w] = words[w];
        }
    }
}

// the MSE mode: the per-row kernel with the search, then its fix-up (rows up to 256 * CH_MAXU units)
template <class P, int OUT>
static int launch_chan_mse(bool asym, const uint4* x, void* s, int8_t* z, uint8_t* out, int64_t rows, int units, const Common& cm, ct_mse_block* B,
                           cudaStream_t st) {
    const int per_thread = (units + 255) / 256;
#define CT_CHAN_LAUNCH(A, U) observe_channel_kernel<P, OUT, A, U, true><<<(unsigned)rows, 256, 0, st>>>(x, s, z, out, rows, units, cm, B)
    if (asym) { if (per_thread <= 2) CT_CHAN_LAUNCH(1, 2); else if (per_thread <= 4) CT_CHAN_LAUNCH(1, 4); else CT_CHAN_LAUNCH(1, 8); }
    else { if (per_thread <= 2) CT_CHAN_LAUNCH(0, 2); else if (per_thread <= 4) CT_CHAN_LAUNCH(0, 4); else CT_CHAN_LAUNCH(0, 8); }
#undef CT_CHAN_LAUNCH
    CT_CUDA_TRY(cudaGetLastError());
    if (asym) mse_fixup_channel_kernel<P, OUT, 1><<<(unsigned)rows, 256, 0, st>>>(B, x, s, z, out, (int64_t)units * 8, cm.qmin, cm.qmax);
    else mse_fixup_channel_kernel<P, OUT, 0><<<(unsigned)rows, 256, 0, st>>>(B, x, s, z, out, (int64_t)units * 8, cm.qmin, cm.qmax);
    count_launch(2);
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

template <class P, int OUT>
static int launch_chan(bool asym, const uint4* x, void* s, int8_t* z, uint8_t* out, int64_t rows, int units, const Common& cm, cudaStream_t st,
                       ct_mse_block* B) {
    if (B) return launch_chan_mse<P, OUT>(asym, x, s, z, out, rows, units, cm, B, st);
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
static int launch_chan_p(int outk, bool asym, const uint4* x, void* s, int8_t* z, uint8_t* out, int64_t rows, int units, const Common& cm, cudaStream_t st,
                        ct_mse_block* B) {
    switch (outk) {
    case CO_PACK4: return launch_chan<P, CO_PACK4>(asym, x, s, z, out, rows, units, cm, st, B);
    case CO_PACK8: return launch_chan<P, CO_PACK8>(asym, x, s, z, out, rows, units, cm, st, B);
    case CO_I8: return launch_chan<P, CO_I8>(asym, x, s, z, out, rows, units, cm, st, B);
    default: return launch_chan<P, CO_F8>(false, x, s, z, out, rows, units, cm, st, B);
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
    // the MSE mode (d->aux) runs on the per-row kernel only: rows up to 16384 columns, on a device, with an 8-byte aligned block
    ct_mse_block* B = reinterpret_cast<ct_mse_block*>(d->aux);
    const bool width_ok = d->cols <= (B ? 8LL * 256 * CH_MAXU : 8LL * 256 * CH_MAXU * CH_MAXC);
    if (B && (device == CT_DEVICE_CPU || (reinterpret_cast<uintptr_t>(B) & 7u) != 0 || !width_ok)) {
        set_error("the channel observer's MSE mode runs on a CUDA device, rows up to %d columns, an 8-byte aligned ct_mse_block", 8 * 256 * CH_MAXU);
        return CT_E_UNSUPPORTED;
    }
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
    if (B) CT_CUDA_TRY(cudaMemsetAsync(reinterpret_cast<uint8_t*>(B) + offsetof(ct_mse_block, any), 0, sizeof(uint64_t), st));
    const uint4* xp = reinterpret_cast<const uint4*>(x);
    if (d->x_dtype == CT_BF16) return launch_chan_p<BF16>(outk, asym, xp, scale_out, reinterpret_cast<int8_t*>(zp_out), reinterpret_cast<uint8_t*>(out), d->rows, (int)(d->cols / 8), cm, st, B);
    return launch_chan_p<F16>(outk, asym, xp, scale_out, reinterpret_cast<int8_t*>(zp_out), reinterpret_cast<uint8_t*>(out), d->rows, (int)(d->cols / 8), cm, st, B);
}

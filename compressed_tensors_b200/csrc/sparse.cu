// sparse.cu -- bitmask packing and the two bitmask-sparse storage formats.
//
//   pack_bitmasks / unpack_bitmasks : utils/helpers.py:306-343 (numpy.packbits, bitorder little):
//       bit k of byte b of row r  <->  column 8*b + k
//   sparse24  (CompressionFormat.sparse_24_bitmask, config/base.py:18): per 4 consecutive elements
//       keep the 2 of largest |x| (ties: lower column first); values [R, C/2] + bitmask [R, C/8]
//   bitmask   (CompressionFormat.sparse_bitmask, config/base.py:17): values = x[x != 0] row-major,
//       bitmask = pack_bitmasks(x != 0), row_offsets = exclusive prefix of per-row counts
// The two compressors themselves are absent from the reference snapshot; the formats follow the
// restatement in oracle/ct_oracle.c ("parity unpinned"), only the mask bit order is pinned.
//
// Thread mapping: one lane owns 8 consecutive columns = one bitmask byte; the byte is formed with
// compare + shift inside the lane, and lanes exchange bytes with warp shuffles so that every
// fourth lane issues one aligned 32-bit store of four mask bytes.
#include <cstdlib>
#include <cub/device/device_scan.cuh>

#include "engine.h"
#include "quant_core.cuh"
#include "sparse_common.cuh"

namespace ctb {

// ---------------------------------------------------------------------------------------------
// element access by byte width
// ---------------------------------------------------------------------------------------------
template <int ES> struct Raw;
template <> struct Raw<1> { using T = uint8_t; };
template <> struct Raw<2> { using T = uint16_t; };
template <> struct Raw<4> { using T = uint32_t; };

// magnitude key: larger key <=> larger |x| (for non-NaN floats, and for int8)
template <int DT> __device__ __forceinline__ uint32_t abs_key(uint32_t raw) {
    if (DT == CT_I8) { int v = (int)(int8_t)raw; return (uint32_t)(v < 0 ? -v : v); }
    if (DT == CT_F8E4M3) return raw & 0x7fu;
    if (DT == CT_F32 || DT == CT_I32) {
        if (DT == CT_I32) { int v = (int)raw; return (uint32_t)(v < 0 ? -(int64_t)v : v); }
        return raw & 0x7fffffffu;
    }
    return raw & 0x7fffu;  // bf16 / f16
}
template <int DT> __device__ __forceinline__ bool is_nonzero(uint32_t raw) {
    if (DT == CT_I8 || DT == CT_I32 || DT == CT_U8) return raw != 0;
    if (DT == CT_F8E4M3) return (raw & 0x7fu) != 0;
    if (DT == CT_F32) return (raw & 0x7fffffffu) != 0;
    return (raw & 0x7fffu) != 0;   // -0.0 == 0
}

__device__ __forceinline__ void store_mask_byte(uint8_t* bitmask_row_base, int64_t byte_idx, uint32_t byte, bool valid, bool can_vec) {
    // combine 4 neighbouring lanes' bytes; lane%4==0 stores a word when the 4 bytes are in range & aligned
    uint32_t v = valid ? byte : 0u;
    v |= __shfl_down_sync(0xffffffffu, v, 1) << 8;
    v |= __shfl_down_sync(0xffffffffu, v, 2) << 16;
    if (can_vec) {
        if ((threadIdx.x & 3) == 0 && valid) *reinterpret_cast<uint32_t*>(bitmask_row_base + byte_idx) = v;
    } else if (valid) {
        bitmask_row_base[byte_idx] = (uint8_t)byte;
    }
}

// ---------------------------------------------------------------------------------------------
// pack / unpack bitmasks
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pack_bitmasks_kernel(const uint8_t* __restrict__ bm, uint8_t* __restrict__ out,
                                                            int64_t rows, int64_t cols, int64_t nb) {
    const int64_t total = rows * nb;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / nb, b = t - r * nb;
        const uint8_t* src = bm + r * cols + b * 8;
        const int nvalid = (int)min((int64_t)8, cols - b * 8);
        uint32_t byte = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k)
            if (k < nvalid && src[k]) byte |= 1u << k;
        out[t] = (uint8_t)byte;
    }
}
__global__ void __launch_bounds__(256) unpack_bitmasks_kernel(const uint8_t* __restrict__ packed, uint8_t* __restrict__ bm,
                                                              int64_t rows, int64_t cols, int64_t nb) {
    const int64_t total = rows * cols;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = i / cols, c = i - r * cols;
        bm[i] = (packed[r * nb + (c >> 3)] >> (c & 7)) & 1u;
    }
}

// ---------------------------------------------------------------------------------------------
// sparse24: lane = 8 columns = 2 quads.  cols % 8 == 0 fast layout; cols % 4 == 0 handled via nvalid.
// ---------------------------------------------------------------------------------------------
template <int DT, int ES>
__global__ void __launch_bounds__(256) sparse24_compress_kernel(const void* __restrict__ xin, void* __restrict__ vout,
                                                                uint8_t* __restrict__ bitmask, int64_t rows, int64_t cols, int64_t nb) {
    using T = typename Raw<ES>::T;
    const T* x = reinterpret_cast<const T*>(xin);
    T* values = reinterpret_cast<T*>(vout);
    const int64_t nb_pad = (nb + 3) & ~(int64_t)3;   // whole groups of 4 lanes stay on one row
    const int64_t total = rows * nb_pad;
    const bool vec_ok = (nb % 4 == 0) && ((reinterpret_cast<uintptr_t>(bitmask) & 3) == 0);
    const int64_t span = ((total + 31) / 32) * 32;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < span; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / nb_pad, b = t - r * nb_pad;
        const bool valid = (t < total) && (b < nb);
        uint32_t byte = 0;
        if (valid) {
            const int64_t c0 = b * 8;
            const int nq = (cols - c0 >= 8) ? 2 : 1;
            uint32_t raw[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) raw[k] = (k < nq * 4) ? (uint32_t)x[r * cols + c0 + k] : 0u;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                if (q < nq) {
                    uint32_t key[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) key[j] = abs_key<DT>(raw[q * 4 + j]);
                    uint32_t keep = 0;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        int beat = 0;
#pragma unroll
                        for (int m = 0; m < 4; ++m)
                            if (m != j && (key[m] > key[j] || (key[m] == key[j] && m < j))) ++beat;
                        if (beat < 2) keep |= 1u << j;
                    }
                    byte |= keep << (4 * q);
                    // the two kept elements in column order
                    const int i0 = __ffs(keep) - 1;
                    const int i1 = 31 - __clz(keep);
                    T* dst = values + r * (cols / 2) + (c0 / 2) + q * 2;
                    dst[0] = (T)raw[q * 4 + i0];
                    dst[1] = (T)raw[q * 4 + i1];
                }
            }
        }
        store_mask_byte(bitmask + r * nb, b, byte, valid, vec_ok);
    }
}

template <int ES>
__global__ void __launch_bounds__(256) sparse24_decompress_kernel(const void* __restrict__ vin, const uint8_t* __restrict__ bitmask,
                                                                  void* __restrict__ out, int64_t rows, int64_t cols, int64_t nb) {
    using T = typename Raw<ES>::T;
    const T* values = reinterpret_cast<const T*>(vin);
    T* o = reinterpret_cast<T*>(out);
    const int64_t total = rows * nb;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / nb, b = t - r * nb;
        const uint32_t byte = bitmask[t];
        const int64_t c0 = b * 8;
        const int nvalid = (int)min((int64_t)8, cols - c0);
        // values consumed before this byte in the row: 2 per full quad (valid 2:4 masks)
        int64_t vi = r * (cols / 2) + c0 / 2;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (k < nvalid) {
                T v = 0;
                if ((byte >> k) & 1u) v = values[vi++];
                o[r * cols + c0 + k] = v;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// sparse24, vectorised variants for 2-byte elements (bf16 / fp16), cols % 8 == 0, 16-byte aligned tensors and a mask size that is
// a multiple of 4 bytes: one thread = 8 elements = one 16-byte load, one 8-byte store of the 4 kept values, one mask byte
// (four lanes combine theirs into one 32-bit store).  Plain grid launch, one thread per unit: the hardware block scheduler
// balances the SMs (same effect as the dynamic tile schedule of stream.cuh; see tools/ubench/mix_ceiling.cu).
// Semantics identical to the generic kernels above (ties: lower column first; -0.0 counts as magnitude 0).
// ---------------------------------------------------------------------------------------------
// Every thread handles S24_U units, all loads issued before the first use: with one 16-byte load per thread a block lives for one
// DRAM round trip and the SM cannot keep enough bytes in flight; four loads per thread fix that.
constexpr int S24_U = 4;

__global__ void __launch_bounds__(256) sparse24_compress_vec16_kernel(const uint4* __restrict__ x, uint2* __restrict__ values,
                                                                      uint32_t* __restrict__ mask_words, int64_t n_units) {
    const int64_t t0 = (int64_t)blockIdx.x * (256 * S24_U) + threadIdx.x;
    uint4 v[S24_U];
#pragma unroll
    for (int u = 0; u < S24_U; ++u) {
        const int64_t t = t0 + u * 256;
        v[u] = (t < n_units) ? ldg_stream16(x + t) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < S24_U; ++u) {
        const int64_t t = t0 + u * 256;
        const bool valid = t < n_units;
        uint32_t p0, p1;
        uint32_t w = quad_select16(v[u].x, v[u].y, p0) | (quad_select16(v[u].z, v[u].w, p1) << 4);
        if (valid) stg_stream8(values + t, make_uint2(p0, p1));
        w |= __shfl_down_sync(0xffffffffu, w, 1) << 8;
        w |= __shfl_down_sync(0xffffffffu, w, 2) << 16;
        if ((threadIdx.x & 3) == 0 && valid) mask_words[t >> 2] = w;   // n_units % 4 == 0: the four lanes are valid together
    }
}

__global__ void __launch_bounds__(256) sparse24_decompress_vec16_kernel(const uint2* __restrict__ values, const uint8_t* __restrict__ bitmask,
                                                                        uint4* __restrict__ out, int64_t n_units) {
    const int64_t t0 = (int64_t)blockIdx.x * (256 * S24_U) + threadIdx.x;
    uint32_t bytes[S24_U];
    uint2 vals[S24_U];
#pragma unroll
    for (int u = 0; u < S24_U; ++u) {
        const int64_t t = t0 + u * 256;
        bytes[u] = (t < n_units) ? __ldg(bitmask + t) : 0u;
        vals[u] = (t < n_units) ? ldg_stream8(values + t) : make_uint2(0, 0);
    }
#pragma unroll
    for (int u = 0; u < S24_U; ++u) {
    const int64_t t = t0 + u * 256;
    if (t >= n_units) continue;
    const uint32_t byte = bytes[u];
    const uint2 v = vals[u];
    if (__popc(byte) > 4) {
        // not a 2:4 mask: more set bits than the unit's own 4 values.  Same sequential rule as the generic kernel (rare, slow).
        const uint16_t* src16 = reinterpret_cast<const uint16_t*>(values) + t * 4;
        uint16_t* o = reinterpret_cast<uint16_t*>(out) + t * 8;
        int vi = 0;
        for (int k = 0; k < 8; ++k) o[k] = ((byte >> k) & 1u) ? src16[vi++] : (uint16_t)0;
        continue;
    }
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t ba = (byte >> (2 * j)) & 1u, bb = (byte >> (2 * j + 1)) & 1u;
        const uint32_t ia = __popc(byte & ((1u << (2 * j)) - 1u)), ib = __popc(byte & ((1u << (2 * j + 1)) - 1u));   // values consumed before
        const uint32_t w = __byte_perm(v.x, v.y, 0x1010u + (ia & 3u) * 0x22u + (ib & 3u) * 0x2200u);
        o[j] = w & ((ba ? 0xffffu : 0u) | (bb ? 0xffff0000u : 0u));
    }
    stg_stream16(out + t, make_uint4(o[0], o[1], o[2], o[3]));
    }
}

static bool vec16_ok(int dtype, int64_t rows, int64_t cols, const void* a, const void* b, const void* c) {
    const int64_t n_units = rows * cols / 8;
    return (dtype == CT_BF16 || dtype == CT_F16) && cols % 8 == 0 && n_units % 4 == 0 && n_units < ((int64_t)1 << 39) &&
           aligned16(a) && aligned16(b) && aligned16(c);
}

// ---------------------------------------------------------------------------------------------
// unstructured bitmask: count -> scan -> scatter
// ---------------------------------------------------------------------------------------------
template <int DT, int ES>
__global__ void __launch_bounds__(256) bitmask_count_kernel(const void* __restrict__ xin, uint8_t* __restrict__ bitmask,
                                                            int64_t* __restrict__ counts, int64_t rows, int64_t cols, int64_t nb) {
    using T = typename Raw<ES>::T;
    const T* x = reinterpret_cast<const T*>(xin);
    __shared__ int warp_sums[8];
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        int local = 0;
        for (int64_t b = threadIdx.x; b < nb; b += blockDim.x) {
            const int64_t c0 = b * 8;
            const int nvalid = (int)min((int64_t)8, cols - c0);
            uint32_t byte = 0;
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (k < nvalid && is_nonzero<DT>((uint32_t)x[r * cols + c0 + k])) byte |= 1u << k;
            bitmask[r * nb + b] = (uint8_t)byte;
            local += __popc(byte);
        }
        for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xffffffffu, local, o);
        if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = local;
        __syncthreads();
        if (threadIdx.x == 0) {
            int s = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += warp_sums[w];
            counts[r] = s;
        }
        __syncthreads();
    }
}

// one block per row: per-thread popcounts over the row's mask bytes -> block exclusive scan -> scatter
template <int ES, bool COMPRESS>
__global__ void __launch_bounds__(256) bitmask_move_kernel(const void* __restrict__ src, const uint8_t* __restrict__ bitmask,
                                                           const int64_t* __restrict__ row_offsets, void* __restrict__ dst,
                                                           int64_t rows, int64_t cols, int64_t nb) {
    using T = typename Raw<ES>::T;
    __shared__ int warp_tot[8];
    __shared__ int carry_s;
    const T* s = reinterpret_cast<const T*>(src);
    T* d = reinterpret_cast<T*>(dst);
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x) {
        if (threadIdx.x == 0) carry_s = 0;
        __syncthreads();
        const int64_t base = row_offsets[r];
        for (int64_t b0 = 0; b0 < nb; b0 += blockDim.x) {
            const int64_t b = b0 + threadIdx.x;
            const uint32_t byte = (b < nb) ? bitmask[r * nb + b] : 0u;
            const int cnt = __popc(byte);
            // block exclusive scan of cnt
            int incl = cnt;
            for (int o = 1; o < 32; o <<= 1) {
                int n = __shfl_up_sync(0xffffffffu, incl, o);
                if ((threadIdx.x & 31) >= o) incl += n;
            }
            if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
            __syncthreads();
            int woff = 0;
            for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) woff += warp_tot[w];
            int64_t pos = base + carry_s + woff + incl - cnt;
            if (b < nb) {
                const int64_t c0 = b * 8;
                const int nvalid = (int)min((int64_t)8, cols - c0);
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (k < nvalid) {
                        const bool on = (byte >> k) & 1u;
                        if (COMPRESS) {
                            if (on) d[pos++] = s[r * cols + c0 + k];
                        } else {
                            T v = 0;
                            if (on) v = s[pos++];
                            d[r * cols + c0 + k] = v;
                        }
                    }
                }
            }
            __syncthreads();
            if (threadIdx.x == blockDim.x - 1) carry_s += woff + incl;
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------------------------
// unstructured bitmask, vectorised variants for 2-byte elements, cols % 8 == 0, 16-byte aligned dense tensor.
//   count : one block per row, 16-byte loads (4 per thread in flight), mask bytes combined four at a time into 32-bit stores
//   move  : one block per row, up to 4 segments of 256 units (2048 elements) per iteration: 16-byte access to the dense side
//           (4 loads per thread in flight), block scan of the popcounts, the kept elements staged in shared memory so that the
//           compact side is read / written coalesced, as 4-byte words
// Plain grid launch over the rows (hardware block scheduler = dynamic balance).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t nonzero_byte16(const uint4& v) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t byte = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        byte |= ((w[j] & 0x7fffu) != 0u ? 1u : 0u) << (2 * j);            // -0.0 == 0
        byte |= ((w[j] & 0x7fff0000u) != 0u ? 1u : 0u) << (2 * j + 1);
    }
    return byte;
}

__global__ void __launch_bounds__(256) bitmask_count_vec16_kernel(const uint4* __restrict__ x, uint8_t* __restrict__ bitmask,
                                                                  int64_t* __restrict__ counts, int units /* per row, % 4 == 0 */) {
    __shared__ int warp_sums[8];
    const int64_t r = blockIdx.x;
    const uint4* row = x + r * units;
    uint32_t* mrow = reinterpret_cast<uint32_t*>(bitmask + r * units);
    int local = 0;
    for (int b0 = 0; b0 < units; b0 += 256 * 4) {
        uint4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = b0 + u * 256 + threadIdx.x;
            v[u] = (i < units) ? ldg_stream16(row + i) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = b0 + u * 256 + threadIdx.x;
            uint32_t w = nonzero_byte16(v[u]);
            local += __popc(w);
            w |= __shfl_down_sync(0xffffffffu, w, 1) << 8;
            w |= __shfl_down_sync(0xffffffffu, w, 2) << 16;
            if ((threadIdx.x & 3) == 0 && i < units) mrow[i >> 2] = w;
        }
    }
    for (int o = 16; o > 0; o >>= 1) local += __shfl_down_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < 8; ++w) t += warp_sums[w];
        counts[r] = t;
    }
}

// U segments of 256 units (2048 elements) per block iteration: U independent 16-byte loads per thread in flight, U warp scans
// interleaved, ONE pair of block barriers for 2048 * U elements, and the compact side moved as 4-byte words.
template <bool COMPRESS, int U>
__global__ void __launch_bounds__(256) bitmask_move_vec16_kernel(const void* __restrict__ src, const uint8_t* __restrict__ bitmask,
                                                                 const int64_t* __restrict__ row_offsets, void* __restrict__ dst, int units) {
    __shared__ __align__(16) uint16_t stage[2048 * U];
    __shared__ int warp_tot[U][8];
    const int64_t r = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t pos = row_offsets[r];            // first compact element of this iteration
    const uint16_t* cin = reinterpret_cast<const uint16_t*>(src);     // compact side when expanding
    uint16_t* cout = reinterpret_cast<uint16_t*>(dst);                // compact side when compressing
    const uint4* din = reinterpret_cast<const uint4*>(src) + r * units;   // dense side when compressing
    uint4* dout = reinterpret_cast<uint4*>(dst) + r * units;              // dense side when expanding
    for (int b0 = 0; b0 < units; b0 += 256 * U) {
        uint4 v[U];
        uint32_t byte[U];
        int cnt[U], incl[U], off[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = b0 + u * 256 + threadIdx.x;
            v[u] = make_uint4(0, 0, 0, 0);
            byte[u] = 0;
            if (i < units) {
                if (COMPRESS) v[u] = ldg_stream16(din + i);             // the mask is recomputed: one load less
                else byte[u] = __ldg(bitmask + r * units + i);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (COMPRESS) byte[u] = nonzero_byte16(v[u]);
            cnt[u] = __popc(byte[u]);
            incl[u] = cnt[u];
        }
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int n = __shfl_up_sync(0xffffffffu, incl[u], o);
                if (lane >= o) incl[u] += n;
            }
        }
        if (lane == 31) {
#pragma unroll
            for (int u = 0; u < U; ++u) warp_tot[u][warp] = incl[u];
        }
        __syncthreads();
        int total = 0;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            int before = 0, seg = 0;
#pragma unroll
            for (int w = 0; w < 8; ++w) {
                const int t = warp_tot[u][w];
                if (w < warp) before += t;
                seg += t;
            }
            off[u] = total + before + incl[u] - cnt[u];      // this thread's first slot in the iteration's compact run
            total += seg;
        }
        // compact run [pos, pos + total): one 2-byte element to reach 4-byte alignment, then pairs, then a possible last element
        const uintptr_t caddr = reinterpret_cast<uintptr_t>((COMPRESS ? static_cast<const uint16_t*>(cout) : cin) + pos);
        const int head = (int)((caddr >> 1) & 1) & (total > 0 ? 1 : 0);
        const int pairs = (total - head) >> 1;
        const int tail = total - head - 2 * pairs;
        if (COMPRESS) {
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const uint32_t w[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
                int o = off[u];
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if ((byte[u] >> k) & 1u) stage[o++] = (uint16_t)(w[k >> 1] >> (16 * (k & 1)));
            }
            __syncthreads();
            if (threadIdx.x == 0 && head) cout[pos] = stage[0];
            uint32_t* c32 = reinterpret_cast<uint32_t*>(cout + pos + head);
            for (int j = threadIdx.x; j < pairs; j += 256) c32[j] = (uint32_t)stage[head + 2 * j] | ((uint32_t)stage[head + 2 * j + 1] << 16);   // coalesced
            if (threadIdx.x == 32 && tail) cout[pos + total - 1] = stage[total - 1];
        } else {
            if (threadIdx.x == 0 && head) stage[0] = cin[pos];
            const uint32_t* c32 = reinterpret_cast<const uint32_t*>(cin + pos + head);
            for (int j = threadIdx.x; j < pairs; j += 256) {                                                                                       // coalesced
                const uint32_t two = __ldg(c32 + j);
                stage[head + 2 * j] = (uint16_t)two;
                stage[head + 2 * j + 1] = (uint16_t)(two >> 16);
            }
            if (threadIdx.x == 32 && tail) stage[total - 1] = cin[pos + total - 1];
            __syncthreads();
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = b0 + u * 256 + threadIdx.x;
                if (i < units) {
                    uint32_t e[8];
                    int o = off[u];
#pragma unroll
                    for (int k = 0; k < 8; ++k) e[k] = ((byte[u] >> k) & 1u) ? (uint32_t)stage[o++] : 0u;
                    stg_stream16(dout + i, make_uint4(e[0] | (e[1] << 16), e[2] | (e[3] << 16), e[4] | (e[5] << 16), e[6] | (e[7] << 16)));
                }
            }
        }
        pos += total;
        __syncthreads();   // stage / warp_tot are reused by the next iteration
    }
}

// ------------------------------------------------------------------------------------------------------------------------------
// Expansion with row_offsets, pipelined (round 2).  The per-row kernel above is not issue-bound but latency-bound: a CTA lives for one row and goes through two DEPENDENT trips to DRAM (mask bytes ->
// counts -> the row's values) with nothing else in flight.  Both loads depend only on row_offsets, so here persistent CTAs walk the
// rows (r = blockIdx.x + k * gridDim.x); a PRODUCER warp keeps the next rows' mask bytes and value runs coming with bulk copies
// into a BYTE ring in shared memory (an entry is as large as the row's run actually is, so a sparse tensor has many rows in flight
// and a CTA needs only 1.5 worst-case rows of shared memory: 8 CTAs / SM for 8192 columns), eight consumer warps expand the current
// row out of shared memory.  Entries are released in order (`empty` barriers), the producer allocates behind the oldest one.
//   entry = [ values run, from the 16-byte boundary at or below row_offsets[r] to the one at or above row_offsets[r + 1] | mask bytes ]
// The over-read at the end of a run (< 16 bytes) is only done where it provably stays inside `values` (it ends at or before
// row_offsets[rows - 1] <= nnz); the last row and rows ending within 8 elements of it get a worst-case entry and fetch their values
// after the scan instead.
// ------------------------------------------------------------------------------------------------------------------------------
constexpr int EXR_SLOTS = 8;                 // rows in flight per CTA (barrier pairs)
constexpr int EXR_CONSUMERS = 256;
constexpr int EXR_THREADS = EXR_CONSUMERS + 32;

__device__ __forceinline__ void exr_consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(EXR_CONSUMERS) : "memory"); }

template <int U>
__global__ void __launch_bounds__(EXR_THREADS, (U <= 4 ? 6 : 4)) bitmask_expand_rows_kernel(const uint16_t* __restrict__ values, const uint8_t* __restrict__ bitmask,
                                                                          const int64_t* __restrict__ row_offsets, uint4* __restrict__ dense,
                                                                          int units, int rows, uint32_t ring_bytes, uint32_t vcap) {
    extern __shared__ __align__(128) uint8_t smem_raw[];     // [full barriers][empty barriers][ring]
    constexpr int NP = (U + 1) / 2;                          // two 16-bit segment counters per register (a segment holds <= 2048 elements)
    __shared__ uint32_t warp_tot[NP][8];
    __shared__ long long pos_s[EXR_SLOTS];
    __shared__ uint32_t off_s[EXR_SLOTS];                    // entry start in the ring; bit 31: the values are already there
    __shared__ uint32_t vpart_s[EXR_SLOTS];                  // bytes of the entry's values part (the mask bytes follow it)
    const uint32_t sbase = smem_u32(smem_raw);
    const uint32_t full0 = sbase, empty0 = sbase + 8u * EXR_SLOTS, ring0 = sbase + 16u * EXR_SLOTS;
    uint8_t* ring = smem_raw + 16 * EXR_SLOTS;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < EXR_SLOTS; ++s) {
            mbar_init_a(full0 + 8u * s, 1);
            mbar_init_a(empty0 + 8u * s, 1);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == EXR_CONSUMERS / 32) {
        // ---------------- producer ----------------
        if (lane != 0) return;
        const uint64_t policy = l2_evict_first_policy();
        const int64_t safe_end = row_offsets[rows - 1];
        uint32_t tail = 0, used = 0;                          // FIFO ring: outstanding bytes are [tail - used, tail) circularly
        uint32_t size_q[EXR_SLOTS];                           // bytes each outstanding entry holds (incl. the gap skipped when wrapping)
        uint32_t issued = 0, released = 0;
        for (int64_t r = blockIdx.x; r < rows; r += gridDim.x, ++issued) {
            const int64_t pos = row_offsets[r];
            const int64_t a0 = pos & ~7LL;
            uint32_t vb = 0;
            bool fast = false;
            if (r + 1 < rows) {
                const int64_t a1 = (row_offsets[r + 1] + 7) & ~7LL;
                if (a1 <= safe_end) { fast = true; vb = (uint32_t)(a1 - a0) * 2u; }
            }
            const uint32_t need = (fast ? vb : vcap) + (uint32_t)units;
            uint32_t start, size;
            while (true) {
                bool ok = issued - released < (uint32_t)EXR_SLOTS;
                if (ok) {
                    if (used == 0) { start = 0; size = need; }
                    else {
                        const uint32_t head = (tail + ring_bytes - used) % ring_bytes;
                        if (head < tail) {                    // outstanding entries do not wrap: free = [tail, end) and [0, head)
                            if (tail + need <= ring_bytes) { start = tail; size = need; }
                            else if (need <= head) { start = 0; size = need + (ring_bytes - tail); }
                            else ok = false;
                        } else {                              // they wrap (or the ring is full): free = [tail, head)
                            if (used < ring_bytes && need <= head - tail) { start = tail; size = need; }
                            else ok = false;
                        }
                    }
                }
                if (ok) break;
                // wait for the oldest outstanding entry
                const uint32_t q = released % EXR_SLOTS;
                mbar_wait_a(empty0 + 8u * q, (released / EXR_SLOTS) & 1u);
                used -= size_q[q];
                ++released;
            }
            const uint32_t q = issued % EXR_SLOTS;
            size_q[q] = size;
            used += size;
            tail = start + need;
            pos_s[q] = pos;
            off_s[q] = start | (fast ? 0x80000000u : 0u);
            const uint32_t bar = full0 + 8u * q, dst = ring0 + start;
            const uint32_t vpart = fast ? vb : vcap;          // the mask bytes follow the values part
            vpart_s[q] = vpart;
            mbar_expect_tx_a(bar, (uint32_t)units + vb);
            bulk_g2s_a(dst + vpart, bitmask + r * units, (uint32_t)units, bar, policy);
            if (vb) bulk_g2s_a(dst, values + a0, vb, bar, policy);
        }
        return;
    }

    // ---------------- consumers ----------------
    uint32_t it = 0;
    for (int64_t r = blockIdx.x; r < rows; r += gridDim.x, ++it) {
        const uint32_t q = it % EXR_SLOTS;
        mbar_wait_a(full0 + 8u * q, (it / EXR_SLOTS) & 1u);
        const uint32_t o = off_s[q];
        const bool fast = (o >> 31) != 0;
        const int64_t pos = pos_s[q];
        const int shift = (int)(pos & 7);                  // run element j sits at entry element shift + j
        uint16_t* sv = reinterpret_cast<uint16_t*>(ring + (o & 0x7fffffffu));
        uint32_t byte[U];
        int cnt[U], off[U];
        uint32_t pk[NP];                                   // segment u's count in the (u & 1) half of pk[u >> 1]
        {
            const uint8_t* mask = reinterpret_cast<const uint8_t*>(sv) + vpart_s[q];
#pragma unroll
            for (int i = 0; i < NP; ++i) pk[i] = 0u;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int i = u * 256 + tid;
                byte[u] = (i < units) ? mask[i] : 0u;
                cnt[u] = __popc(byte[u]);
                pk[u >> 1] |= (uint32_t)cnt[u] << (16 * (u & 1));
            }
        }
        // inclusive scan over the warp, two segments per shuffle
#pragma unroll
        for (int o2 = 1; o2 < 32; o2 <<= 1) {
#pragma unroll
            for (int i = 0; i < NP; ++i) {
                const uint32_t n = __shfl_up_sync(0xffffffffu, pk[i], o2);
                if (lane >= o2) pk[i] += n;
            }
        }
        if (lane == 31) {
#pragma unroll
            for (int i = 0; i < NP; ++i) warp_tot[i][warp] = pk[i];
        }
        exr_consumer_sync();
        // the eight warp totals of every segment: lanes 0 .. 7 scan them (three shuffle rounds), everybody reads its warp's exclusive
        // prefix from lane warp - 1 and the segment totals from lane 7
        int total = 0;
        {
            uint32_t t[NP], before[NP], seg[NP];
#pragma unroll
            for (int i = 0; i < NP; ++i) t[i] = (lane < 8) ? warp_tot[i][lane] : 0u;
#pragma unroll
            for (int o2 = 1; o2 < 8; o2 <<= 1) {
#pragma unroll
                for (int i = 0; i < NP; ++i) {
                    const uint32_t n = __shfl_up_sync(0xffffffffu, t[i], o2);
                    if (lane >= o2) t[i] += n;
                }
            }
#pragma unroll
            for (int i = 0; i < NP; ++i) {
                before[i] = __shfl_sync(0xffffffffu, t[i], (warp + 7) & 7);
                if (warp == 0) before[i] = 0u;
                seg[i] = __shfl_sync(0xffffffffu, t[i], 7);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int sh = 16 * (u & 1);
                off[u] = total + (int)((before[u >> 1] >> sh) & 0xffffu) + (int)((pk[u >> 1] >> sh) & 0xffffu) - cnt[u];
                total += (int)((seg[u >> 1] >> sh) & 0xffffu);
            }
        }
        if (!fast) {                                       // CTA-uniform: the last rows of the tensor
            for (int j = tid; j < total; j += EXR_CONSUMERS) sv[shift + j] = values[pos + j];
            exr_consumer_sync();
        }
        uint4* dout = dense + r * units;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = u * 256 + tid;
            if (i < units) {
                uint32_t e[8];
                int o2 = shift + off[u];
#pragma unroll
                for (int k = 0; k < 8; ++k) e[k] = ((byte[u] >> k) & 1u) ? (uint32_t)sv[o2++] : 0u;
                stg_stream16(dout + i, make_uint4(e[0] | (e[1] << 16), e[2] | (e[3] << 16), e[4] | (e[5] << 16), e[6] | (e[7] << 16)));
            }
        }
        exr_consumer_sync();                               // every consumer is done with the entry and with warp_tot
        if (tid == 0) mbar_arrive_a(empty0 + 8u * q);
    }
}

static bool bitmask_expand_rows_ok(int64_t rows, int units, const void* values) {
    return rows >= 2 && units % 16 == 0 && units <= 2048 && aligned16(values);
}

template <int U>
static int launch_bitmask_expand_rows_u(const void* values, const uint8_t* bitmask, const int64_t* row_offsets, void* dst, int64_t rows, int units,
                                        int device, cudaStream_t st) {
    const uint32_t vcap = (uint32_t)units * 16u + 32u;
    const uint32_t worst = vcap + (uint32_t)units;                 // an entry of a full row
    int pct = 150;                                                 // ring = 1.5 worst-case rows
    // test hook: at 100 % the ring holds exactly one worst-case row, a case no input reaches otherwise
    if (const char* e = getenv("CT_B200_BITMASK_RING_PCT")) pct = atoi(e);
    if (pct < 100) pct = 100;
    if (pct > 600) pct = 600;
    const uint32_t ring = (uint32_t)((uint64_t)worst * pct / 100 + 15) / 16 * 16;
    const int smem = 16 * EXR_SLOTS + (int)ring;
    if (smem > 200 * 1024) { set_error("bitmask expand: ring too large"); return CT_E_SHAPE; }
    auto kfn = bitmask_expand_rows_kernel<U>;
    CT_CUDA_TRY(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    int occ = 0;
    CT_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kfn, EXR_THREADS, smem));
    if (occ < 1) { set_error("bitmask expand: no occupancy"); return CT_E_CUDA; }
    int64_t grid = (int64_t)occ * sm_count(device);
    if (grid > rows) grid = rows;
    kfn<<<(unsigned)grid, EXR_THREADS, smem, st>>>(reinterpret_cast<const uint16_t*>(values), bitmask, row_offsets, reinterpret_cast<uint4*>(dst), units,
                                                   (int)rows, ring, vcap);
    return CT_OK;
}

static int launch_bitmask_expand_rows(const void* values, const uint8_t* bitmask, const int64_t* row_offsets, void* dst, int64_t rows, int units,
                                      int device, cudaStream_t st) {
    if (units <= 256) return launch_bitmask_expand_rows_u<1>(values, bitmask, row_offsets, dst, rows, units, device, st);
    if (units <= 512) return launch_bitmask_expand_rows_u<2>(values, bitmask, row_offsets, dst, rows, units, device, st);
    if (units <= 1024) return launch_bitmask_expand_rows_u<4>(values, bitmask, row_offsets, dst, rows, units, device, st);
    return launch_bitmask_expand_rows_u<8>(values, bitmask, row_offsets, dst, rows, units, device, st);
}

// rows shorter than one 4-segment iteration keep the single-segment shape (less shared memory, more blocks per SM)
template <bool COMPRESS>
static void launch_bitmask_move_vec16(const void* src, const uint8_t* bitmask, const int64_t* row_offsets, void* dst, int64_t rows, int units, cudaStream_t st) {
    const int cap = COMPRESS ? 2 : 4;   // compress keeps its 16-byte loads in registers: 4 segments cost 79 registers (3 blocks per SM)
    if (units > 512 && cap >= 4) bitmask_move_vec16_kernel<COMPRESS, 4><<<(unsigned)rows, 256, 0, st>>>(src, bitmask, row_offsets, dst, units);
    else if (units > 256 && cap >= 2) bitmask_move_vec16_kernel<COMPRESS, 2><<<(unsigned)rows, 256, 0, st>>>(src, bitmask, row_offsets, dst, units);
    else bitmask_move_vec16_kernel<COMPRESS, 1><<<(unsigned)rows, 256, 0, st>>>(src, bitmask, row_offsets, dst, units);
}

static bool bitmask_vec16_ok(int dtype, int64_t rows, int64_t cols, const void* dense, const void* mask) {
    return dt_size(dtype) == 2 && cols % 32 == 0 && cols / 8 < 0x7fffffffLL && rows > 0 && rows < 0x7fffffffLL && aligned16(dense) &&
           (reinterpret_cast<uintptr_t>(mask) & 3u) == 0;
}

static unsigned grid_for(int64_t items) {
    int64_t b = (items + 255) / 256;
    if (b < 1) b = 1;
    if (b > GRID_SMS * 16) b = GRID_SMS * 16;
    return (unsigned)b;
}
static int esize_of(int dt) { return dt_size(dt); }

}  // namespace ctb

using namespace ctb;

#define PRECHECK(device)                                  \
    int rc = check_device(device);                        \
    if (rc) return rc;                                    \
    DeviceGuard guard(device);                            \
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice"); \
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream)

extern "C" {

int ct_pack_bitmasks(const uint8_t* bytemask, uint8_t* packed, int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (rows * cols == 0) return CT_OK;
    if (!bytemask || !packed) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t nb = (cols + 7) / 8;
    pack_bitmasks_kernel<<<grid_for(rows * nb), 256, 0, st>>>(bytemask, packed, rows, cols, nb);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
int ct_unpack_bitmasks(const uint8_t* packed, uint8_t* bytemask, int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (rows * cols == 0) return CT_OK;
    if (!bytemask || !packed) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t nb = (cols + 7) / 8;
    unpack_bitmasks_kernel<<<grid_for(rows * cols), 256, 0, st>>>(packed, bytemask, rows, cols, nb);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

int ct_sparse24_compress(const void* x, int dtype, void* values, uint8_t* bitmask, int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (cols % 4 != 0) { set_error("2:4 compression needs cols %% 4 == 0 (got %lld)", (long long)cols); return CT_E_SHAPE; }
    if (rows * cols == 0) return CT_OK;
    if (!x || !values || !bitmask) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t nb = (cols + 7) / 8;
    if (vec16_ok(dtype, rows, cols, x, values, bitmask)) {
        const int64_t n_units = rows * cols / 8;
        sparse24_compress_vec16_kernel<<<(unsigned)((n_units + 256 * S24_U - 1) / (256 * S24_U)), 256, 0, st>>>(
            reinterpret_cast<const uint4*>(x), reinterpret_cast<uint2*>(values), reinterpret_cast<uint32_t*>(bitmask), n_units);
        count_launch();
        CT_CUDA_TRY(cudaGetLastError());
        return CT_OK;
    }
    const unsigned g = grid_for(rows * ((nb + 3) & ~(int64_t)3));
    switch (dtype) {
    case CT_BF16: sparse24_compress_kernel<CT_BF16, 2><<<g, 256, 0, st>>>(x, values, bitmask, rows, cols, nb); break;
    case CT_F16: sparse24_compress_kernel<CT_F16, 2><<<g, 256, 0, st>>>(x, values, bitmask, rows, cols, nb); break;
    case CT_F32: sparse24_compress_kernel<CT_F32, 4><<<g, 256, 0, st>>>(x, values, bitmask, rows, cols, nb); break;
    case CT_I8: sparse24_compress_kernel<CT_I8, 1><<<g, 256, 0, st>>>(x, values, bitmask, rows, cols, nb); break;
    case CT_F8E4M3: sparse24_compress_kernel<CT_F8E4M3, 1><<<g, 256, 0, st>>>(x, values, bitmask, rows, cols, nb); break;
    default: set_error("unsupported dtype %d", dtype); return CT_E_DTYPE;
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

int ct_sparse24_decompress(const void* values, int dtype, const uint8_t* bitmask, void* out, int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (cols % 4 != 0) { set_error("2:4 decompression needs cols %% 4 == 0"); return CT_E_SHAPE; }
    if (rows * cols == 0) return CT_OK;
    if (!out || !values || !bitmask) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t nb = (cols + 7) / 8;
    if (vec16_ok(dtype, rows, cols, values, out, values)) {   // the mask is read bytewise: no alignment needed
        const int64_t n_units = rows * cols / 8;
        sparse24_decompress_vec16_kernel<<<(unsigned)((n_units + 256 * S24_U - 1) / (256 * S24_U)), 256, 0, st>>>(
            reinterpret_cast<const uint2*>(values), bitmask, reinterpret_cast<uint4*>(out), n_units);
        count_launch();
        CT_CUDA_TRY(cudaGetLastError());
        return CT_OK;
    }
    const unsigned g = grid_for(rows * nb);
    switch (esize_of(dtype)) {
    case 1: sparse24_decompress_kernel<1><<<g, 256, 0, st>>>(values, bitmask, out, rows, cols, nb); break;
    case 2: sparse24_decompress_kernel<2><<<g, 256, 0, st>>>(values, bitmask, out, rows, cols, nb); break;
    case 4: sparse24_decompress_kernel<4><<<g, 256, 0, st>>>(values, bitmask, out, rows, cols, nb); break;
    default: set_error("unsupported dtype %d", dtype); return CT_E_DTYPE;
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

int64_t ct_bitmask_workspace_bytes(int64_t rows, int64_t cols) {
    (void)cols;
    size_t tmp = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp, (const int64_t*)nullptr, (int64_t*)nullptr, (int)(rows + 1));
    return (int64_t)((rows + 1) * sizeof(int64_t) + ((tmp + 255) & ~(size_t)255) + 256);
}

int ct_bitmask_count(const void* x, int dtype, uint8_t* bitmask, int64_t* row_offsets, int64_t* nnz_out, void* workspace,
                     int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (!row_offsets || !nnz_out || !workspace) { set_error("null pointer"); return CT_E_ARG; }
    if (rows == 0) { CT_CUDA_TRY(cudaMemsetAsync(nnz_out, 0, sizeof(int64_t), st)); return CT_OK; }
    if (!x || !bitmask) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t nb = (cols + 7) / 8;
    int64_t* counts = reinterpret_cast<int64_t*>(workspace);               // rows + 1 entries, last = 0
    void* tmp = reinterpret_cast<uint8_t*>(workspace) + (((rows + 1) * sizeof(int64_t) + 255) & ~(size_t)255);
    CT_CUDA_TRY(cudaMemsetAsync(counts + rows, 0, sizeof(int64_t), st));
    const unsigned g = (unsigned)(rows < GRID_SMS * 8 ? rows : GRID_SMS * 8);
    if (bitmask_vec16_ok(dtype, rows, cols, x, bitmask) && (dtype == CT_BF16 || dtype == CT_F16)) {
        bitmask_count_vec16_kernel<<<(unsigned)rows, 256, 0, st>>>(reinterpret_cast<const uint4*>(x), bitmask, counts, (int)(cols / 8));
    } else
    switch (dtype) {
    case CT_BF16: bitmask_count_kernel<CT_BF16, 2><<<g, 256, 0, st>>>(x, bitmask, counts, rows, cols, nb); break;
    case CT_F16: bitmask_count_kernel<CT_F16, 2><<<g, 256, 0, st>>>(x, bitmask, counts, rows, cols, nb); break;
    case CT_F32: bitmask_count_kernel<CT_F32, 4><<<g, 256, 0, st>>>(x, bitmask, counts, rows, cols, nb); break;
    case CT_I8: bitmask_count_kernel<CT_I8, 1><<<g, 256, 0, st>>>(x, bitmask, counts, rows, cols, nb); break;
    case CT_F8E4M3: bitmask_count_kernel<CT_F8E4M3, 1><<<g, 256, 0, st>>>(x, bitmask, counts, rows, cols, nb); break;
    default: set_error("unsupported dtype %d", dtype); return CT_E_DTYPE;
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    // exclusive scan over rows+1 counts into a (rows+1)-long temp, then split: first `rows` -> row_offsets, last -> nnz
    size_t tmp_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, counts, counts, (int)(rows + 1));
    CT_CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, counts, counts, (int)(rows + 1), st));
    count_launch();
    CT_CUDA_TRY(cudaMemcpyAsync(row_offsets, counts, rows * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    CT_CUDA_TRY(cudaMemcpyAsync(nnz_out, counts + rows, sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    return CT_OK;
}

int ct_bitmask_compress(const void* x, int dtype, const uint8_t* bitmask, const int64_t* row_offsets, void* values,
                        int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (rows * cols == 0) return CT_OK;
    if (!x || !bitmask || !row_offsets) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t nb = (cols + 7) / 8;
    const unsigned g = (unsigned)(rows < GRID_SMS * 8 ? rows : GRID_SMS * 8);
    if ((dtype == CT_BF16 || dtype == CT_F16) && bitmask_vec16_ok(dtype, rows, cols, x, bitmask)) {
        launch_bitmask_move_vec16<true>(x, bitmask, row_offsets, values, rows, (int)(cols / 8), st);
    } else
    switch (esize_of(dtype)) {
    case 1: bitmask_move_kernel<1, true><<<g, 256, 0, st>>>(x, bitmask, row_offsets, values, rows, cols, nb); break;
    case 2: bitmask_move_kernel<2, true><<<g, 256, 0, st>>>(x, bitmask, row_offsets, values, rows, cols, nb); break;
    case 4: bitmask_move_kernel<4, true><<<g, 256, 0, st>>>(x, bitmask, row_offsets, values, rows, cols, nb); break;
    default: set_error("unsupported dtype %d", dtype); return CT_E_DTYPE;
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

/* one call, no host round trip: values has capacity rows * cols, nnz stays on the device */
int ct_bitmask_compress_onepass(const void* x, int dtype, void* values, uint8_t* bitmask, int64_t* row_offsets, int64_t* nnz_out,
                                int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (!row_offsets || !nnz_out) { set_error("null pointer"); return CT_E_ARG; }
    if (rows * cols == 0) {
        CT_CUDA_TRY(cudaMemsetAsync(nnz_out, 0, sizeof(int64_t), st));
        if (rows > 0) CT_CUDA_TRY(cudaMemsetAsync(row_offsets, 0, rows * sizeof(int64_t), st));
        return CT_OK;
    }
    if (!x || !values || !bitmask) { set_error("null pointer"); return CT_E_ARG; }
    if (bitmask_lookback_ok(dtype, rows, cols, x, bitmask, values))
        return launch_bitmask_lookback<true>(x, bitmask, values, row_offsets, nnz_out, rows, cols, device, st);
    // every other dtype / shape: the two-phase kernels with a stream-ordered workspace (still no host synchronisation)
    void* ws = nullptr;
    rc = scratch_alloc(&ws, (size_t)ct_bitmask_workspace_bytes(rows, cols), device, st);
    if (rc) return rc;
    rc = ct_bitmask_count(x, dtype, bitmask, row_offsets, nnz_out, ws, rows, cols, device, stream);
    if (!rc) rc = ct_bitmask_compress(x, dtype, bitmask, row_offsets, values, rows, cols, device, stream);
    cudaFreeAsync(ws, st);
    return rc;
}

int ct_bitmask_decompress(const void* values, int dtype, const uint8_t* bitmask, const int64_t* row_offsets, void* out,
                          int64_t rows, int64_t cols, int device, void* stream) {
    PRECHECK(device);
    if (rows * cols == 0) return CT_OK;
    if (!out || !bitmask) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t nb = (cols + 7) / 8;
    const unsigned g = (unsigned)(rows < GRID_SMS * 8 ? rows : GRID_SMS * 8);
    // With the format's row_offsets the expansion is ONE pass already (every row knows where its values start): the pipelined row
    // kernel, or the per-row kernel for shapes it declines.  The look-back kernel (flat tiles, the scan recomputed from the mask
    // popcounts, slower) serves callers that do not have row_offsets.
    if (values && !row_offsets && bitmask_lookback_ok(dtype, rows, cols, out, bitmask, values))
        return launch_bitmask_lookback<false>(values, const_cast<uint8_t*>(bitmask), out, nullptr, nullptr, rows, cols, device, st);
    if (!row_offsets) { set_error("bitmask_decompress without row_offsets needs a 2-byte dtype, cols %% 8 == 0 and aligned tensors"); return CT_E_UNSUPPORTED; }
    if (bitmask_vec16_ok(dtype, rows, cols, out, bitmask) && (reinterpret_cast<uintptr_t>(bitmask) & 15u) == 0 &&
        bitmask_expand_rows_ok(rows, (int)(cols / 8), values)) {
        const int rc = launch_bitmask_expand_rows(values, bitmask, row_offsets, out, rows, (int)(cols / 8), device, st);
        if (rc) return rc;
    } else if (bitmask_vec16_ok(dtype, rows, cols, out, bitmask)) {
        launch_bitmask_move_vec16<false>(values, bitmask, row_offsets, out, rows, (int)(cols / 8), st);
    } else
    switch (esize_of(dtype)) {
    case 1: bitmask_move_kernel<1, false><<<g, 256, 0, st>>>(values, bitmask, row_offsets, out, rows, cols, nb); break;
    case 2: bitmask_move_kernel<2, false><<<g, 256, 0, st>>>(values, bitmask, row_offsets, out, rows, cols, nb); break;
    case 4: bitmask_move_kernel<4, false><<<g, 256, 0, st>>>(values, bitmask, row_offsets, out, rows, cols, nb); break;
    default: set_error("unsupported dtype %d", dtype); return CT_E_DTYPE;
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// 2:4 "semi-structured" values + metadata in the CUTLASS / marlin-24 layout
// (utils/semi_structured_conversions.py:33-60 reorder offsets, :66-197 from dense, :204-298 to dense).
// One thread per metadata element: QPE (4 for int16 meta, 8 for int32 meta) groups of KS dense
// elements (4, or 2 for fp32) each contribute a 4-bit code idx0 | idx1 << 2 and 2 (1) kept values.
// ---------------------------------------------------------------------------------------------
namespace ctb {

__device__ __forceinline__ int64_t meta_offset(int64_t r, int64_t c, int64_t m, int meta_bytes) {
    const int64_t gy = (meta_bytes == 2) ? 32 : 16;
    int64_t rr = r / 64 * 64 + (r % 2) * 2 + (r % 8) / 4 + ((r % gy) % 4) / 2 * 32 + ((r % 64) / 8) * 4;
    const int tr = (rr % 2 == 0) && (c % 2 == 1);
    const int bl = (rr % 2 == 1) && (c % 2 == 0);
    rr += tr - bl;
    const int64_t cc = c - (tr - bl);
    return (cc / 2) * m * 2 + rr * 2 + (cc % 2);
}

// ES = element bytes of the dense data (1, 2, 4); KS = dense elements per code (4, or 2 for fp32)
template <int DT, int ES, int KS, int MB>
__global__ void __launch_bounds__(256) semi_from_dense_kernel(const void* __restrict__ din, void* __restrict__ sout, void* __restrict__ mout,
                                                              int64_t m, int64_t k, int64_t ncols) {
    using T = typename Raw<ES>::T;
    constexpr int QPE = MB * 2;
    const T* dense = reinterpret_cast<const T*>(din);
    T* sparse = reinterpret_cast<T*>(sout);
    const int64_t total = m * ncols;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / ncols, c = t - r * ncols;
        uint32_t word = 0;
#pragma unroll
        for (int q = 0; q < QPE; ++q) {
            const int64_t base = r * k + (c * QPE + q) * KS;
            T v[KS];
#pragma unroll
            for (int i = 0; i < KS; ++i) v[i] = dense[base + i];
            int m0, m1, m3;
            if (KS == 4) { m0 = is_nonzero<DT>((uint32_t)v[0]); m1 = is_nonzero<DT>((uint32_t)v[1]); m3 = is_nonzero<DT>((uint32_t)v[KS - 1]); }
            else { m0 = m1 = is_nonzero<DT>((uint32_t)v[0]); m3 = is_nonzero<DT>((uint32_t)v[KS - 1]); }
            const int e0 = m0 & m1, e1 = (!m0) & m1, e2 = (!m0) & (!m1);
            const int idx0 = e1 | (e2 << 1);
            const int idx1 = (e0 | e2 | m3) | ((e1 | (!m1)) << 1);
            word |= (uint32_t)(idx0 | (idx1 << 2)) << (4 * q);
            const int64_t so = r * (k / 2) + (c * QPE + q) * (KS / 2);
            if (KS == 4) {
                T a = v[0], b = v[1];
                // select by index without dynamic register indexing
                a = (idx0 == 1) ? v[1] : ((idx0 == 2) ? v[2] : v[0]);
                b = (idx1 == 1) ? v[1] : ((idx1 == 2) ? v[2] : v[KS - 1]);
                sparse[so] = a;
                sparse[so + 1] = b;
            } else {
                sparse[so] = (idx0 / 2 == 0) ? v[0] : v[KS - 1];
            }
        }
        const int64_t off = meta_offset(r, c, m, MB);
        if (MB == 2) reinterpret_cast<int16_t*>(mout)[off] = (int16_t)word;
        else reinterpret_cast<int32_t*>(mout)[off] = (int32_t)word;
    }
}

// sparse [m, kh] in ES-byte units (fp32 data is moved as pairs of 16-bit halves) -> dense [m, 2 kh]
template <int ES, int MB>
__global__ void __launch_bounds__(256) semi_to_dense_kernel(const void* __restrict__ sin, const void* __restrict__ min_, void* __restrict__ dout,
                                                            int64_t m, int64_t kh, int64_t ncols) {
    using T = typename Raw<ES>::T;
    constexpr int QPE = MB * 2;
    const T* sparse = reinterpret_cast<const T*>(sin);
    T* dense = reinterpret_cast<T*>(dout);
    const int64_t total = m * ncols;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / ncols, c = t - r * ncols;
        const int64_t off = meta_offset(r, c, m, MB);
        const uint32_t word = (MB == 2) ? (uint32_t)(uint16_t)reinterpret_cast<const int16_t*>(min_)[off] : (uint32_t)reinterpret_cast<const int32_t*>(min_)[off];
#pragma unroll
        for (int q = 0; q < QPE; ++q) {
            const int idx0 = (word >> (4 * q)) & 3, idx1 = (word >> (4 * q + 2)) & 3;
            const int64_t quad = c * QPE + q;
            const T a = sparse[r * kh + quad * 2], b = sparse[r * kh + quad * 2 + 1];
            T* d = dense + r * 2 * kh + quad * 4;
#pragma unroll
            for (int i = 0; i < 4; ++i) d[i] = (i == idx1) ? b : ((i == idx0) ? a : (T)0);   // idx1 written last, like scatter_
        }
    }
}

}  // namespace ctb

extern "C" {

int ct_semi_structured_from_dense(const void* dense, int dtype, void* sparse, void* meta, int64_t m, int64_t k, int device, void* stream) {
    PRECHECK(device);
    const int mb = (dtype == CT_I8) ? 4 : 2;
    const int ks = (dtype == CT_F32) ? 2 : 4;
    if (m % 64 != 0) { set_error("semi-structured layout needs rows %% 64 == 0 (got %lld)", (long long)m); return CT_E_SHAPE; }
    if (k % (ks * mb * 2) != 0) { set_error("Number of columns of dense matrix %lld must be divisible by %d", (long long)k, ks * mb * 2); return CT_E_SHAPE; }
    if (m * k == 0) return CT_OK;
    if (!dense || !sparse || !meta) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t ncols = k / (ks * mb * 2);
    const unsigned g = grid_for(m * ncols);
    switch (dtype) {
    case CT_I8: semi_from_dense_kernel<CT_I8, 1, 4, 4><<<g, 256, 0, st>>>(dense, sparse, meta, m, k, ncols); break;
    case CT_F16: semi_from_dense_kernel<CT_F16, 2, 4, 2><<<g, 256, 0, st>>>(dense, sparse, meta, m, k, ncols); break;
    case CT_BF16: semi_from_dense_kernel<CT_BF16, 2, 4, 2><<<g, 256, 0, st>>>(dense, sparse, meta, m, k, ncols); break;
    case CT_F32: semi_from_dense_kernel<CT_F32, 4, 2, 2><<<g, 256, 0, st>>>(dense, sparse, meta, m, k, ncols); break;
    default: set_error("Invalid datatype %d of dense matrix", dtype); return CT_E_DTYPE;
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

/* k = number of sparse columns; dense is [m, 2k] */
int ct_semi_structured_to_dense(const void* sparse, int dtype, const void* meta, void* dense, int64_t m, int64_t k, int device, void* stream) {
    PRECHECK(device);
    const int mb = (dtype == CT_I8) ? 4 : 2;
    const int64_t kh = (dtype == CT_F32) ? 2 * k : k;
    if (m % 64 != 0) { set_error("semi-structured layout needs rows %% 64 == 0 (got %lld)", (long long)m); return CT_E_SHAPE; }
    if ((2 * kh) % (4 * mb * 2) != 0) { set_error("sparse column count %lld inconsistent with the metadata layout", (long long)k); return CT_E_SHAPE; }
    if (m * k == 0) return CT_OK;
    if (!dense || !sparse || !meta) { set_error("null pointer"); return CT_E_ARG; }
    const int64_t ncols = 2 * kh / (4 * mb * 2);
    const unsigned g = grid_for(m * ncols);
    switch (dtype) {
    case CT_I8: semi_to_dense_kernel<1, 4><<<g, 256, 0, st>>>(sparse, meta, dense, m, kh, ncols); break;
    case CT_F16: case CT_BF16: case CT_F32: semi_to_dense_kernel<2, 2><<<g, 256, 0, st>>>(sparse, meta, dense, m, kh, ncols); break;
    default: set_error("Invalid datatype %d of sparse matrix", dtype); return CT_E_DTYPE;
    }
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

}  // extern "C"

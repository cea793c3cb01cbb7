// bitmask_onepass.cu -- unstructured bitmask compression / expansion in ONE pass over the dense tensor.
//
//   format (CompressionFormat.sparse_bitmask, config/base.py:17; restated in oracle/ct_oracle.c, "parity unpinned"):
//       values = x[x != 0] row-major, bitmask = pack_bitmasks(x != 0) (utils/helpers.py:306-317), row_offsets = exclusive prefix of the
//       per-row counts, nnz = values.numel()
//
// Stream compaction needs a device-wide exclusive scan of the per-tile non-zero counts.  The two-phase kernels of sparse.cu
// (count -> cub scan -> move) read the dense tensor twice and need the host to learn nnz before `values` can be allocated.  Here the
// scan is a DECOUPLED LOOK-BACK over one 64-bit descriptor per tile ({status, count} in a single word, so publishing it needs no
// fence): a tile publishes its own count as soon as it has it, then sums its predecessors' descriptors backwards until it meets one
// that already holds an inclusive prefix.  Tiles are claimed from a ticket counter, so every predecessor of a running tile has
// itself been claimed by a resident CTA (forward progress).  The dense tensor is read exactly once:
//       compress  : 2 B in + 2 B x density out + 1/8 B mask per element  (3.125 B at 50 % zeros)
//       expand    : 1/8 B mask + 2 B x density in, 2 B out
// `values` is written into a caller buffer of capacity rows * cols; nnz stays on the device.
//
// Work decomposition (2-byte dtypes, cols % 8 == 0): unit = 8 elements = one 16-byte access and one mask byte; tile = 128 threads x 8
// units, scan order = unit order.  The kept elements of a tile are staged in shared memory so that the compact side is moved coalesced.
//
// Why the kernels are shaped as they are:
//   * One tile per CTA, its ticket taken when the CTA starts, so processing order is ticket order.  A CTA that claims a ticket ahead of
//     its work (a persistent CTA that prefetches its next tile) publishes that tile's count late, and every successor waits for it.
//   * The whole CTA looks back, politely: each predecessor's descriptor is read once per round, and a round is repeated after a
//     nanosleep only while a descriptor that is actually needed is unpublished.  Threads that spin on their descriptors saturate the
//     L2 and stretch the very round trip the prefix frontier advances by.
//   * Compression publishes its tile's count as soon as it is known and collects its prefix only after the gather: by then the
//     predecessors have mostly published, so the wait overlaps the tile's own work instead of preceding it.
//   * A tile lives through mostly serial latencies (ticket, bulk load, barriers, descriptor read, write-out), so what counts is how
//     many tiles an SM keeps in flight.  A scatter from a register-resident tile needs fewer instructions than the gather in shared
//     memory, but 72 registers per thread instead of 32 (sm_90a) and so fewer CTAs per SM; measured on the B200 it was slower.

#include "engine.h"

namespace ctb {

constexpr int BM_THREADS = 128;                    // threads per CTA
constexpr int BM_WARPS = BM_THREADS / 32;
constexpr int BM_UPT = 8;                          // units per thread
constexpr int BM_TILE = BM_UPT * BM_THREADS;       // units per tile (16 KB of bf16)

constexpr unsigned long long DESC_A = 1ull << 62;   // value = this tile's count
constexpr unsigned long long DESC_P = 2ull << 62;   // value = inclusive prefix up to and including this tile
constexpr unsigned long long DESC_VAL = (1ull << 62) - 1;

__device__ __forceinline__ unsigned long long ld_desc(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_desc(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr));
    return v;
}

// exclusive prefix of `tile` (sum of the counts of all tiles before it); every thread of the CTA takes part and returns it.
// Thread t inspects tile base - t; warp w therefore covers distances 32 w .. 32 w + 31, nearest first.
// PUBLISH = false: the caller published the aggregate itself (lookback_publish), earlier.
__device__ __forceinline__ void lookback_publish(unsigned long long* desc, uint32_t tile, uint32_t total) {
    if (threadIdx.x == 0) st_desc(desc + tile, (tile == 0 ? DESC_P : DESC_A) | (unsigned long long)total);
}
template <bool PUBLISH = true>
__device__ __forceinline__ unsigned long long lookback_cta(unsigned long long* desc, uint32_t tile, uint32_t total, unsigned long long* lb_sum, int* lb_p) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (PUBLISH) lookback_publish(desc, tile, total);
    unsigned long long excl = 0;
    if (tile == 0) return 0;
    int64_t base = (int64_t)tile - 1;
    while (true) {
        const int64_t idx = base - (int64_t)threadIdx.x;
        unsigned long long d = DESC_P;                 // before the first tile: prefix 0
        if (idx >= 0) d = ld_desc(desc + idx);
        // a descriptor matters only if no nearer one already holds a prefix: nearer lanes of this warp, or any nearer warp
        while (true) {
            const uint32_t has_p = __ballot_sync(0xffffffffu, (d >> 62) == 2);
            const uint32_t is_x = __ballot_sync(0xffffffffu, (d >> 62) == 0);
            const uint32_t needed = has_p ? ((2u << (__ffs(has_p) - 1)) - 1u) : 0xffffffffu;     // lanes up to the nearest prefix
            if ((is_x & needed) == 0) break;
            __nanosleep(40);
            if ((d >> 62) == 0) d = ld_desc(desc + idx);   // only the unpublished ones are read again
        }
        const uint32_t has_p = __ballot_sync(0xffffffffu, (d >> 62) == 2);
        const int stop = has_p ? (__ffs(has_p) - 1) : 31;
        unsigned long long part = (lane <= stop) ? (d & DESC_VAL) : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        if (lane == 0) { lb_sum[warp] = part; lb_p[warp] = has_p != 0; }
        __syncthreads();
        bool found = false;
#pragma unroll
        for (int w = 0; w < BM_WARPS; ++w) {
            if (!found) { excl += lb_sum[w]; found = lb_p[w] != 0; }
        }
        __syncthreads();
        if (found) break;
        base -= BM_THREADS;
    }
    if (threadIdx.x == 0) st_desc(desc + tile, DESC_P | (excl + (unsigned long long)total));
    return excl;
}

// per-thread scan bookkeeping shared by both directions: counts of the thread's 8 units (unit k * 128 + t, scan order = unit order)
// -> off[k] = first slot of unit k in the tile's compact run; returns the tile's total
__device__ __forceinline__ int tile_scan(const int (&cnt)[BM_UPT], int (&off)[BM_UPT], int (*warp_tot)[BM_WARPS]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl[BM_UPT];
#pragma unroll
    for (int k = 0; k < BM_UPT; ++k) incl[k] = cnt[k];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
        for (int k = 0; k < BM_UPT; ++k) {
            const int n = __shfl_up_sync(0xffffffffu, incl[k], o);
            if (lane >= o) incl[k] += n;
        }
    }
    if (lane == 31) {
#pragma unroll
        for (int k = 0; k < BM_UPT; ++k) warp_tot[k][warp] = incl[k];
    }
    __syncthreads();
    int total = 0;
#pragma unroll
    for (int k = 0; k < BM_UPT; ++k) {
        int before = 0, seg = 0;
#pragma unroll
        for (int w = 0; w < BM_WARPS; ++w) {
            const int t = warp_tot[k][w];
            if (w < warp) before += t;
            seg += t;
        }
        off[k] = total + before + incl[k] - cnt[k];
        total += seg;
    }
    return total;
}

// the compact run [excl, excl + total) from the staging buffer (run element j at stage element j) to `values`, as 16-byte vectors aligned
// to GLOBAL 16-byte boundaries.  The run starts at an arbitrary element, so global vector c holds stage elements [8c - shift, 8c - shift + 8)
// (shift = excl mod 8, tile-uniform); its first and last vector are stored element by element, because their other elements belong to
// the neighbouring tiles.  A vector's window is fetched as five 4-byte words from the 4-byte boundary at or below its first element (one
// funnel shift by 16 when the run position is odd); two 16-byte loads and a switch over the word offset compile to a select tree.  May
// read up to 16 bytes BELOW stage0 (vector 0 of a run that does not start on a 16-byte boundary; those halves are never stored): the
// caller's buffer is preceded by >= 16 bytes of its own shared memory.
__device__ __forceinline__ void run_to_global_words(uint16_t* values, unsigned long long excl, int total, uint32_t stage0) {
    const uint32_t shift = (uint32_t)(excl & 7ull);
    const unsigned long long g0 = excl - shift;
    const uint32_t span = shift + (uint32_t)total;
    const uint32_t nvec = (span + 7) >> 3;
    uint4* gv = reinterpret_cast<uint4*>(values + g0);
    const uint32_t sh = (shift & 1u) << 4;
    const uint32_t base = stage0 - 2u * shift - 2u * (shift & 1u);        // word that holds stage element -shift (4-byte aligned)
    for (uint32_t c = threadIdx.x; c < nvec; c += BM_THREADS) {
        const bool first = (c == 0), last = (8 * c + 8 > span);
        const uint32_t a = base + 16u * c;
        uint32_t w[5], o[4];
#pragma unroll
        for (int i = 0; i < 5; ++i) asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[i]) : "r"(a + 4u * i));
#pragma unroll
        for (int i = 0; i < 4; ++i) o[i] = __funnelshift_r(w[i], w[i + 1], sh);
        if (!first && !last) stg_stream16(gv + c, make_uint4(o[0], o[1], o[2], o[3]));
        else {
            uint16_t* ge = values + g0 + 8ull * c;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const uint32_t pos = 8 * c + e;
                if (pos >= shift && pos < span) ge[e] = (uint16_t)(o[e >> 1] >> (16 * (e & 1)));
            }
        }
    }
}

// non-zero byte of 8 halves: per word  min(|x| per half, 1)  ->  bit 0 / bit 16; folded into 8 bits
__device__ __forceinline__ uint32_t nz_byte16_fast(const uint4& v) {
    const uint32_t r0 = __vminu2(v.x & 0x7fff7fffu, 0x00010001u), r1 = __vminu2(v.y & 0x7fff7fffu, 0x00010001u);
    const uint32_t r2 = __vminu2(v.z & 0x7fff7fffu, 0x00010001u), r3 = __vminu2(v.w & 0x7fff7fffu, 0x00010001u);
    const uint32_t t = r0 + r1 * 4u + r2 * 16u + r3 * 64u;        // even elements at bits 0,2,4,6; odd ones at 16,18,20,22
    return (t | (t >> 15)) & 0xffu;
}
// popcount of every byte of x, in that byte
__device__ __forceinline__ uint32_t byte_popc4(uint32_t x) {
    x = x - ((x >> 1) & 0x55555555u);
    x = (x & 0x33333333u) + ((x >> 2) & 0x33333333u);
    return (x + (x >> 4)) & 0x0f0f0f0fu;
}

// ------------------------------------------------------------------------------------------------------------------------------
// Compression.  The tile arrives in shared memory with one bulk copy; thread t owns its 8 consecutive units 8 t .. 8 t + 7.
//   A: mask bytes, the thread's count, the CTA scan; the tile's count is published at once.
//   B: the tile's run is cut into vectors of 8 kept elements, aligned to the start of the RUN (not to global 16-byte boundaries, which
//      would need the prefix); the thread that owns a vector's first element records where that element sits in the tile.
//   C: one thread per vector walks the mask from there and gathers its 8 kept elements, compacting the tile in place.
//   D: the prefix (published by now), row offsets, and the write-out of the run to globally aligned vectors (run_to_global_words).
// ------------------------------------------------------------------------------------------------------------------------------
constexpr uint32_t BM_SMEM = 16 + BM_TILE * 16 + 32;    // + two vectors of slack: the write-out reads up to one vector past the run

__global__ void __launch_bounds__(BM_THREADS) bitmask_compress_late_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ bitmask,
                                                                           uint16_t* __restrict__ values, int64_t* __restrict__ row_offsets,
                                                                           int64_t* __restrict__ nnz_out, unsigned long long* __restrict__ desc,
                                                                           uint32_t* __restrict__ ticket, uint32_t n_units, uint32_t n_tiles, FastDiv upr) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    __shared__ __align__(16) uint32_t mask_w[BM_TILE / 4 + 4];   // the tile's mask bytes (+ zero padding for the walkers' look-ahead)
    __shared__ uint16_t start_s[BM_TILE + 8];                     // element index (within the tile) of the first element of run vector v
    __shared__ int warp_tot[BM_WARPS];
    __shared__ unsigned long long lb_sum[BM_WARPS];
    __shared__ int lb_p[BM_WARPS];
    __shared__ uint32_t tile_s;
    const uint32_t sbase = smem_u32(smem_raw);
    const uint32_t bar = sbase, data = sbase + 16;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        const uint32_t tile = atomicAdd(ticket, 1u);
        tile_s = tile;
        mbar_init_a(bar, 1);
        mbar_fence_init();
        const uint32_t nu = min((uint32_t)BM_TILE, n_units - tile * BM_TILE);
        mbar_expect_tx_a(bar, nu * 16);
        bulk_g2s_a(data, src + (size_t)tile * (BM_TILE * 16), nu * 16, bar, l2_evict_first_policy());
    }
    if (tid < 4) mask_w[BM_TILE / 4 + tid] = 0u;
    __syncthreads();
    const uint32_t tile = tile_s;
    const uint32_t u0 = tile * BM_TILE;
    const uint32_t nu = min((uint32_t)BM_TILE, n_units - u0);
    mbar_wait_a(bar, 0);

    // ---- A: mask bytes of the thread's 8 consecutive units, counts, scan ----
    const uint32_t uf = 8u * (uint32_t)tid;
    uint8_t* mask_b = reinterpret_cast<uint8_t*>(mask_w);
    {
        const uint32_t sw = (uint32_t)(tid & 7);
        const uint32_t tdata = data + uf * 16;
        uint8_t* tmask = mask_b + uf;
        if (nu == (uint32_t)BM_TILE) {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t p = (uint32_t)k ^ sw;
                tmask[p] = (uint8_t)nz_byte16_fast(lds128(tdata + p * 16));
            }
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const uint32_t p = (uint32_t)k ^ sw;
                uint32_t b = 0;
                if (uf + p < nu) b = nz_byte16_fast(lds128(tdata + p * 16));
                tmask[p] = (uint8_t)b;
            }
        }
    }
    const uint32_t lo = mask_w[2 * tid], hi = mask_w[2 * tid + 1];
    if (uf + 4 <= nu) reinterpret_cast<uint32_t*>(bitmask + u0 + uf)[0] = lo;
    if (uf + 8 <= nu) reinterpret_cast<uint32_t*>(bitmask + u0 + uf)[1] = hi;
    const int clo = __popc(lo), cnt = clo + __popc(hi);
    int incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < BM_WARPS; ++w) {
        const int t = warp_tot[w];
        if (w < warp) before += t;
        total += t;
    }
    const int toff = before + incl - cnt;
    lookback_publish(desc, tile, (uint32_t)total);        // the successors' look-back can pass this tile from here on

    // ---- B: run vector v starts at run element 8 v; the thread that owns that element records where it sits in the tile ----
    // Unit by unit (8 fixed steps, no data-dependent trip count): a unit holds <= 8 kept elements, so at most one vector boundary
    // (run index = 0 mod 8) falls into it -- r kept elements into the unit, an 8-bit select.  The per-unit counts and their running sums
    // come from one byte-wise popcount and one multiply per mask word.  (The first form looped over the thread's boundaries with a
    // 32-bit select each: 28 % of the kernel's instructions, and a warp ran as long as its busiest lane.)
    const uint32_t nvec = ((uint32_t)total + 7) >> 3;
    if (cnt > 0) {
        const uint32_t clo4 = byte_popc4(lo), chi4 = byte_popc4(hi);
        const uint32_t plo = clo4 * 0x01010101u, phi = chi4 * 0x01010101u + (uint32_t)clo * 0x01010101u;   // inclusive, <= 64 per byte
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int sh = 8 * (k & 3);
            const uint32_t cntk = ((k < 4 ? clo4 : chi4) >> sh) & 0xffu;
            const uint32_t first = (uint32_t)toff + (((k < 4 ? plo : phi) >> sh) & 0xffu) - cntk;   // run index of the unit's first kept element
            const uint32_t r = (0u - first) & 7u;
            if (r < cntk) {
                uint32_t x = ((k < 4 ? lo : hi) >> sh) & 0xffu, n = r, pos = 0;
#pragma unroll
                for (int w = 4; w >= 1; w >>= 1) {
                    const uint32_t c = __popc(x & ((1u << w) - 1u));
                    if (n >= c) { n -= c; x >>= w; pos += w; }
                }
                start_s[(first + r) >> 3] = (uint16_t)((uf + k) * 8 + pos);
            }
        }
    }
    __syncthreads();

    // ---- C: gather, in place.  Pass k: vectors T k .. T k + T - 1 (T threads) are read into registers, barrier, written to elements 8 v .. 8 v + 7.
    // A source element is never below its destination, and the sources of LATER passes lie at or above the end of this pass's
    // destinations, so one barrier per pass is enough.
    for (uint32_t vb = 0; vb < nvec; vb += BM_THREADS) {
        const uint32_t v = vb + (uint32_t)tid;
        uint32_t h[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) h[e] = 0u;
        if (v < nvec) {
            const uint32_t bit = start_s[v];
            uint32_t wi = bit >> 5;
            const uint32_t s = bit & 31u;
            uint32_t cur = __funnelshift_r(mask_w[wi], mask_w[wi + 1], s);      // kept-flags of elements bit .. bit + 31
            uint32_t ebase = data + bit * 2;                                     // shared address of element `bit`
            if (8 * v + 8 <= (uint32_t)total) {
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    while (cur == 0u) {                                          // the next kept element is further than 32 positions away
                        ++wi;
                        ebase += 64;
                        cur = __funnelshift_r(mask_w[wi], mask_w[wi + 1], s);
                    }
                    const uint32_t pos = (uint32_t)__ffs(cur) - 1u;
                    cur &= cur - 1u;
                    unsigned short t;
                    asm volatile("ld.shared.u16 %0, [%1];" : "=h"(t) : "r"(ebase + 2 * pos));
                    h[e] = t;
                }
            } else {
                const uint32_t ne = (uint32_t)total - 8 * v;                     // the run's last vector: 1 .. 7 elements
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    if ((uint32_t)e < ne) {
                        while (cur == 0u) {
                            ++wi;
                            ebase += 64;
                            cur = __funnelshift_r(mask_w[wi], mask_w[wi + 1], s);
                        }
                        const uint32_t pos = (uint32_t)__ffs(cur) - 1u;
                        cur &= cur - 1u;
                        unsigned short t;
                        asm volatile("ld.shared.u16 %0, [%1];" : "=h"(t) : "r"(ebase + 2 * pos));
                        h[e] = t;
                    }
                }
            }
        }
        __syncthreads();
        if (v < nvec)
            asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(data + 16u * v), "r"(h[0] | (h[1] << 16)), "r"(h[2] | (h[3] << 16)),
                         "r"(h[4] | (h[5] << 16)), "r"(h[6] | (h[7] << 16))
                         : "memory");
    }
    __syncthreads();

    // ---- D: the prefix (published long ago by now), row offsets, write-out ----
    const unsigned long long excl = lookback_cta<false>(desc, tile, (uint32_t)total, lb_sum, lb_p);
    if (tid == 0 && tile == n_tiles - 1) *nnz_out = (int64_t)(excl + (unsigned long long)total);
    if (row_offsets && uf < nu) {
        const uint32_t g = u0 + uf;
        uint32_t r = fd_div(g, upr);
        uint32_t k = (r * upr.d == g) ? 0u : (r + 1) * upr.d - g;          // units until the next row start
        if (k != 0) ++r;
        while (k < 8 && uf + k < nu) {
            const uint32_t below = (k < 4) ? __popc(lo & ((1u << (8 * k)) - 1u)) : (uint32_t)clo + __popc(hi & ((1u << (8 * (k - 4))) - 1u));
            row_offsets[r] = (int64_t)(excl + (unsigned long long)toff + below);
            k += upr.d;
            ++r;
        }
    }
    run_to_global_words(values, excl, total, data);
}

// expansion: mask bytes -> counts -> scan -> look-back -> the tile's run of `values` into shared memory (aligned 16-byte loads, so that
// run element j sits at stage element j + shift) -> dense tile, 16-byte stores
__global__ void __launch_bounds__(BM_THREADS) bitmask_expand_tile_kernel(const uint16_t* __restrict__ values, const uint8_t* __restrict__ bitmask,
                                                                         uint4* __restrict__ dense, unsigned long long* __restrict__ desc,
                                                                         uint32_t* __restrict__ ticket, uint32_t n_units, uint32_t n_tiles) {
    __shared__ __align__(16) uint16_t stage[8 * BM_TILE + 16];
    __shared__ uint32_t mask_s[BM_TILE / 4];
    __shared__ int warp_tot[BM_UPT][BM_WARPS];
    __shared__ unsigned long long lb_sum[BM_WARPS];
    __shared__ int lb_p[BM_WARPS];
    __shared__ uint32_t tile_s;
    const int tid = threadIdx.x;
    if (tid == 0) tile_s = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t tile = tile_s;
    const uint32_t u0 = tile * BM_TILE;
    const uint32_t nu = min((uint32_t)BM_TILE, n_units - u0);
    // the tile's mask bytes: 2 coalesced words per thread (n_units % 4 == 0)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const uint32_t wi = j * BM_THREADS + tid;
        mask_s[wi] = (wi * 4 < nu) ? __ldg(reinterpret_cast<const uint32_t*>(bitmask + u0) + wi) : 0u;
    }
    __syncthreads();
    uint32_t bytes_lo = 0, bytes_hi = 0;
    int cnt[BM_UPT], off[BM_UPT];
#pragma unroll
    for (int k = 0; k < BM_UPT; ++k) {
        const uint32_t i = k * BM_THREADS + tid;
        const uint32_t b = (i < nu) ? reinterpret_cast<const uint8_t*>(mask_s)[i] : 0u;
        if (k < 4) bytes_lo |= b << (8 * k);
        else bytes_hi |= b << (8 * (k - 4));
        cnt[k] = __popc(b);
    }
    const int total = tile_scan(cnt, off, warp_tot);
    const unsigned long long excl = lookback_cta(desc, tile, (uint32_t)total, lb_sum, lb_p);

    const uint32_t shift = (uint32_t)(excl & 7ull);
    const uint32_t nvec = (shift + (uint32_t)total + 7) >> 3;
    const uint4* gv = reinterpret_cast<const uint4*>(values + (excl - shift));
    const uint32_t span = shift + (uint32_t)total;
    for (uint32_t c = tid; c < nvec; c += BM_THREADS) {
        if (8 * c + 8 <= span) reinterpret_cast<uint4*>(stage)[c] = ldg_stream16(gv + c);    // c == 0 may include up to 7 elements of the previous tile's run
        else {
            for (uint32_t pos = 8 * c; pos < span; ++pos) stage[pos] = values[excl - shift + pos];   // the last vector: never read past the run (= past `values`)
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BM_UPT; ++k) {
        const uint32_t i = k * BM_THREADS + tid;
        if (i < nu) {
            const uint32_t b = (k < 4 ? bytes_lo >> (8 * k) : bytes_hi >> (8 * (k - 4))) & 0xffu;
            uint32_t e[8];
            int o = (int)shift + off[k];
#pragma unroll
            for (int q = 0; q < 8; ++q) e[q] = ((b >> q) & 1u) ? (uint32_t)stage[o++] : 0u;
            stg_stream16(dense + u0 + i, make_uint4(e[0] | (e[1] << 16), e[2] | (e[3] << 16), e[4] | (e[5] << 16), e[6] | (e[7] << 16)));
        }
    }
}

bool bitmask_lookback_ok(int dtype, int64_t rows, int64_t cols, const void* dense, const void* mask, const void* values) {
    const int64_t n_units = rows * cols / 8;
    return dt_size(dtype) == 2 && cols % 8 == 0 && n_units % 4 == 0 && n_units > 0 && n_units < 0x7fffffffLL && aligned16(dense) &&
           (reinterpret_cast<uintptr_t>(mask) & 3u) == 0 && aligned16(values);
}

// scratch of one launch: [16 B ticket][n_tiles descriptors], zeroed; stream-ordered like the job tables of dispatch.cu
template <bool COMPRESS>
int launch_bitmask_lookback(const void* src, uint8_t* bitmask, void* dst, int64_t* row_offsets, int64_t* nnz_out, int64_t rows, int64_t cols,
                            int device, cudaStream_t st) {
    const int64_t n_units = rows * cols / 8;
    const uint32_t n_tiles = (uint32_t)((n_units + BM_TILE - 1) / BM_TILE);
    uint8_t* scratch = nullptr;
    const size_t bytes = 16 + (size_t)n_tiles * sizeof(unsigned long long);
    int rc = scratch_alloc(reinterpret_cast<void**>(&scratch), bytes, device, st);
    if (rc) return rc;
    CT_CUDA_TRY(cudaMemsetAsync(scratch, 0, bytes, st));
    unsigned long long* desc = reinterpret_cast<unsigned long long*>(scratch + 16);
    uint32_t* ticket = reinterpret_cast<uint32_t*>(scratch);
    if (COMPRESS) {
        CT_CUDA_TRY(cudaFuncSetAttribute(bitmask_compress_late_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BM_SMEM));
        bitmask_compress_late_kernel<<<n_tiles, BM_THREADS, BM_SMEM, st>>>(reinterpret_cast<const uint8_t*>(src), bitmask, reinterpret_cast<uint16_t*>(dst),
                                                                           row_offsets, nnz_out, desc, ticket, (uint32_t)n_units, n_tiles,
                                                                           make_fastdiv((uint64_t)(cols / 8)));
    } else {
        bitmask_expand_tile_kernel<<<n_tiles, BM_THREADS, 0, st>>>(reinterpret_cast<const uint16_t*>(src), bitmask, reinterpret_cast<uint4*>(dst),
                                                                   desc, ticket, (uint32_t)n_units, n_tiles);
    }
    count_launch();
    cudaFreeAsync(scratch, st);
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}
template int launch_bitmask_lookback<true>(const void*, uint8_t*, void*, int64_t*, int64_t*, int64_t, int64_t, int, cudaStream_t);
template int launch_bitmask_lookback<false>(const void*, uint8_t*, void*, int64_t*, int64_t*, int64_t, int64_t, int, cudaStream_t);

}  // namespace ctb

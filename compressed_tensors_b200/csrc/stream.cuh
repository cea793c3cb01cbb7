// stream.cuh -- the persistent streaming pipeline every hot-path op is instantiated on.
//
// Work decomposition (all hot-path ops are elementwise over a flat, contiguous tensor):
//   chunk = 8 consecutive elements
//   unit  = Op::GROUP consecutive chunks = one thread's piece of work.  GROUP is chosen per op so
//           that the thread's OUTPUT is one 16-byte store (4-bit packing: 32 elements -> 4 words;
//           1-byte codes: 16 elements) and the scale / reciprocal is fetched once per unit.
//   tile  = TILE_CHUNKS chunks = 8192 elements (16 KB of bf16) = one CTA's unit of work
//   job   = one tensor; a launch covers a table of jobs (whole-model batches); tiles are numbered
//           globally and CLAIMED from a device counter by a persistent grid of n_SM * ctas_per_sm CTAs
//           (dynamic schedule, see stream_tma_kernel; small launches keep a static round-robin deal).
//
// The pipeline is warp-specialised.  One producer lane issues 1-D bulk async copies
// (cp.async.bulk, the TMA engine without a tensor map; L2 priority per op, see InputEvictFirst) of
// whole input tiles into a ring of shared-memory stages, each guarded by a full/empty mbarrier pair (waits use the hardware
// suspend hint, so the idle producer does not burn issue slots).  NCW consumer warps wait on the
// full barrier, read their units from shared memory with bank-conflict-free swizzled LDS.128, do
// the arithmetic in registers and write with coalesced 16-byte streaming stores.  The scale loads
// of a tile are issued BEFORE the barrier wait and consumed after it.
#pragma once

#include "common.cuh"

namespace ctb {

constexpr int TILE_CHUNKS = 1024;   // default tile: 1024 chunks = 8192 elements (16 KB of bf16)
// An op may ask for another tile size (`static constexpr int TILE`).  The four headline 16-bit ops run on 2048-chunk tiles with a
// 3-stage x 2-CTA ring: half the per-tile bookkeeping of the consumer warps for the same bytes in flight.
constexpr int BIG_TILE_CHUNKS = 2048;
constexpr int CHUNK_ELEMS = 8;
constexpr int NCW = 8;              // consumer warps
constexpr int MAX_STAGES = 12;

struct Job {
    const uint8_t* in;     // streamed input
    const void* scale;
    const void* zp;
    uint8_t* out;
    uint32_t n_chunks;     // numel / 8
    uint32_t tile_begin;   // global id of this job's first tile
    uint32_t tile_end;
    uint32_t _pad;
    FastDiv dc;            // flat mode: chunks per scale element (scale index = chunk / dc); 2-D mode: chunks per column block
    // 2-D mode (BLOCK strategy, one-row group scales): sidx = (row / rd) * srs + (chunk_in_row / dc)
    FastDiv cpr;           // chunks per row (d == 0: flat mode)
    FastDiv rd;            // rows per scale row (block height; "infinite" for a one-row scale)
    uint32_t srs;          // scale row stride
    uint32_t _pad2;
    const void* aux;       // FP4 ops: the tensor's global scale (one float32) or nullptr
};

struct JobTable {
    const Job* jobs;       // device array when n > 1
    int n;
    Job one;               // inline copy when n == 1 (no table upload needed)
};

// launch-uniform constants
struct Common {
    uint32_t qmin2, qmax2;   // clamp bounds duplicated in both halves, in the compute dtype (16-bit T)
    float qmin, qmax;        // same as fp32
    int bits;
};

__device__ __forceinline__ uint32_t job_tile_end(const JobTable& t, int j) { return t.n == 1 ? t.one.tile_end : t.jobs[j].tile_end; }
// by-value copy: the job lives in registers until a tile of another tensor comes up
__device__ __forceinline__ Job job_at(const JobTable& t, int j) {
    if (t.n == 1) return t.one;
    return t.jobs[j];
}

// ------------------------------------------------------------------------------------
// Op concept:
//   static constexpr int IN_BYTES;     streamed input bytes per chunk (4, 8, 16 or 32)
//   static constexpr int GROUP;        chunks per unit (1, 2 or 4)
//   struct Raw;                        raw scale / zero-point bits of a unit (plain loads only)
//   static Raw prefetch(J, gc0);       issued BEFORE the data arrives; no dependent arithmetic
//   static void run(J, cm, raw, gc0, w[GROUP][IN_BYTES/4], off);   gc0 = first chunk of the unit;
//                                      w[k] holds chunk (k + off) mod GROUP (see swz_off)
//   optional:  struct Tile;  static Tile tile(J);   evaluated once per (thread, tile) and passed to run() as a 7th argument:
//                                      per-tensor constants that are too expensive to rebuild per unit
// ------------------------------------------------------------------------------------

template <class Op, class = void> struct HasTile { static constexpr bool value = false; };
template <class Op> struct HasTile<Op, decltype((void)sizeof(typename Op::Tile))> { static constexpr bool value = true; };
template <class Op, class = void> struct TileOf { static constexpr int value = TILE_CHUNKS; };
template <class Op> struct TileOf<Op, decltype((void)Op::TILE)> { static constexpr int value = Op::TILE; };
// L2 priority of the streamed input tiles: evict_first unless the op declares `static constexpr bool INPUT_EVICT_FIRST = false`.
// Measured on H100 (DESIGN §6): the 4:1 read:write mix of 16-bit quantize + pack runs 4% faster at the default priority,
// while the 1:2 mixes of dequantize and unpack run 0.5% slower without the hint.
template <class Op, class = void> struct InputEvictFirst { static constexpr bool value = true; };
template <class Op> struct InputEvictFirst<Op, decltype((void)Op::INPUT_EVICT_FIRST)> { static constexpr bool value = Op::INPUT_EVICT_FIRST; };
struct NoTile {};
template <class Op> __device__ __forceinline__ auto op_tile(const Job& J) {
    if constexpr (HasTile<Op>::value) return Op::tile(J);
    else return NoTile{};
}
template <class Op, class W, class T>
__device__ __forceinline__ void op_run(const Job& J, const Common& cm, const typename Op::Raw& r, uint32_t gc0, const W& w, int off, const T& tc) {
    if constexpr (HasTile<Op>::value) Op::run(J, cm, r, gc0, w, off, tc);
    else Op::run(J, cm, r, gc0, w, off);
}

template <int BYTES>
__device__ __forceinline__ void lds_chunk(uint32_t saddr, uint32_t (&w)[BYTES / 4]) {
    if constexpr (BYTES == 4) {
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w[0]) : "r"(saddr));
    } else if constexpr (BYTES == 8) {
        asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(w[0]), "=r"(w[1]) : "r"(saddr));
    } else if constexpr (BYTES == 16) {
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(saddr));
    } else {
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]) : "r"(saddr));
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7]) : "r"(saddr + 16));
    }
}

// Bank-conflict-free reads of a unit from shared memory: lane l reads chunk (k + swz_off(l)) mod GROUP
// in its k-th LDS.128, so the 8 lanes of a quarter warp always cover 8 different 16-byte bank groups
// (unit stride = GROUP * 16 bytes).  Register k of the thread therefore holds chunk (k + off) mod GROUP;
// the op rotates its per-chunk outputs back before the store (rotate_out below).
template <int GROUP>
__device__ __forceinline__ int swz_off(int lane) {
    if constexpr (GROUP == 4) return (lane >> 1) & 3;
    else if constexpr (GROUP == 2) return (lane >> 2) & 1;
    else return 0;
}
// o holds GROUP blocks of WPC words, block k belonging to chunk (k + off) mod GROUP: put them in chunk order
template <int GROUP, int WPC>
__device__ __forceinline__ void rotate_out(uint32_t (&o)[GROUP * WPC], int off) {
    if constexpr (GROUP == 2) {
        const bool sw = off & 1;
#pragma unroll
        for (int i = 0; i < WPC; ++i) {
            const uint32_t a = o[i], b = o[WPC + i];
            o[i] = sw ? b : a;
            o[WPC + i] = sw ? a : b;
        }
    } else if constexpr (GROUP == 4) {
        const bool r1 = off & 1, r2 = off & 2;
#pragma unroll
        for (int i = 0; i < WPC; ++i) {
            uint32_t a0 = o[i], a1 = o[WPC + i], a2 = o[2 * WPC + i], a3 = o[3 * WPC + i];
            // block k -> position k+1
            uint32_t b0 = r1 ? a3 : a0, b1 = r1 ? a0 : a1, b2 = r1 ? a1 : a2, b3 = r1 ? a2 : a3;
            // block k -> position k+2
            o[i] = r2 ? b2 : b0;
            o[WPC + i] = r2 ? b3 : b1;
            o[2 * WPC + i] = r2 ? b0 : b2;
            o[3 * WPC + i] = r2 ? b1 : b3;
        }
    }
}

// ------------------------------------------------------------------------------------
// TMA bulk-copy ring
// ------------------------------------------------------------------------------------
// Tile schedule.  `sched` != nullptr: DYNAMIC -- the producer lane of every CTA claims tile ids from a
// zero-initialised device counter with atomicAdd, one claim in flight ahead of its use.  A static
// round-robin deal makes the launch wait for the slowest SM: SMs do not all see the same memory
// bandwidth, so equal shares finish at different times (tools/ubench/mix_ceiling.cu compares the two).  `sched` == nullptr: static deal (launches of fewer than DYNAMIC_MIN_TILES_PER_SM tiles per SM, dispatch.cu).
// Either way the producer publishes {tile, next tile} of a stage in shared memory before it arms the
// stage's full barrier; consumers pick both up after the wait (release/acquire through the mbarrier).
constexpr uint32_t SMEM_HDR = 384;   // full[12] | empty[12] | ids[12] (8 bytes each), then the data ring

__device__ __forceinline__ void sts_v2(uint32_t saddr, uint32_t a, uint32_t b) {
    asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(saddr), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ void lds_v2(uint32_t saddr, uint32_t& a, uint32_t& b) {
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "r"(saddr) : "memory");
}

template <class Op>
__global__ void __launch_bounds__(32 * (NCW + 1)) stream_tma_kernel(const __grid_constant__ JobTable tbl,
                                                                   const __grid_constant__ Common cm,
                                                                   uint32_t total_tiles, int stages, uint32_t* sched) {
    constexpr int TILE_CHUNKS = TileOf<Op>::value;     // shadows the default on purpose: everything below is per-op
    constexpr int TILE_BYTES = TILE_CHUNKS * Op::IN_BYTES;
    constexpr int CTHREADS = NCW * 32;
    constexpr int G = Op::GROUP;
    constexpr int UNITS = TILE_CHUNKS / G;
    constexpr int ITERS = UNITS / CTHREADS;
    static_assert(UNITS % CTHREADS == 0, "tile must split evenly over the consumer threads");
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const uint32_t sbase = smem_u32(smem_raw);
    const uint32_t full0 = sbase;                        // full[s]  at sbase + 8 s
    const uint32_t empty0 = sbase + 8 * MAX_STAGES;      // empty[s] at sbase + 96 + 8 s
    const uint32_t ids0 = sbase + 16 * MAX_STAGES;       // ids[s]   at sbase + 192 + 8 s
    const uint32_t data0 = sbase + SMEM_HDR;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < stages; ++s) {
            mbar_init_a(full0 + 8 * s, 1);
            mbar_init_a(empty0 + 8 * s, NCW);
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == NCW) {
        // ---------------- producer ----------------
        if (lane == 0) {
            const uint64_t policy = l2_evict_first_policy();
            int s = 0, j = 0;
            uint32_t ph = 0;
            // cur / nxt are known, nn is the claim in flight
            uint32_t cur, nxt, nn;
            if (sched) {
                cur = atomicAdd(sched, 2u);
                nxt = cur + 1;                    // the first claim takes two tiles: both ids are needed at once
            } else {
                cur = blockIdx.x;
                nxt = cur + gridDim.x;
            }
            if (cur >= total_tiles) {             // nothing left for this CTA: tell the consumers
                sts_v2(ids0, cur, cur);
                mbar_arrive_a(full0);
            } else {
                Job J = job_at(tbl, 0);
                while (cur < total_tiles) {
                    if (sched) nn = (nxt < total_tiles) ? atomicAdd(sched, 1u) : nxt;
                    else nn = nxt + gridDim.x;
                    if (cur >= J.tile_end) {
                        while (cur >= job_tile_end(tbl, j)) ++j;
                        J = job_at(tbl, j);
                    }
                    const uint32_t lt = cur - J.tile_begin;
                    const uint32_t base = lt * TILE_CHUNKS;
                    const uint32_t chunks = min((uint32_t)TILE_CHUNKS, J.n_chunks - base);
                    const uint32_t bytes = chunks * Op::IN_BYTES;
                    mbar_wait_a(empty0 + 8 * s, ph ^ 1u);
                    sts_v2(ids0 + 8 * s, cur, nxt);
                    mbar_expect_tx_a(full0 + 8 * s, bytes);
                    if constexpr (InputEvictFirst<Op>::value)
                        bulk_g2s_a(data0 + (uint32_t)s * TILE_BYTES, J.in + (size_t)lt * TILE_BYTES, bytes, full0 + 8 * s, policy);
                    else
                        bulk_g2s_a(data0 + (uint32_t)s * TILE_BYTES, J.in + (size_t)lt * TILE_BYTES, bytes, full0 + 8 * s);
                    if (++s == stages) { s = 0; ph ^= 1u; }
                    cur = nxt;
                    nxt = nn;
                }
            }
        }
    } else {
        // ---------------- consumers ----------------
        const int ctid = threadIdx.x;  // 0 .. CTHREADS-1
        int s = 0, j = 0;
        uint32_t ph = 0;
        const int off = (Op::IN_BYTES == 16) ? swz_off<G>(lane) : 0;
        // The scale / zero-point loads run ONE TILE AHEAD of the arithmetic: they miss L2 (each is
        // used once) and would otherwise expose a full DRAM round trip per tile.
        Job Jn = job_at(tbl, 0);
        typename Op::Raw raw_next[ITERS];
        uint32_t tile, nxt;
        mbar_wait_a(full0, 0);
        lds_v2(ids0, tile, nxt);
        if (tile < total_tiles) {
            while (tile >= job_tile_end(tbl, j)) ++j;
            Jn = job_at(tbl, j);
            const uint32_t base = (tile - Jn.tile_begin) * TILE_CHUNKS;
            const uint32_t chunks = min((uint32_t)TILE_CHUNKS, Jn.n_chunks - base);
#pragma unroll
            for (int it = 0; it < ITERS; ++it) {
                const uint32_t c0 = (uint32_t)(it * CTHREADS + ctid) * G;
                if (c0 < chunks) raw_next[it] = Op::prefetch(Jn, base + c0);
            }
        }
        // per-tensor constants of the op (Op::tile): rebuilt only when the next tile belongs to another tensor
        decltype(op_tile<Op>(Jn)) tc{};
        bool new_job = true;
        while (tile < total_tiles) {
            // invariant: full[s] of `tile` has been waited for, `nxt` is the tile after it
            const Job J = Jn;
            const uint32_t base = (tile - J.tile_begin) * TILE_CHUNKS;
            const uint32_t chunks = min((uint32_t)TILE_CHUNKS, J.n_chunks - base);
            if (new_job) { tc = op_tile<Op>(J); new_job = false; }
            typename Op::Raw raw[ITERS];
#pragma unroll
            for (int it = 0; it < ITERS; ++it) raw[it] = raw_next[it];
            if (nxt < total_tiles) {
                if (nxt >= Jn.tile_end) {
                    while (nxt >= job_tile_end(tbl, j)) ++j;
                    Jn = job_at(tbl, j);
                    new_job = true;
                }
                const uint32_t nbase = (nxt - Jn.tile_begin) * TILE_CHUNKS;
                const uint32_t nchunks = min((uint32_t)TILE_CHUNKS, Jn.n_chunks - nbase);
#pragma unroll
                for (int it = 0; it < ITERS; ++it) {
                    const uint32_t c0 = (uint32_t)(it * CTHREADS + ctid) * G;
                    if (c0 < nchunks) raw_next[it] = Op::prefetch(Jn, nbase + c0);
                }
            }
            const uint32_t sp = data0 + (uint32_t)s * TILE_BYTES;
#pragma unroll
            for (int it = 0; it < ITERS; ++it) {
                const uint32_t c0 = (uint32_t)(it * CTHREADS + ctid) * G;
                if (c0 < chunks) {
                    uint32_t w[G][Op::IN_BYTES / 4];
#pragma unroll
                    for (int k = 0; k < G; ++k) lds_chunk<Op::IN_BYTES>(sp + (c0 + ((k + off) & (G - 1))) * Op::IN_BYTES, w[k]);
                    op_run<Op>(J, cm, raw[it], base + c0, w, off, tc);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive_a(empty0 + 8 * s);
            if (++s == stages) { s = 0; ph ^= 1u; }
            tile = nxt;
            if (tile >= total_tiles) break;
            mbar_wait_a(full0 + 8 * s, ph);
            uint32_t t2;
            lds_v2(ids0 + 8 * s, t2, nxt);
        }
    }
}

// ------------------------------------------------------------------------------------
// host-side launcher shared by all ops
// ------------------------------------------------------------------------------------
struct LaunchPlan {
    JobTable tbl;
    Common cm;
    uint32_t total_tiles;
    uint32_t* sched = nullptr;   // zeroed device counter for the dynamic tile schedule (nullptr = static deal); owned by dispatch.cu
};

// Ring shape of an op: its measured preference (`static constexpr int PREF_STAGES, PREF_CTAS`), 4 stages x 3 CTAs per SM for ops
// that declare none, cut to fit: stages in [2, MAX_STAGES], then stages and after them CTAs reduced until stages * tile * ctas
// stays within ~200 KB of shared memory per SM.
struct RingShape {
    int stages, ctas;
};
template <class Op, class = void> struct PrefRing { static constexpr RingShape value{4, 3}; };
template <class Op> struct PrefRing<Op, decltype((void)Op::PREF_CTAS)> { static constexpr RingShape value{Op::PREF_STAGES, Op::PREF_CTAS}; };
constexpr bool ring_fits(RingShape r, size_t tile_bytes) { return (size_t)r.stages * tile_bytes * r.ctas + 1024 * r.ctas <= 200 * 1024; }
template <class Op>
constexpr RingShape ring_shape() {
    constexpr size_t TILE_BYTES = (size_t)TileOf<Op>::value * Op::IN_BYTES;
    RingShape r = PrefRing<Op>::value;
    if (r.stages < 2) r.stages = 2;
    if (r.stages > MAX_STAGES) r.stages = MAX_STAGES;
    while (!ring_fits(r, TILE_BYTES) && r.stages > 2) --r.stages;
    while (!ring_fits(r, TILE_BYTES) && r.ctas > 1) --r.ctas;
    return r;
}

template <class Op>
int launch_stream(const LaunchPlan& lp, int device, cudaStream_t stream) {
    if (lp.total_tiles == 0) return CT_OK;
    constexpr size_t TILE_BYTES = (size_t)TileOf<Op>::value * Op::IN_BYTES;
    constexpr RingShape ring = ring_shape<Op>();
    static_assert(ring_fits(ring, TILE_BYTES), "the op's tile does not fit a ring in 200 KB of shared memory");
    constexpr size_t smem = SMEM_HDR + (size_t)ring.stages * TILE_BYTES;
    auto kfn = stream_tma_kernel<Op>;
    CT_CUDA_TRY(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    uint32_t grid = (uint32_t)(sm_count(device) * ring.ctas);
    if (grid > lp.total_tiles) grid = lp.total_tiles;
    kfn<<<grid, 32 * (NCW + 1), smem, stream>>>(lp.tbl, lp.cm, lp.total_tiles, ring.stages, grid < lp.total_tiles ? lp.sched : nullptr);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

// A streaming kernel as the host plans it: its launcher and the tile size the host counts the launch's tiles in.
// A null `launch` means there is no instantiation for what was asked.
struct StreamKernel {
    int (*launch)(const LaunchPlan&, int device, cudaStream_t);
    int tile_chunks;
};
template <class Op>
constexpr StreamKernel stream_kernel() { return {&launch_stream<Op>, TileOf<Op>::value}; }

}  // namespace ctb

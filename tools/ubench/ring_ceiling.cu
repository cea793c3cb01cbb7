// The W4A16 headline's memory pattern with no arithmetic: the ceiling of the streaming ring itself.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ring_ceiling ring_ceiling.cu && ./ring_ceiling
//
// Same shape as the headline launch (stream_tma_kernel on QuantPackOp<bf16, 4 bits, G = 4>):
//   * 6.98 G bf16 elements (the Llama-3-8B weight set, 13.96 GB) as one flat stream;
//   * 2048-chunk (32 KB) tiles, a 3-stage ring, 2 CTAs per SM, 8 consumer warps + 1 producer warp;
//   * one producer lane claims tiles from a device counter (one claim in flight) and issues one cp.async.bulk per tile with an
//     L2 evict_first policy;
//   * every consumer thread reads 2 units of 32 elements per tile with 4 swizzled LDS.128 each and writes 16 bytes per unit
//     (2 B read : 0.5 B written per element), the words XOR-folded instead of quantised.
// Variants, one knob at a time:
//   scales     one 2-byte g128 scale per unit, loaded one tile ahead with __ldg (the headline's Op::prefetch)
//   store      none (read-only ring) / plain st.global.L1::no_allocate / the same with an L2 evict_first cache hint /
//              a bulk-store epilogue (each tile's 8 KB of words staged in shared memory, one evict_first cp.async.bulk per tile)
//              / st.global.cs
//   read       one evict_first bulk load per tile (the default) / the same without an L2 hint / four 8 KB loads per tile /
//              plus an L2 prefetch of the tile the producer just claimed
//   early      the warp arrives on the stage's empty barrier after its loads, before its stores
// Times are compared with the headline through the headline's algorithmic bytes (2 + 0.5 + 2/128 B per element).
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

constexpr int NCW = 8;
constexpr int STAGES = 3;
constexpr int CTAS = 2;
constexpr int TILE_CHUNKS = 2048;                  // chunk = 8 bf16 = 16 bytes
constexpr int TILE_BYTES = TILE_CHUNKS * 16;
constexpr int G = 4;                               // chunks per unit
constexpr int CTHREADS = NCW * 32;
constexpr int ITERS = TILE_CHUNKS / G / CTHREADS;  // units per thread per tile (2)
constexpr int CHUNKS_PER_SCALE = 16;               // group size 128
constexpr uint32_t HDR = 128;                      // full[3] | empty[3] | ids[3], then the ring

constexpr int OUT_TILE = TILE_CHUNKS * 4;          // 8 KB of packed words per tile

enum Store { ST_NONE = 0, ST_PLAIN = 1, ST_EVICT_FIRST = 2, ST_BULK = 3, ST_CS = 4 };
// how the producer reads a tile
enum Read { RD_EVICT_FIRST = 0, RD_NO_HINT = 1, RD_SPLIT4 = 2, RD_PREFETCH = 3 };

__device__ __forceinline__ void mbar_init(uint32_t b, uint32_t n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(b), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(b) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t b, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t b, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra.uni WAIT_DONE;\n\t"
        "bra.uni WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t}" ::"r"(b), "r"(parity), "r"(0x989680u) : "memory");
}
__device__ __forceinline__ uint64_t evict_first() {
    uint64_t p;
    asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void sts_v2(uint32_t a, uint32_t x, uint32_t y) { asm volatile("st.shared.v2.u32 [%0], {%1,%2};" ::"r"(a), "r"(x), "r"(y) : "memory"); }
__device__ __forceinline__ void lds_v2(uint32_t a, uint32_t& x, uint32_t& y) { asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(x), "=r"(y) : "r"(a) : "memory"); }
__device__ __forceinline__ uint4 lds16(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
template <int ST>
__device__ __forceinline__ void store16(void* p, uint4 v) {
    if constexpr (ST == ST_PLAIN) {
        asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    } else if constexpr (ST == ST_EVICT_FIRST) {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w),
                     "l"(evict_first()) : "memory");
    } else if constexpr (ST == ST_CS) {
        asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
    }
}

template <bool SCALES, int ST, bool EARLY, int RD = RD_EVICT_FIRST>
__global__ void __launch_bounds__(32 * (NCW + 1)) ring(const uint8_t* __restrict__ in, const unsigned short* __restrict__ scale, uint8_t* __restrict__ out,
                                                       uint32_t total_tiles, uint32_t* ctr, uint32_t* sink) {
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t full0 = sbase, empty0 = sbase + 8 * STAGES, ids0 = sbase + 16 * STAGES, data0 = sbase + HDR;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full0 + 8 * s, 1);
            mbar_init(empty0 + 8 * s, NCW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == NCW) {
        if (lane != 0) return;
        const uint64_t policy = evict_first();
        int s = 0;
        uint32_t ph = 0, cur = atomicAdd(ctr, 2u), nxt = cur + 1, nn;
        if (cur >= total_tiles) {
            sts_v2(ids0, cur, cur);
            mbar_arrive(full0);
            return;
        }
        while (cur < total_tiles) {
            nn = (nxt < total_tiles) ? atomicAdd(ctr, 1u) : nxt;
            mbar_wait(empty0 + 8 * s, ph ^ 1u);
            sts_v2(ids0 + 8 * s, cur, nxt);
            mbar_expect_tx(full0 + 8 * s, TILE_BYTES);
            if constexpr (RD == RD_NO_HINT) {
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(data0 + s * TILE_BYTES),
                             "l"(in + (size_t)cur * TILE_BYTES), "r"(TILE_BYTES), "r"(full0 + 8 * s) : "memory");
            } else if constexpr (RD == RD_SPLIT4) {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(data0 + s * TILE_BYTES + q * (TILE_BYTES / 4)),
                                 "l"(in + (size_t)cur * TILE_BYTES + q * (TILE_BYTES / 4)), "r"(TILE_BYTES / 4), "r"(full0 + 8 * s), "l"(policy) : "memory");
            } else {
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(data0 + s * TILE_BYTES),
                             "l"(in + (size_t)cur * TILE_BYTES), "r"(TILE_BYTES), "r"(full0 + 8 * s), "l"(policy) : "memory");
            }
            if (RD == RD_PREFETCH && nn < total_tiles && nn != nxt)
                asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(in + (size_t)nn * TILE_BYTES), "r"(TILE_BYTES) : "memory");
            if (++s == STAGES) { s = 0; ph ^= 1u; }
            cur = nxt;
            nxt = nn;
        }
        return;
    }
    const int ctid = threadIdx.x;
    const int off = (lane >> 1) & 3;   // the headline's swizzle: the 8 lanes of a quarter warp hit 8 different 16-byte bank groups
    int s = 0;
    uint32_t ph = 0, tile, nxt, acc = 0, n_done = 0;
    uint32_t raw_next[ITERS] = {}, raw[ITERS];
    mbar_wait(full0, 0);
    lds_v2(ids0, tile, nxt);
    if (SCALES && tile < total_tiles) {
#pragma unroll
        for (int it = 0; it < ITERS; ++it) raw_next[it] = __ldg(scale + ((size_t)tile * TILE_CHUNKS + (it * CTHREADS + ctid) * G) / CHUNKS_PER_SCALE);
    }
    while (tile < total_tiles) {
#pragma unroll
        for (int it = 0; it < ITERS; ++it) raw[it] = raw_next[it];
        if (SCALES && nxt < total_tiles) {
#pragma unroll
            for (int it = 0; it < ITERS; ++it) raw_next[it] = __ldg(scale + ((size_t)nxt * TILE_CHUNKS + (it * CTHREADS + ctid) * G) / CHUNKS_PER_SCALE);
        }
        const uint32_t sp = data0 + s * TILE_BYTES;
        uint4 o[ITERS];
#pragma unroll
        for (int it = 0; it < ITERS; ++it) {
            const uint32_t c0 = (it * CTHREADS + ctid) * G;
            uint4 v = make_uint4(raw[it], 0, 0, 0);
#pragma unroll
            for (int k = 0; k < G; ++k) {
                const uint4 w = lds16(sp + (c0 + ((k + off) & (G - 1))) * 16);
                v.x ^= w.x; v.y ^= w.y; v.z ^= w.z; v.w ^= w.w;
            }
            o[it] = v;
            if (!EARLY && ST != ST_BULK) store16<ST>(out + ((size_t)tile * TILE_CHUNKS + c0) * 4, v);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * s);
        if constexpr (ST == ST_BULK) {
            // the tile's 8 KB of words go through a double-buffered staging area and leave with one bulk store; the barrier
            // after thread 0's wait frees the buffer the NEXT tile writes (the store issued one tile ago has read it)
            const uint32_t ob = data0 + STAGES * TILE_BYTES + (n_done & 1) * OUT_TILE;
#pragma unroll
            for (int it = 0; it < ITERS; ++it)
                asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(ob + (it * CTHREADS + ctid) * 16), "r"(o[it].x), "r"(o[it].y), "r"(o[it].z),
                             "r"(o[it].w) : "memory");
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            if (ctid == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            asm volatile("bar.sync 1, %0;" ::"r"(CTHREADS) : "memory");
            if (ctid == 0) {
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(out + (size_t)tile * OUT_TILE), "r"(ob),
                             "r"(OUT_TILE), "l"(evict_first()) : "memory");
                asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            }
            ++n_done;
        }
#pragma unroll
        for (int it = 0; it < ITERS; ++it) {
            if (EARLY && ST != ST_BULK) store16<ST>(out + ((size_t)tile * TILE_CHUNKS + (it * CTHREADS + ctid) * G) * 4, o[it]);
            if (ST == ST_NONE) acc ^= o[it].x ^ o[it].y ^ o[it].z ^ o[it].w;
        }
        if (++s == STAGES) { s = 0; ph ^= 1u; }
        tile = nxt;
        if (tile >= total_tiles) break;
        mbar_wait(full0 + 8 * s, ph);
        uint32_t t2;
        lds_v2(ids0 + 8 * s, t2, nxt);
    }
    if (ST == ST_BULK && ctid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    if (ST == ST_NONE && acc == 0x9e3779b9u) atomicAdd(sink, 1u);   // keeps the loads of the read-only ring alive
}

static int n_sms;

template <bool SCALES, int ST, bool EARLY, int RD = RD_EVICT_FIRST>
void run(const char* name, const uint8_t* in, const unsigned short* scale, uint8_t* out, uint32_t tiles, uint32_t* ctr, uint32_t* sink, double alg_bytes) {
    auto k = ring<SCALES, ST, EARLY, RD>;
    const int smem = HDR + STAGES * TILE_BYTES + (ST == ST_BULK ? 2 * OUT_TILE : 0);   // 2 x 114,816 B still fit an SM's 228 KB
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    int resident = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&resident, k, 32 * (NCW + 1), smem);
    if (resident < CTAS) {
        printf("{\"variant\": \"%s\", \"error\": \"%d CTAs per SM fit, the ring needs %d\"}\n", name, resident, CTAS);
        return;
    }
    cudaEvent_t a, b;
    cudaEventCreate(&a);
    cudaEventCreate(&b);
    const int reps = 10;
    float best = 1e9f, sum = 0.f;
    for (int it = 0; it < reps + 3; ++it) {
        cudaMemsetAsync(ctr, 0, 4);
        cudaEventRecord(a);
        k<<<n_sms * CTAS, 32 * (NCW + 1), smem>>>(in, scale, out, tiles, ctr, sink);
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        float ms;
        cudaEventElapsedTime(&ms, a, b);
        if (it >= 3) { sum += ms; if (ms < best) best = ms; }
    }
    const double moved = (double)tiles * TILE_BYTES * (1.0 + (ST != ST_NONE ? 0.25 : 0.0) + (SCALES ? 1.0 / 64 : 0.0));
    printf("{\"variant\": \"%s\", \"ms_best\": %.4f, \"ms_mean\": %.4f, \"alg_GBps_best\": %.1f, \"moved_GBps_best\": %.1f}\n", name, best, sum / reps,
           alg_bytes / best / 1e6, moved / best / 1e6);
    fflush(stdout);
    cudaEventDestroy(a);
    cudaEventDestroy(b);
}

int main() {
    const size_t n_elems = 6979321856ull;   // 32 Llama-3-8B layers x {q, k, v, o, gate, up, down}
    const uint32_t tiles = (uint32_t)(n_elems / 8 / TILE_CHUNKS);
    const double alg_bytes = n_elems * (2.0 + 0.5 + 2.0 / 128);
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    n_sms = prop.multiProcessorCount;
    uint8_t *in, *out;
    unsigned short* scale;
    uint32_t *ctr, *sink;
    if (cudaMalloc(&in, n_elems * 2) != cudaSuccess || cudaMalloc(&out, n_elems / 2) != cudaSuccess || cudaMalloc(&scale, n_elems / 64) != cudaSuccess ||
        cudaMalloc(&ctr, 4) != cudaSuccess || cudaMalloc(&sink, 4) != cudaSuccess) {
        printf("{\"status\": \"alloc failed\"}\n");
        return 1;
    }
    cudaMemset(in, 1, n_elems * 2);
    cudaMemset(out, 0, n_elems / 2);
    cudaMemset(scale, 2, n_elems / 64);
    printf("{\"device\": \"%s\", \"sms\": %d, \"elements\": %zu, \"tiles\": %u, \"alg_bytes\": %.0f}\n", prop.name, n_sms, n_elems, tiles, alg_bytes);
    run<true, ST_PLAIN, false>("scales+plain_store (the headline's pattern)", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<false, ST_PLAIN, false>("no_scales+plain_store", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_EVICT_FIRST, false>("scales+evict_first_store", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<false, ST_EVICT_FIRST, false>("no_scales+evict_first_store", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_PLAIN, true>("scales+plain_store+early_release", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_EVICT_FIRST, true>("scales+evict_first_store+early_release", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_PLAIN, false, RD_NO_HINT>("scales+plain_store, loads without L2 hint", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_PLAIN, false, RD_SPLIT4>("scales+plain_store, 4 bulk loads of 8 KB per tile", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_PLAIN, false, RD_PREFETCH>("scales+plain_store, L2 prefetch of the claimed tile", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_CS, false>("scales+st.global.cs", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_BULK, true>("scales+bulk_store_epilogue+early_release", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<false, ST_BULK, true>("no_scales+bulk_store_epilogue+early_release", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_NONE, false>("scales, read only (no stores)", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<false, ST_NONE, false>("no_scales, read only (no stores)", in, scale, out, tiles, ctr, sink, alg_bytes);
    run<true, ST_PLAIN, false>("scales+plain_store (repeat)", in, scale, out, tiles, ctr, sink, alg_bytes);
    const cudaError_t e = cudaDeviceSynchronize();
    printf("{\"status\": \"%s\"}\n", cudaGetErrorString(e));
    return e == cudaSuccess ? 0 : 1;
}

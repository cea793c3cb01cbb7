// common.cuh -- shared device/host helpers for the sm_90a kernels.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>
#include <vector>

#include "../../include/ct_b200.h"

namespace ctb {

// ------------------------------------------------------------------------------------
// error plumbing (thread-local message, never throws)
// ------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
void count_launch(int n = 1);

#define CT_CUDA_TRY(expr)                                   \
    do {                                                    \
        cudaError_t _e = (expr);                            \
        if (_e != cudaSuccess) return ctb::cuda_fail(_e, #expr); \
    } while (0)

constexpr int DYNAMIC_MIN_TILES_PER_SM = 24;   // below this many tiles per SM a launch keeps the static deal (no scratch, no memset)
constexpr int GRID_SMS = 132;   // SMs of an H100 SXM: grid size of the grid-stride kernels, sm_count() when the device is unknown
int sm_count(int device);
int64_t l2_bytes(int device);   // L2 cache size of the device (0 when unknown)
int scratch_alloc(void** p, size_t bytes, int device, cudaStream_t stream);   // stream-ordered, free with cudaFreeAsync

// Job tables of multi-job launches normally reach the device with one cudaMemcpyAsync from a host image -- a pageable-memory copy,
// which a stream capture rejects.  While the stream is being captured the table travels as KERNEL PARAMETERS instead (PER jobs per
// launch of a one-warp kernel; parameters are copied into the graph node at capture time), so a whole-model call can be captured
// once and replayed.
template <class J, int PER> struct JobBlock { J j[PER]; };
template <class J, int PER>
__global__ void upload_jobs_kernel(J* dst, const __grid_constant__ JobBlock<J, PER> blk, int n) {
    if ((int)threadIdx.x < n) dst[threadIdx.x] = blk.j[threadIdx.x];
}
// writes `head` zero bytes at dst, then jobs[0, n) (device memory, stream-ordered)
template <class J, int PER>
int upload_jobs(uint8_t* dst, size_t head, const J* jobs, size_t n, cudaStream_t stream) {
    static_assert(PER <= 32, "one thread per job of a block");
    cudaStreamCaptureStatus capturing = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(stream, &capturing);
    if (capturing == cudaStreamCaptureStatusActive) {
        if (head) CT_CUDA_TRY(cudaMemsetAsync(dst, 0, head, stream));
        for (size_t o = 0; o < n; o += PER) {
            JobBlock<J, PER> blk;
            const int cnt = (int)(n - o < (size_t)PER ? n - o : PER);
            memcpy(blk.j, jobs + o, (size_t)cnt * sizeof(J));
            upload_jobs_kernel<J, PER><<<1, 32, 0, stream>>>(reinterpret_cast<J*>(dst + head) + o, blk, cnt);
        }
        count_launch((int)((n + PER - 1) / PER));
        CT_CUDA_TRY(cudaGetLastError());
        return CT_OK;
    }
    std::vector<uint8_t> img(head + n * sizeof(J), 0);
    memcpy(img.data() + head, jobs, n * sizeof(J));
    CT_CUDA_TRY(cudaMemcpyAsync(dst, img.data(), img.size(), cudaMemcpyHostToDevice, stream));
    return CT_OK;
}

// RAII device guard
struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int device) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (prev != device && cudaSetDevice(device) != cudaSuccess) ok = false;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

static inline bool is_float_dt(int dt) { return dt == CT_F32 || dt == CT_F16 || dt == CT_BF16; }
static inline int dt_size(int dt) {
    switch (dt) {
    case CT_F32: case CT_I32: return 4;
    case CT_F16: case CT_BF16: return 2;
    case CT_I8: case CT_U8: case CT_F8E4M3: case CT_E8M0: return 1;
    case CT_I64: return 8;
    default: return 0;
    }
}
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ------------------------------------------------------------------------------------
// unsigned division by a runtime-invariant 32-bit divisor (n < 2^31)
// ------------------------------------------------------------------------------------
struct FastDiv {
    uint32_t d;      // divisor (0xFFFFFFFF: "infinite", quotient always 0)
    uint32_t magic;
    uint32_t shift;
};
static inline FastDiv make_fastdiv(uint64_t d) {
    FastDiv f;
    if (d >= 0x7FFFFFFFull) { f.d = 0xFFFFFFFFu; f.magic = 0; f.shift = 31; return f; }
    f.d = (uint32_t)d;
    uint32_t s = 0;
    while ((1ull << s) < d) ++s;
    f.shift = s;
    f.magic = (uint32_t)(((1ull << 32) * ((1ull << s) - d)) / d + 1);
    return f;
}
__device__ __forceinline__ uint32_t fd_div(uint32_t n, const FastDiv& f) {
    // valid for n < 2^31
    return (__umulhi(n, f.magic) + n) >> f.shift;
}

// ------------------------------------------------------------------------------------
// global memory access: 128-bit streaming loads / stores
// ------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ldg_stream8(const void* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream16(void* p, const uint4& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
// one thread writes 32 contiguous bytes, p 32-byte aligned: two 128-bit stores (the widest global store sm_90 has)
__device__ __forceinline__ void stg_stream32(void* p, const uint32_t (&o)[8]) {
    stg_stream16(p, make_uint4(o[0], o[1], o[2], o[3]));
    stg_stream16(reinterpret_cast<uint8_t*>(p) + 16, make_uint4(o[4], o[5], o[6], o[7]));
}
__device__ __forceinline__ void stg_stream8(void* p, const uint2& v) {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ void stg_stream4(void* p, uint32_t v) {
    asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// ------------------------------------------------------------------------------------
// mbarrier + 1-D bulk async copy (TMA engine, no tensor map) -- sm_90+
// ------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    while (!mbar_try_wait(bar, parity)) {}
}
// global -> shared bulk copy, completion counted in bytes on `bar`; L2 evict-first policy (read-once stream)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
// ---- same primitives on precomputed 32-bit shared addresses (no generic->shared conversion in loops)
__device__ __forceinline__ void mbar_init_a(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_a(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// try_wait with a suspend-time hint: the hardware parks the thread until the phase completes (or
// the hint expires), so a waiting producer lane does not compete for issue slots
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra.uni WAIT_DONE;\n\t"
        "bra.uni WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t}"
        ::"r"(bar), "r"(parity), "r"(0x989680u) : "memory");
}
__device__ __forceinline__ void bulk_g2s_a(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar, uint64_t policy) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
        ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar), "l"(policy) : "memory");
}
// the same copy at the default L2 priority
__device__ __forceinline__ void bulk_g2s_a(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(bar) : "memory");
}
// shared -> global bulk store (bulk async-group completion)
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

}  // namespace ctb

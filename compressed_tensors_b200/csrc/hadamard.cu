// hadamard.cu -- ct_hadamard_transform: y = x · M / sqrt(n) along the last dimension of every row, M one of the structured
// matrices of the `hadamard` / `random-hadamard` transform factories (transform/factory/), block-diagonal (D / n blocks) when the
// row is longer than n, as _multihead_matmul applies it.
//
// Identities (H = Sylvester's matrix of order n, H[i][j] = (-1)^popcount(i & j), symmetric; Q = n signs; perm a permutation):
//   hadamard                    M = H                            M^T = M
//   hadamard, randomize         M = H[perm][:, perm]             M^T = M              (H symmetric)
//   random-hadamard             M = diag(Q) · H                  M^T = H · diag(Q)
//   random-hadamard, randomize  M = (diag(Q) · H)[perm][:, perm]  M^T[i][j] = Q[perm[j]] H[perm[j]][perm[i]]
// so, with z[perm[i]] = x[i] (scatter; z = x without perm) and u = FWHT(z) = z · H:
//   forward   y[j] = u'[perm[j]],                 u' = FWHT(z ∘ Q)     signs before the butterflies
//   inverse   y[j] = Q[perm[j]] · u[perm[j]]      u  = FWHT(z)         signs after (identity for the Hadamard forms without Q)
// then y / sqrt(n) in the compute precision and one conversion to the output dtype.
//
// Butterfly order (the CPU twin in cpu_twin.cu uses the same one, so both give the same bits): stage h = 1, 2, 4, ..., n/2 in turn, each pair
// (a, b) = (z[i], z[i + h]) with (i & h) == 0 becoming (a + b, a - b).  Sign flips are exact.  The division is IEEE, by
// C(sqrt(n)) -- never a multiplication by the reciprocal.  fp64 results reach 16-bit outputs through fp32, as torch's CPU
// conversion does (two roundings).
//
// Layout: a CTA takes a tile of TE = max(n, 4096) elements (TE / n transform rows) of the strided [B, H, S, D] tensor, loads it with
// 16-byte loads into shared memory as C (scattered by perm, signs applied), runs the stages there three at a time in registers
// (radix-8 passes, one barrier each; a pad word every 32 floats / 16 doubles keeps the strided passes off shared bank conflicts),
// and writes the gathered, scaled, converted tile with 16-byte streaming stores.  fp64 at n = 2^15 (256 KB) does not fit in
// shared memory: that case keeps its tile in a stream-ordered global scratch slice per CTA instead (L2-resident, same code).
#include <cmath>
#include <cstring>

#include "engine.h"
#include "hadamard.cuh"

namespace ctb {

constexpr int HAD_THREADS = 256;
constexpr int HAD_MIN_TILE_LOG2 = 12;     // 4096 elements per tile at least
constexpr int HAD_MAX_LOG2 = 15;

template <class C> struct PadShift;
template <> struct PadShift<float> { static constexpr int v = 5; };
template <> struct PadShift<double> { static constexpr int v = 4; };
template <class C>
__host__ __device__ __forceinline__ uint32_t padi(uint32_t i) { return i + (i >> PadShift<C>::v); }
template <class C>
static inline size_t tile_bytes(int tile_log2) { return (size_t)padi<C>(1u << tile_log2) * sizeof(C); }

struct HadJobK {
    const uint8_t* x;
    uint8_t* out;
    int64_t sb, sh, ss;       // byte strides of b, h, s
    FastDiv per_row, S, H;    // transform rows per D-row (D / n), sequence length, heads
    uint32_t rows;            // transform rows in all
    int logn, tile_log2;
    const int8_t* sign;
    const int64_t* perm;
    int inverse;
    int vec;                  // 16-byte loads / stores (aligned, D * es % 16 == 0)
    double scale;             // sqrt(n)
    uint8_t* scratch;         // global tile buffers (fp64 at n = 2^15), else NULL
};

// byte offset of element i of transform row r
__device__ __forceinline__ int64_t had_offset(const HadJobK& J, uint32_t r, uint32_t i, int es) {
    const uint32_t bhs = fd_div(r, J.per_row);
    const uint32_t k = r - bhs * J.per_row.d;
    const uint32_t bh = fd_div(bhs, J.S);
    const uint32_t s = bhs - bh * J.S.d;
    const uint32_t b = fd_div(bh, J.H);
    const uint32_t h = bh - b * J.H.d;
    return (int64_t)b * J.sb + (int64_t)h * J.sh + (int64_t)s * J.ss + (((int64_t)k << J.logn) + i) * es;
}

// R butterfly stages (bits b .. b + R - 1 of the element index) over the whole tile, in registers
template <class C, int R>
__device__ __forceinline__ void had_pass(C* t, int b, uint32_t te) {
    const uint32_t groups = te >> R;
    const uint32_t lowmask = (1u << b) - 1u;
    for (uint32_t g = threadIdx.x; g < groups; g += HAD_THREADS) {
        const uint32_t base = ((g & ~lowmask) << R) | (g & lowmask);
        C v[1 << R];
#pragma unroll
        for (int j = 0; j < (1 << R); ++j) v[j] = t[padi<C>(base + ((uint32_t)j << b))];
#pragma unroll
        for (int s = 0; s < R; ++s)
#pragma unroll
            for (int j = 0; j < (1 << R); ++j)
                if (!(j & (1 << s))) {
                    const C a = v[j], c = v[j | (1 << s)];
                    v[j] = a + c;
                    v[j | (1 << s)] = a - c;
                }
#pragma unroll
        for (int j = 0; j < (1 << R); ++j) t[padi<C>(base + ((uint32_t)j << b))] = v[j];
    }
}

template <class C, int DT, bool GMEM>
__global__ void __launch_bounds__(HAD_THREADS) hadamard_kernel(const __grid_constant__ HadJobK J) {
    using E = Elem<DT>;
    using T = typename E::T;
    constexpr int es = sizeof(T);
    constexpr int V = 16 / es;                    // elements per 16-byte chunk
    extern __shared__ __align__(16) uint8_t had_smem[];
    C* t = GMEM ? reinterpret_cast<C*>(J.scratch) + (size_t)blockIdx.x * padi<C>(1u << J.tile_log2) : reinterpret_cast<C*>(had_smem);
    const uint32_t te = 1u << J.tile_log2;
    const uint32_t n = 1u << J.logn;
    const uint32_t rows_per_tile = te >> J.logn;
    const uint32_t n_tiles = (J.rows + rows_per_tile - 1) / rows_per_tile;
    const C scale = (C)J.scale;

    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint32_t row0 = tile * rows_per_tile;
        const uint32_t tile_rows = min(rows_per_tile, J.rows - row0);
        const uint32_t valid = tile_rows << J.logn;
        // load: scatter by perm, signs before the butterflies (forward)
        auto put = [&](uint32_t e, T raw) {
            const uint32_t i = e & (n - 1);
            const uint32_t k = J.perm ? (uint32_t)J.perm[i] : i;
            C v = E::template load<C>(raw);
            if (J.sign && !J.inverse && J.sign[k] < 0) v = -v;
            t[padi<C>((e & ~(n - 1)) | k)] = v;
        };
        if (J.vec) {
            for (uint32_t e = threadIdx.x * V; e < valid; e += HAD_THREADS * V) {
                const uint4 w = ldg_stream16(J.x + had_offset(J, row0 + (e >> J.logn), e & (n - 1), es));
                const T* p = reinterpret_cast<const T*>(&w);
#pragma unroll
                for (int j = 0; j < V; ++j) put(e + j, p[j]);
            }
        } else {
            for (uint32_t e = threadIdx.x; e < valid; e += HAD_THREADS)
                put(e, *reinterpret_cast<const T*>(J.x + had_offset(J, row0 + (e >> J.logn), e & (n - 1), es)));
        }
        __syncthreads();
        for (int b = 0; b < J.logn; b += 3) {
            const int r = J.logn - b;
            if (r >= 3) had_pass<C, 3>(t, b, te);
            else if (r == 2) had_pass<C, 2>(t, b, te);
            else had_pass<C, 1>(t, b, te);
            __syncthreads();
        }
        // store: signs after (inverse), gather by perm, divide, convert
        auto get = [&](uint32_t e) -> T {
            const uint32_t i = e & (n - 1);
            const uint32_t k = J.perm ? (uint32_t)J.perm[i] : i;
            C v = t[padi<C>((e & ~(n - 1)) | k)];
            if (J.sign && J.inverse && J.sign[k] < 0) v = -v;
            return E::store(v / scale);
        };
        if (J.vec) {
            for (uint32_t e = threadIdx.x * V; e < valid; e += HAD_THREADS * V) {
                uint4 w;
                T* p = reinterpret_cast<T*>(&w);
#pragma unroll
                for (int j = 0; j < V; ++j) p[j] = get(e + j);
                stg_stream16(J.out + had_offset(J, row0 + (e >> J.logn), e & (n - 1), es), w);
            }
        } else {
            for (uint32_t e = threadIdx.x; e < valid; e += HAD_THREADS)
                *reinterpret_cast<T*>(J.out + had_offset(J, row0 + (e >> J.logn), e & (n - 1), es)) = get(e);
        }
        __syncthreads();   // the tile buffer is reused by the next tile
    }
}

template <class C, int DT, bool GMEM>
static int launch_had(const HadJobK& J, unsigned grid, cudaStream_t st) {
    const size_t smem = GMEM ? 0 : tile_bytes<C>(J.tile_log2);
    if (smem > 48 * 1024)
        CT_CUDA_TRY(cudaFuncSetAttribute(hadamard_kernel<C, DT, GMEM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    hadamard_kernel<C, DT, GMEM><<<grid, HAD_THREADS, smem, st>>>(J);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

template <class C>
static int launch_had_dt(int dt, bool gmem, const HadJobK& J, unsigned grid, cudaStream_t st) {
    switch (dt) {
    case CT_BF16: return gmem ? launch_had<C, CT_BF16, true>(J, grid, st) : launch_had<C, CT_BF16, false>(J, grid, st);
    case CT_F16: return gmem ? launch_had<C, CT_F16, true>(J, grid, st) : launch_had<C, CT_F16, false>(J, grid, st);
    default: return gmem ? launch_had<C, CT_F32, true>(J, grid, st) : launch_had<C, CT_F32, false>(J, grid, st);
    }
}

static int had_unsupported(const char* why) {
    set_error("hadamard_transform: %s", why);
    return CT_E_UNSUPPORTED;
}

}  // namespace ctb

using namespace ctb;

extern "C" int ct_hadamard_transform(const ct_hadamard_job* job, int device, void* stream) {
    if (!job) { set_error("null job"); return CT_E_ARG; }
    const ct_hadamard_job& j = *job;
    if (j.log2_n < 1 || j.log2_n > HAD_MAX_LOG2) { set_error("transform order 2^%d outside 2^1 .. 2^15", j.log2_n); return CT_E_SHAPE; }
    if (!is_float_dt(j.dtype)) { set_error("dtype %d: bf16 / fp16 / fp32 only", j.dtype); return CT_E_DTYPE; }
    if (j.precision != CT_F32 && j.precision != CT_F64) { set_error("precision must be fp32 or fp64"); return CT_E_DTYPE; }
    for (int k = 0; k < 4; ++k)
        if (j.shape[k] < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    const int64_t n = (int64_t)1 << j.log2_n;
    if (j.shape[3] % n != 0) { set_error("the order %lld does not divide the last dimension %lld", (long long)n, (long long)j.shape[3]); return CT_E_SHAPE; }
    const int64_t numel = j.shape[0] * j.shape[1] * j.shape[2] * j.shape[3];
    if (numel == 0) return CT_OK;
    if (!j.x || !j.out) { set_error("null tensor pointer"); return CT_E_ARG; }
    if (j.stride[3] != 1) return had_unsupported("needs a contiguous last dimension");
    if (device == CT_DEVICE_CPU) {
        cpu_hadamard(j);
        return CT_OK;
    }
    const int64_t rows = numel >> j.log2_n;
    if (rows >= 0x7fffffffLL || j.shape[1] >= 0x7fffffffLL || j.shape[2] >= 0x7fffffffLL) return had_unsupported("tensor too large");
    int rc = check_device(device);
    if (rc) return rc;

    const int es = dt_size(j.dtype);
    HadJobK K;
    memset(&K, 0, sizeof(K));
    K.x = reinterpret_cast<const uint8_t*>(j.x);
    K.out = reinterpret_cast<uint8_t*>(j.out);
    K.sb = j.stride[0] * es;
    K.sh = j.stride[1] * es;
    K.ss = j.stride[2] * es;
    K.per_row = make_fastdiv((uint64_t)(j.shape[3] >> j.log2_n));
    K.S = make_fastdiv((uint64_t)(j.shape[2] > 0 ? j.shape[2] : 1));
    K.H = make_fastdiv((uint64_t)(j.shape[1] > 0 ? j.shape[1] : 1));
    K.rows = (uint32_t)rows;
    K.logn = j.log2_n;
    K.tile_log2 = j.log2_n > HAD_MIN_TILE_LOG2 ? j.log2_n : HAD_MIN_TILE_LOG2;
    K.sign = j.sign;
    K.perm = j.perm;
    K.inverse = j.inverse ? 1 : 0;
    bool vec = aligned16(j.x) && aligned16(j.out) && (j.shape[3] * es) % 16 == 0;
    for (int k = 0; k < 3; ++k)
        if ((j.stride[k] * es) % 16 != 0 && j.shape[k] > 1) vec = false;
    K.vec = vec ? 1 : 0;
    K.scale = std::sqrt((double)n);

    const bool f64 = j.precision == CT_F64;
    const size_t tb = f64 ? tile_bytes<double>(K.tile_log2) : tile_bytes<float>(K.tile_log2);
    const bool gmem = tb > 200 * 1024;
    const uint32_t rows_per_tile = 1u << (K.tile_log2 - K.logn);
    const uint64_t tiles = (rows + rows_per_tile - 1) / rows_per_tile;
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    unsigned grid = (unsigned)(tiles < 0x7fffffffull ? tiles : 0x7fffffffull);
    if (gmem) {
        grid = (unsigned)(tiles < (uint64_t)(2 * sm_count(device)) ? tiles : (uint64_t)(2 * sm_count(device)));
        void* scratch = nullptr;
        rc = scratch_alloc(&scratch, (size_t)grid * tb, device, st);
        if (rc) return rc;
        K.scratch = reinterpret_cast<uint8_t*>(scratch);
        rc = launch_had_dt<double>(j.dtype, true, K, grid, st);
        cudaFreeAsync(scratch, st);
        return rc;
    }
    return f64 ? launch_had_dt<double>(j.dtype, false, K, grid, st) : launch_had_dt<float>(j.dtype, false, K, grid, st);
}

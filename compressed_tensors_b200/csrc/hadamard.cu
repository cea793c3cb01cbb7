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
// With a K x K +-1 core C (core_order = K, n = K · 2^m), H above is replaced by G = (C ⊗ H_{2^m})^T = C^T ⊗ H_{2^m}, the matrix the
// reference's random_hadamard_matrix builds from its table of known Hadamard matrices (diag(Q) · G).  Viewing an n-block as
// Z[K][2^m] (index a · 2^m + b):
//   z · G       = Y,  Y[c][:] = sum_a C[c][a] · FWHT(Z[a][:])      (forward: signs before, as above)
//   z · G^T     = Y,  Y[c][:] = sum_a C[a][c] · FWHT(Z[a][:])      (inverse: C^T, signs after)
// so the four forms keep their scatter / sign / gather steps, the butterflies run on each of the K rows of 2^m, and a core stage
// mixes the K rows.  Its sums run sequentially, a = 0, 1, ..., K - 1, starting from the a = 0 term; a term with C = -1 is subtracted
// (exact sign flip, no multiplication).  The CPU twin uses the same order.
//
// Butterfly order (the CPU twin in cpu_twin.cu uses the same one, so both give the same bits): stage h = 1, 2, 4, ..., n/2 in turn, each pair
// (a, b) = (z[i], z[i + h]) with (i & h) == 0 becoming (a + b, a - b).  Sign flips are exact.  The division is IEEE, by
// C(sqrt(n)) -- never a multiplication by the reciprocal.  fp64 results reach 16-bit outputs through fp32, as torch's CPU
// conversion does (two roundings).
//
// Layout: a CTA takes a tile of whole n-blocks, TE = max(n, 4096) elements for a power of two (TE / n transform rows) and a multiple of
// 8 rows of about 4096 elements with a core, of the strided [B, H, S, D] tensor, loads it with 16-byte loads into shared memory
// (scattered by perm, signs applied), runs the stages there three at a time in registers (radix-8 passes, one barrier each; a pad
// word every 32 floats / 16 doubles keeps the strided passes off shared bank conflicts), mixes the rows with the core (below), and
// writes the gathered, scaled, converted tile with 16-byte streaming stores.  fp64 tiles above 200 KB (2^15, or K · 2^m > 24094)
// do not fit in shared memory: that case keeps its tile in a stream-ordered global scratch slice per CTA instead (L2-resident,
// same code).
// Core stage: the signs of C (C^T under inverse) sit in shared memory as a bitmask, 32 bytes per a (bit c of row a set when the
// coefficient of row a in output c is -1).  A thread owns CORE_G consecutive outputs c of one column (block, b): it reads the column's
// K values once and keeps CORE_G sums in registers; the columns of a chunk are read before any is written back (two barriers).
#include <cmath>
#include <cstring>

#include "engine.h"
#include "hadamard.cuh"

namespace ctb {

constexpr int HAD_THREADS = 256;
constexpr int HAD_MIN_TILE_LOG2 = 12;     // 4096 elements per tile at least
constexpr int HAD_MAX_LOG2 = 15;
constexpr int HAD_MAX_CORE = 256;
constexpr int CORE_G = 8;                 // outputs c per thread in the core stage (one mask byte)
constexpr int CORE_MASK_BYTES = HAD_MAX_CORE * HAD_MAX_CORE / 8;

template <class C> struct PadShift;
template <> struct PadShift<float> { static constexpr int v = 5; };
template <> struct PadShift<double> { static constexpr int v = 4; };
template <class C>
__host__ __device__ __forceinline__ uint32_t padi(uint32_t i) { return i + (i >> PadShift<C>::v); }
template <class C>
static inline size_t tile_bytes(uint32_t te) { return (size_t)padi<C>(te) * sizeof(C); }

struct HadJobK {
    const uint8_t* x;
    uint8_t* out;
    int64_t sb, sh, ss;       // byte strides of b, h, s
    FastDiv per_row, S, H;    // transform rows per D-row (D / n), sequence length, heads
    FastDiv nd;               // n (with a core)
    uint32_t rows;            // transform rows in all
    uint32_t n, te;           // order, elements per tile (a whole number of n-blocks)
    int logn;                 // log2 of the butterfly length: n without a core, 2^m with one
    int K;                    // core order, 0 without a core
    const int8_t* core;       // K x K, row-major
    const int8_t* sign;
    const int64_t* perm;
    int inverse;
    int vec;                  // 16-byte loads / stores (aligned, D * es % 16 == 0, tiles start on 16 bytes)
    double scale;             // sqrt(n)
    uint8_t* scratch;         // global tile buffers (fp64 tiles above 200 KB), else NULL
};

// n-block of element e of a tile, and e's index in it
template <bool CORE>
__device__ __forceinline__ uint32_t had_block(const HadJobK& J, uint32_t e) { return CORE ? fd_div(e, J.nd) : e >> J.logn; }
template <bool CORE>
__device__ __forceinline__ uint32_t had_index(const HadJobK& J, uint32_t e, uint32_t blk) { return CORE ? e - blk * J.n : e & (J.n - 1); }

// byte offset of element i of transform row r
template <bool CORE>
__device__ __forceinline__ int64_t had_offset(const HadJobK& J, uint32_t r, uint32_t i, int es) {
    const uint32_t bhs = fd_div(r, J.per_row);
    const uint32_t k = r - bhs * J.per_row.d;
    const uint32_t bh = fd_div(bhs, J.S);
    const uint32_t s = bhs - bh * J.S.d;
    const uint32_t b = fd_div(bh, J.H);
    const uint32_t h = bh - b * J.H.d;
    return (int64_t)b * J.sb + (int64_t)h * J.sh + (int64_t)s * J.ss + ((int64_t)k * J.n + i) * es;
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

// the sign bitmask of the core stage: byte g of row a holds, in bit i, whether output c = CORE_G * g + i takes row a negated
// (C[c][a] < 0 forward, C[a][c] < 0 under inverse)
__device__ __forceinline__ void core_mask(const HadJobK& J, uint32_t* mask) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int words = (J.K + 31) >> 5;
    for (int w = warp; w < J.K * words; w += HAD_THREADS / 32) {
        const int a = w / words, c = ((w - a * words) << 5) + lane;
        const bool neg = c < J.K && (J.inverse ? J.core[a * J.K + c] : J.core[c * J.K + a]) < 0;
        const uint32_t bits = __ballot_sync(0xffffffffu, neg);
        if (lane == 0) mask[a * (HAD_MAX_CORE / 32) + (w - a * words)] = bits;
    }
}

// Y[c][b] = sum_a (+-) X[a][b] for every column (block, b) of the tile, sequentially over a
template <class C>
__device__ __forceinline__ void core_stage(const HadJobK& J, C* t, const uint8_t* mask, uint32_t tile_blocks) {
    const uint32_t m = 1u << J.logn;
    const uint32_t cg = (J.K + CORE_G - 1) / CORE_G;             // output groups per column
    const uint32_t cols_per_chunk = HAD_THREADS / cg;
    const uint32_t g = threadIdx.x / cols_per_chunk, col_in = threadIdx.x - g * cols_per_chunk;
    const uint32_t cols = tile_blocks << J.logn;
    const int c0 = (int)g * CORE_G;
    for (uint32_t col0 = 0; col0 < cols; col0 += cols_per_chunk) {
        const uint32_t col = col0 + col_in;
        const bool active = g < cg && col < cols;
        C acc[CORE_G];
        uint32_t base = 0;
        if (active) {
            base = (col >> J.logn) * J.n + (col & (m - 1));
            {
                const C v = t[padi<C>(base)];
                const uint32_t bits = mask[g];
#pragma unroll
                for (int i = 0; i < CORE_G; ++i) acc[i] = ((bits >> i) & 1u) ? -v : v;
            }
            for (int a = 1; a < J.K; ++a) {
                const C v = t[padi<C>(base + ((uint32_t)a << J.logn))];
                const uint32_t bits = mask[a * (HAD_MAX_CORE / 8) + g];
#pragma unroll
                for (int i = 0; i < CORE_G; ++i) acc[i] = ((bits >> i) & 1u) ? acc[i] - v : acc[i] + v;
            }
        }
        __syncthreads();
        if (active) {
#pragma unroll
            for (int i = 0; i < CORE_G; ++i)
                if (c0 + i < J.K) t[padi<C>(base + ((uint32_t)(c0 + i) << J.logn))] = acc[i];
        }
        __syncthreads();
    }
}

template <class C, int DT, bool GMEM, bool CORE>
__global__ void __launch_bounds__(HAD_THREADS, CORE ? 2 : 0) hadamard_kernel(const __grid_constant__ HadJobK J) {
    using E = Elem<DT>;
    using T = typename E::T;
    constexpr int es = sizeof(T);
    constexpr int V = 16 / es;                    // elements per 16-byte chunk
    extern __shared__ __align__(16) uint8_t had_smem[];
    uint32_t* mask = reinterpret_cast<uint32_t*>(had_smem);
    const size_t mask_bytes = CORE ? CORE_MASK_BYTES : 0;
    const uint32_t te = J.te;
    C* t = GMEM ? reinterpret_cast<C*>(J.scratch) + (size_t)blockIdx.x * padi<C>(te) : reinterpret_cast<C*>(had_smem + mask_bytes);
    const uint32_t n = J.n;
    const uint32_t rows_per_tile = CORE ? te / n : te >> J.logn;
    const uint32_t n_tiles = (J.rows + rows_per_tile - 1) / rows_per_tile;
    const C scale = (C)J.scale;
    const bool mix = CORE && J.core != nullptr;
    if (mix) core_mask(J, mask);                  // read before the first barrier below

    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint32_t row0 = tile * rows_per_tile;
        const uint32_t tile_rows = min(rows_per_tile, J.rows - row0);
        const uint32_t valid = tile_rows * n;
        // load: scatter by perm, signs before the butterflies (forward)
        auto put = [&](uint32_t e, T raw) {
            const uint32_t blk = had_block<CORE>(J, e);
            const uint32_t i = had_index<CORE>(J, e, blk);
            const uint32_t k = J.perm ? (uint32_t)J.perm[i] : i;
            C v = E::template load<C>(raw);
            if (J.sign && !J.inverse && J.sign[k] < 0) v = -v;
            t[padi<C>(blk * n + k)] = v;
        };
        if (J.vec) {
            for (uint32_t e = threadIdx.x * V; e < valid; e += HAD_THREADS * V) {
                const uint32_t blk = had_block<CORE>(J, e);
                const uint4 w = ldg_stream16(J.x + had_offset<CORE>(J, row0 + blk, had_index<CORE>(J, e, blk), es));
                const T* p = reinterpret_cast<const T*>(&w);
#pragma unroll
                for (int j = 0; j < V; ++j) put(e + j, p[j]);
            }
        } else {
            for (uint32_t e = threadIdx.x; e < valid; e += HAD_THREADS) {
                const uint32_t blk = had_block<CORE>(J, e);
                put(e, *reinterpret_cast<const T*>(J.x + had_offset<CORE>(J, row0 + blk, had_index<CORE>(J, e, blk), es)));
            }
        }
        __syncthreads();
        for (int b = 0; b < J.logn; b += 3) {
            const int r = J.logn - b;
            if (r >= 3) had_pass<C, 3>(t, b, te);
            else if (r == 2) had_pass<C, 2>(t, b, te);
            else had_pass<C, 1>(t, b, te);
            __syncthreads();
        }
        if (mix) core_stage<C>(J, t, reinterpret_cast<const uint8_t*>(mask), tile_rows);
        // store: signs after (inverse), gather by perm, divide, convert
        auto get = [&](uint32_t e) -> T {
            const uint32_t blk = had_block<CORE>(J, e);
            const uint32_t i = had_index<CORE>(J, e, blk);
            const uint32_t k = J.perm ? (uint32_t)J.perm[i] : i;
            C v = t[padi<C>(blk * n + k)];
            if (J.sign && J.inverse && J.sign[k] < 0) v = -v;
            return E::store(v / scale);
        };
        if (J.vec) {
            for (uint32_t e = threadIdx.x * V; e < valid; e += HAD_THREADS * V) {
                uint4 w;
                T* p = reinterpret_cast<T*>(&w);
#pragma unroll
                for (int j = 0; j < V; ++j) p[j] = get(e + j);
                const uint32_t blk = had_block<CORE>(J, e);
                stg_stream16(J.out + had_offset<CORE>(J, row0 + blk, had_index<CORE>(J, e, blk), es), w);
            }
        } else {
            for (uint32_t e = threadIdx.x; e < valid; e += HAD_THREADS) {
                const uint32_t blk = had_block<CORE>(J, e);
                *reinterpret_cast<T*>(J.out + had_offset<CORE>(J, row0 + blk, had_index<CORE>(J, e, blk), es)) = get(e);
            }
        }
        __syncthreads();   // the tile buffer is reused by the next tile
    }
}

template <class C, int DT, bool GMEM, bool CORE>
static int launch_had(const HadJobK& J, unsigned grid, cudaStream_t st) {
    const size_t smem = (CORE ? CORE_MASK_BYTES : 0) + (GMEM ? 0 : tile_bytes<C>(J.te));
    if (smem > 48 * 1024)
        CT_CUDA_TRY(cudaFuncSetAttribute(hadamard_kernel<C, DT, GMEM, CORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    hadamard_kernel<C, DT, GMEM, CORE><<<grid, HAD_THREADS, smem, st>>>(J);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

template <class C, bool GMEM, bool CORE>
static int launch_had_dt(int dt, const HadJobK& J, unsigned grid, cudaStream_t st) {
    switch (dt) {
    case CT_BF16: return launch_had<C, CT_BF16, GMEM, CORE>(J, grid, st);
    case CT_F16: return launch_had<C, CT_F16, GMEM, CORE>(J, grid, st);
    default: return launch_had<C, CT_F32, GMEM, CORE>(J, grid, st);
    }
}

template <class C, bool GMEM>
static int launch_had_core(bool core, int dt, const HadJobK& J, unsigned grid, cudaStream_t st) {
    return core ? launch_had_dt<C, GMEM, true>(dt, J, grid, st) : launch_had_dt<C, GMEM, false>(dt, J, grid, st);
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
    const bool has_core = j.core_order != 0;
    if (has_core) {
        if (j.core_order < 1 || j.core_order > HAD_MAX_CORE) { set_error("core order %d outside 1 .. %d", j.core_order, HAD_MAX_CORE); return CT_E_SHAPE; }
        if (j.log2_n < 0 || j.log2_n > HAD_MAX_LOG2 || ((int64_t)j.core_order << j.log2_n) > ((int64_t)1 << HAD_MAX_LOG2)) {
            set_error("transform order %d * 2^%d outside 1 .. 2^15", j.core_order, j.log2_n);
            return CT_E_SHAPE;
        }
        if (!j.core && j.core_order > 1) { set_error("null core of order %d", j.core_order); return CT_E_ARG; }
    } else if (j.log2_n < 1 || j.log2_n > HAD_MAX_LOG2) { set_error("transform order 2^%d outside 2^1 .. 2^15", j.log2_n); return CT_E_SHAPE; }
    if (!is_float_dt(j.dtype)) { set_error("dtype %d: bf16 / fp16 / fp32 only", j.dtype); return CT_E_DTYPE; }
    if (j.precision != CT_F32 && j.precision != CT_F64) { set_error("precision must be fp32 or fp64"); return CT_E_DTYPE; }
    for (int k = 0; k < 4; ++k)
        if (j.shape[k] < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    const int64_t n = (int64_t)(has_core ? j.core_order : 1) << j.log2_n;
    if (j.shape[3] % n != 0) { set_error("the order %lld does not divide the last dimension %lld", (long long)n, (long long)j.shape[3]); return CT_E_SHAPE; }
    const int64_t numel = j.shape[0] * j.shape[1] * j.shape[2] * j.shape[3];
    if (numel == 0) return CT_OK;
    if (!j.x || !j.out) { set_error("null tensor pointer"); return CT_E_ARG; }
    if (j.stride[3] != 1) return had_unsupported("needs a contiguous last dimension");
    if (device == CT_DEVICE_CPU) {
        cpu_hadamard(j);
        return CT_OK;
    }
    const int64_t rows = numel / n;
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
    K.per_row = make_fastdiv((uint64_t)(j.shape[3] / n));
    K.S = make_fastdiv((uint64_t)(j.shape[2] > 0 ? j.shape[2] : 1));
    K.H = make_fastdiv((uint64_t)(j.shape[1] > 0 ? j.shape[1] : 1));
    K.nd = make_fastdiv((uint64_t)n);
    K.rows = (uint32_t)rows;
    K.n = (uint32_t)n;
    K.logn = j.log2_n;
    K.K = has_core ? j.core_order : 0;
    K.core = has_core ? j.core : nullptr;
    if (has_core) {
        uint32_t rpt = (uint32_t)((1 << HAD_MIN_TILE_LOG2) / n);
        rpt = rpt >= 8 ? rpt & ~7u : (rpt ? rpt : 1);
        K.te = rpt * (uint32_t)n;
    } else {
        K.te = 1u << (j.log2_n > HAD_MIN_TILE_LOG2 ? j.log2_n : HAD_MIN_TILE_LOG2);
    }
    K.sign = j.sign;
    K.perm = j.perm;
    K.inverse = j.inverse ? 1 : 0;
    bool vec = aligned16(j.x) && aligned16(j.out) && (j.shape[3] * es) % 16 == 0 && ((int64_t)K.te * es) % 16 == 0;
    for (int k = 0; k < 3; ++k)
        if ((j.stride[k] * es) % 16 != 0 && j.shape[k] > 1) vec = false;
    K.vec = vec ? 1 : 0;
    K.scale = std::sqrt((double)n);

    const bool f64 = j.precision == CT_F64;
    const size_t tb = f64 ? tile_bytes<double>(K.te) : tile_bytes<float>(K.te);
    const bool gmem = tb > 200 * 1024;
    const uint32_t rows_per_tile = K.te / (uint32_t)n;
    const uint64_t tiles = (rows + rows_per_tile - 1) / rows_per_tile;
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // with a core every CTA first reads the K x K core into its mask: persistent CTAs (a few per SM) read it once each
    const uint64_t cap = gmem ? (uint64_t)(2 * sm_count(device)) : has_core ? (uint64_t)(8 * sm_count(device)) : 0x7fffffffull;
    unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
    if (gmem) {
        void* scratch = nullptr;
        rc = scratch_alloc(&scratch, (size_t)grid * tb, device, st);
        if (rc) return rc;
        K.scratch = reinterpret_cast<uint8_t*>(scratch);
        rc = launch_had_core<double, true>(has_core, j.dtype, K, grid, st);
        cudaFreeAsync(scratch, st);
        return rc;
    }
    return f64 ? launch_had_core<double, false>(has_core, j.dtype, K, grid, st) : launch_had_core<float, false>(has_core, j.dtype, K, grid, st);
}

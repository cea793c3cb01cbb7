// fake_heads.cu -- ct_fake_quantize_heads: fake quantization of attention K / V / Q in their strided [B, H, S, D] layout.
//
// transformers passes key / value / query states to the attention hooks as transposed views of [B, S, H, D] projections, so a
// row (b, h, s) of D elements is contiguous but rows are not.  A plain vectorised grid covers every chunk of 8 elements of up to
// two tensors in one launch: no contiguous copy in, none out.  The arithmetic is FakeQuantOp::apply (ops.cuh), the function the
// streaming fake_quantize kernel runs, so both paths give the same bits.  Tensors here run from one decode token to a few tens of
// MB at prefill: each thread keeps HEADS_UNROLL chunks in flight, which is what the 16-byte loads need to cover DRAM latency.
#include <cstring>

#include "engine.h"
#include "ops.cuh"

namespace ctb {

constexpr int HEADS_THREADS = 256;
constexpr int HEADS_UNROLL = 4;
constexpr int HEADS_CHUNKS_PER_BLOCK = HEADS_THREADS * HEADS_UNROLL;

struct HeadJobK {
    const uint8_t* x;
    uint8_t* out;
    const void* scale;
    const void* zp;
    int64_t sb, sh, ss;      // byte strides of b, h, s
    FastDiv cpr, S, H;       // chunks per row (D / 8), sequence length, heads
    uint32_t n_chunks;
    uint32_t per_head;
};
struct HeadLaunch {
    HeadJobK j[2];
    uint32_t blocks0;        // blocks of job 0; the rest of the grid covers job 1
    Common cm;
};

template <class P, int KIND, int ZP>
__global__ void __launch_bounds__(HEADS_THREADS) fake_heads_kernel(const __grid_constant__ HeadLaunch L) {
    using Op = FakeQuantOp<P, KIND, ZP>;
    constexpr int W = Op::IN_BYTES / 4;
    const int ji = blockIdx.x >= L.blocks0 ? 1 : 0;
    const HeadJobK& J = L.j[ji];
    const uint32_t first = (blockIdx.x - (ji ? L.blocks0 : 0u)) * HEADS_CHUNKS_PER_BLOCK + threadIdx.x;
    uint32_t w[HEADS_UNROLL][W];
    RawQP r[HEADS_UNROLL];
    int64_t off[HEADS_UNROLL];
#pragma unroll
    for (int k = 0; k < HEADS_UNROLL; ++k) {
        const uint32_t gc = first + k * HEADS_THREADS;
        if (gc >= J.n_chunks) break;
        const uint32_t row = fd_div(gc, J.cpr);
        const uint32_t c = gc - row * J.cpr.d;
        const uint32_t bh = fd_div(row, J.S);
        const uint32_t s = row - bh * J.S.d;
        const uint32_t b = fd_div(bh, J.H);
        const uint32_t h = bh - b * J.H.d;
        off[k] = (int64_t)b * J.sb + (int64_t)h * J.sh + (int64_t)s * J.ss + (int64_t)c * Op::IN_BYTES;
#pragma unroll
        for (int q = 0; q < W; q += 4) {
            const uint4 v = ldg_stream16(J.x + off[k] + 4 * q);
            w[k][q] = v.x; w[k][q + 1] = v.y; w[k][q + 2] = v.z; w[k][q + 3] = v.w;
        }
        r[k] = load_qp<P, ZP>(J.scale, J.zp, J.per_head ? h : 0u);
    }
#pragma unroll
    for (int k = 0; k < HEADS_UNROLL; ++k) {
        const uint32_t gc = first + k * HEADS_THREADS;
        if (gc >= J.n_chunks) break;
        uint32_t o[W];
        Op::apply(L.cm, r[k], w[k], o);
        store_words<W>(J.out + off[k], o);
    }
}

template <class P>
static int launch_heads(int kind, int zpk, const HeadLaunch& L, unsigned blocks, cudaStream_t st) {
#define CT_HEADS_LAUNCH(K, Z)                                                                \
    if (kind == K && zpk == Z) {                                                             \
        fake_heads_kernel<P, K, Z><<<blocks, HEADS_THREADS, 0, st>>>(L);                     \
        count_launch();                                                                      \
        CT_CUDA_TRY(cudaGetLastError());                                                     \
        return CT_OK;                                                                        \
    }
    CT_HEADS_LAUNCH(QF8, 0)
    CT_HEADS_LAUNCH(QF8, 1)
    CT_HEADS_LAUNCH(QF8, 2)
    CT_HEADS_LAUNCH(QI_WIDE, 0)
    CT_HEADS_LAUNCH(QI_WIDE, 1)
    if constexpr (P::DT != CT_F32) {   // fp32 has no packed-magic rounding: NARROW and WIDE coincide (fast_fake.cu)
        CT_HEADS_LAUNCH(QI_NARROW, 0)
        CT_HEADS_LAUNCH(QI_NARROW, 1)
    }
#undef CT_HEADS_LAUNCH
    set_error("no fake_quantize_heads kernel for kind=%d zp=%d", kind, zpk);
    return CT_E_UNSUPPORTED;
}

static int unsupported(const char* why) {
    set_error("fake_quantize_heads: %s", why);
    return CT_E_UNSUPPORTED;
}

// zero-point kind of a job (0 none, 1 int8, 2 float8_e4m3fn), -1 when unsupported
static int zp_kind(const ct_head_job& j) {
    if (!j.zp) return 0;
    if (j.zp_dtype == CT_I8) return 1;
    if (j.zp_dtype == CT_F8E4M3 && j.qtype == CT_Q_FLOAT) return 2;
    return -1;
}

}  // namespace ctb

using namespace ctb;

extern "C" int ct_fake_quantize_heads(int n, const ct_head_job* jobs, int device, void* stream) {
    if (n < 1 || n > 2 || !jobs) { set_error("fake_quantize_heads takes 1 or 2 jobs"); return CT_E_ARG; }
    const ct_head_job& j0 = jobs[0];
    for (int i = 0; i < n; ++i) {
        const ct_head_job& j = jobs[i];
        if (j.qtype == CT_Q_INT && (j.num_bits < 1 || j.num_bits > 8)) { set_error("num_bits %d outside [1, 8]", j.num_bits); return CT_E_BITS; }
        if (j.qtype == CT_Q_FLOAT && j.num_bits != 8) { set_error("fp8 quantization needs num_bits == 8"); return CT_E_BITS; }
        for (int k = 0; k < 4; ++k)
            if (j.shape[k] < 0) { set_error("negative shape"); return CT_E_SHAPE; }
        if (j.qtype != CT_Q_INT && j.qtype != CT_Q_FLOAT) return unsupported("only integer and fp8 quantization");
        if (!is_float_dt(j.x_dtype) || j.scale_dtype != j.x_dtype) return unsupported("x and scale must share a float dtype");
        if (j.x_dtype != j0.x_dtype || j.qtype != j0.qtype || j.num_bits != j0.num_bits || zp_kind(j) != zp_kind(j0))
            return unsupported("the jobs of one call must share dtypes, quantization type and zero-point kind");
        if (zp_kind(j) < 0) return unsupported("zero point must be int8 (or float8_e4m3fn for fp8)");
        const int64_t es = dt_size(j.x_dtype);
        if (j.stride[3] != 1 || j.shape[3] % 8 != 0) return unsupported("needs a contiguous last dimension with D % 8 == 0");
        if (!aligned16(j.x) || !aligned16(j.out)) return unsupported("x and out must be 16-byte aligned");
        for (int k = 0; k < 3; ++k)
            if ((j.stride[k] * es) % 16 != 0 && j.shape[k] > 1) return unsupported("row strides must be multiples of 16 bytes");
        const int64_t numel = j.shape[0] * j.shape[1] * j.shape[2] * j.shape[3];
        if (numel / 8 >= 0x7fffffffLL || j.shape[1] >= 0x7fffffffLL || j.shape[2] >= 0x7fffffffLL) return unsupported("tensor too large");
        if (numel > 0 && (!j.x || !j.out || !j.scale)) { set_error("null tensor pointer"); return CT_E_ARG; }
    }
    int rc = check_device(device);
    if (rc) return rc;

    HeadLaunch L;
    memset(&L, 0, sizeof(L));
    unsigned blocks[2] = {0, 0};
    for (int i = 0; i < n; ++i) {
        const ct_head_job& j = jobs[i];
        const int64_t es = dt_size(j.x_dtype);
        HeadJobK& k = L.j[i];
        k.x = reinterpret_cast<const uint8_t*>(j.x);
        k.out = reinterpret_cast<uint8_t*>(j.out);
        k.scale = j.scale;
        k.zp = j.zp;
        k.sb = j.stride[0] * es;
        k.sh = j.stride[1] * es;
        k.ss = j.stride[2] * es;
        k.cpr = make_fastdiv((uint64_t)(j.shape[3] / 8 > 0 ? j.shape[3] / 8 : 1));
        k.S = make_fastdiv((uint64_t)(j.shape[2] > 0 ? j.shape[2] : 1));
        k.H = make_fastdiv((uint64_t)(j.shape[1] > 0 ? j.shape[1] : 1));
        k.n_chunks = (uint32_t)(j.shape[0] * j.shape[1] * j.shape[2] * j.shape[3] / 8);
        k.per_head = j.per_head ? 1u : 0u;
        blocks[i] = (k.n_chunks + HEADS_CHUNKS_PER_BLOCK - 1) / HEADS_CHUNKS_PER_BLOCK;
    }
    L.blocks0 = blocks[0];
    const unsigned total = blocks[0] + blocks[1];
    if (total == 0) return CT_OK;
    const int p_dt = j0.x_dtype;
    L.cm = make_common(p_dt, j0.qtype, j0.num_bits);
    const int kind = fake_kind(p_dt, j0.qtype, j0.num_bits);
    const int zpk = zp_kind(j0);
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    switch (p_dt) {
    case CT_BF16: return launch_heads<BF16>(kind, zpk, L, total, st);
    case CT_F16: return launch_heads<F16>(kind, zpk, L, total, st);
    default: return launch_heads<F32>(kind, zpk, L, total, st);
    }
}

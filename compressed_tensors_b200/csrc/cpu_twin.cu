// cpu_twin.cu -- the `device = -1` twins of the per-tensor ABI (SURVEY.md 8(b): "each with a _cpu twin (device = -1)").
//
// HOST code inside libct_b200.so, selected EXPLICITLY by passing device = CT_DEVICE_CPU (-1) together with host pointers: the body the
// reference calls "eager" (utils/impl_backend.py:98-123), what a GPU-less host (HF loading a checkpoint on CPU; BASELINE config 1,
// "int4 round-trip, CPU only") and CT_ENFORCE_EAGER=1 get.  It is never a fallback: device >= 0 without a usable H100 still fails
// with CT_E_NODEV, and nothing here is reachable from a CUDA tensor unless the caller asks for it.
//
// The arithmetic is the SAME SOURCE as the generic CUDA kernels: quant_at / dequant_at / pack_group / unpack_group of generic.cuh and
// quant_core.cuh are __host__ __device__, so the per-op rounding, the clamp-before-round order, the wrapping-sum bit packing and the
// scale addressing cannot drift between the two.  OpenMP over rows.  Nothing under oracle/ is linked or included.
#include <cmath>
#include <cstring>

#include "generic.cuh"
#include "hadamard.cuh"

namespace ctb {

static int cpu_check(const ct_quant_desc& d) {
    if (d.rows < 0 || d.cols < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    if (d.rdiv <= 0 || d.cdiv <= 0) { set_error("rdiv/cdiv must be positive"); return CT_E_SHAPE; }
    if (d.qtype == CT_Q_INT && (d.num_bits < 1 || d.num_bits > 8)) { set_error("num_bits %d outside [1, 8]", d.num_bits); return CT_E_BITS; }
    if (d.qtype == CT_Q_FLOAT && d.num_bits != 8) { set_error("fp8 quantization needs num_bits == 8"); return CT_E_BITS; }
    if (d.qtype != CT_Q_INT && d.qtype != CT_Q_FLOAT) { set_error("the CPU twins cover integer and fp8 quantization (qtype %d)", d.qtype); return CT_E_UNSUPPORTED; }
    if (d.global_scale) { set_error("the CPU twins do not take a global scale"); return CT_E_UNSUPPORTED; }
    return CT_OK;
}

template <int BITS>
static void cpu_pack(const int8_t* in, int32_t* out, int64_t rows, int64_t cols, int packed_dim) {
    if (packed_dim == 1) {
        const int64_t nw = (cols * BITS + 31) / 32, groups = (cols + 31) / 32;
#pragma omp parallel for schedule(static)
        for (int64_t r = 0; r < rows; ++r)
            for (int64_t g = 0; g < groups; ++g) {
                const int64_t c0 = g * 32;
                const int nvalid = (int)(cols - c0 < 32 ? cols - c0 : 32);
                const int8_t* src = in + r * cols + c0;
                uint32_t words[BITS];
                pack_group<BITS>(words, nvalid, [&](int j) { return (int32_t)src[j]; });
                for (int k = 0; k < BITS; ++k)
                    if (g * BITS + k < nw) out[r * nw + g * BITS + k] = (int32_t)words[k];
            }
    } else {
        const int64_t nw = (rows * BITS + 31) / 32, groups = (rows + 31) / 32;
#pragma omp parallel for schedule(static)
        for (int64_t g = 0; g < groups; ++g)
            for (int64_t c = 0; c < cols; ++c) {
                const int64_t r0 = g * 32;
                const int nvalid = (int)(rows - r0 < 32 ? rows - r0 : 32);
                uint32_t words[BITS];
                pack_group<BITS>(words, nvalid, [&](int j) { return (int32_t)in[(r0 + j) * cols + c]; });
                for (int k = 0; k < BITS; ++k)
                    if (g * BITS + k < nw) out[(g * BITS + k) * cols + c] = (int32_t)words[k];
            }
    }
}

template <int BITS>
static void cpu_unpack(const int32_t* in, int8_t* out, int64_t rows, int64_t cols, int packed_dim) {
    if (packed_dim == 1) {
        const int64_t nw = (cols * BITS + 31) / 32, groups = (cols + 31) / 32;
#pragma omp parallel for schedule(static)
        for (int64_t r = 0; r < rows; ++r)
            for (int64_t g = 0; g < groups; ++g) {
                const int64_t c0 = g * 32;
                const int nvalid = (int)(cols - c0 < 32 ? cols - c0 : 32);
                uint32_t words[BITS];
                for (int k = 0; k < BITS; ++k) words[k] = (g * BITS + k < nw) ? (uint32_t)in[r * nw + g * BITS + k] : 0u;
                int8_t* dst = out + r * cols + c0;
                unpack_group<BITS>(words, nvalid, [&](int j, int v) { dst[j] = (int8_t)v; });
            }
    } else {
        const int64_t nw = (rows * BITS + 31) / 32, groups = (rows + 31) / 32;
#pragma omp parallel for schedule(static)
        for (int64_t g = 0; g < groups; ++g)
            for (int64_t c = 0; c < cols; ++c) {
                const int64_t r0 = g * 32;
                const int nvalid = (int)(rows - r0 < 32 ? rows - r0 : 32);
                uint32_t words[BITS];
                for (int k = 0; k < BITS; ++k) words[k] = (g * BITS + k < nw) ? (uint32_t)in[(g * BITS + k) * cols + c] : 0u;
                unpack_group<BITS>(words, nvalid, [&](int j, int v) { out[(r0 + j) * cols + c] = (int8_t)v; });
            }
    }
}

template <int BITS>
static void cpu_quantpack(const GParams& p) {
    const int64_t nw = (p.cols * BITS + 31) / 32, groups = (p.cols + 31) / 32;
    int32_t* out = reinterpret_cast<int32_t*>(p.out);
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < p.rows; ++r)
        for (int64_t g = 0; g < groups; ++g) {
            const int64_t c0 = g * 32;
            const int nvalid = (int)(p.cols - c0 < 32 ? p.cols - c0 : 32);
            uint32_t words[BITS];
            pack_group<BITS>(words, nvalid, [&](int j) {
                const float q = quant_at(p, r, c0 + j);
                return (q != q) ? 0 : (int32_t)q;   // .to(int8)
            });
            for (int k = 0; k < BITS; ++k)
                if (g * BITS + k < nw) out[r * nw + g * BITS + k] = (int32_t)words[k];
        }
}

template <int BITS>
static void cpu_unpackdeq(const GParams& p) {
    const int64_t nw = (p.cols * BITS + 31) / 32, groups = (p.cols + 31) / 32;
    const int32_t* in = reinterpret_cast<const int32_t*>(p.in);
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < p.rows; ++r)
        for (int64_t g = 0; g < groups; ++g) {
            const int64_t c0 = g * 32;
            const int nvalid = (int)(p.cols - c0 < 32 ? p.cols - c0 : 32);
            uint32_t words[BITS];
            for (int k = 0; k < BITS; ++k) words[k] = (g * BITS + k < nw) ? (uint32_t)in[r * nw + g * BITS + k] : 0u;
            unpack_group<BITS>(words, nvalid, [&](int j, int v) {
                store_from_f32(p.out, r * p.cols + c0 + j, p.out_dt, dequant_at(p, (float)v, r, c0 + j));
            });
        }
}

#define CPU_BITS_SWITCH(bits, EXPR)               \
    switch (bits) {                               \
    case 1: { constexpr int B = 1; EXPR; } break; \
    case 2: { constexpr int B = 2; EXPR; } break; \
    case 3: { constexpr int B = 3; EXPR; } break; \
    case 4: { constexpr int B = 4; EXPR; } break; \
    case 5: { constexpr int B = 5; EXPR; } break; \
    case 6: { constexpr int B = 6; EXPR; } break; \
    case 7: { constexpr int B = 7; EXPR; } break; \
    case 8: { constexpr int B = 8; EXPR; } break; \
    default: set_error("num_bits %d outside [1, 8]", bits); return CT_E_BITS; \
    }

int cpu_run_bits(bool pack, const void* in, void* out, int64_t rows, int64_t cols, int bits, int packed_dim) {
    if (bits < 1 || bits > 8) { set_error("num_bits %d outside [1, 8]", bits); return CT_E_BITS; }
    if (packed_dim != 0 && packed_dim != 1) { set_error("packed_dim must be 0 or 1"); return CT_E_ARG; }
    if (rows < 0 || cols < 0) { set_error("negative shape"); return CT_E_SHAPE; }
    if (rows * cols == 0) return CT_OK;
    if (!in || !out) { set_error("null tensor pointer"); return CT_E_ARG; }
    if (pack) { CPU_BITS_SWITCH(bits, (cpu_pack<B>(reinterpret_cast<const int8_t*>(in), reinterpret_cast<int32_t*>(out), rows, cols, packed_dim))); }
    else { CPU_BITS_SWITCH(bits, (cpu_unpack<B>(reinterpret_cast<const int32_t*>(in), reinterpret_cast<int8_t*>(out), rows, cols, packed_dim))); }
    return CT_OK;
}

// one tensor of a quantization op on the host; same dtype checks as the device path (dispatch.cu) has done before this is called
int cpu_run_one(int op, const ct_quant_desc& d, const void* in, const void* scale, const void* zp, const int32_t* g_idx, void* out) {
    int rc = cpu_check(d);
    if (rc) return rc;
    const int64_t n = d.rows * d.cols;
    if (n == 0) return CT_OK;
    if (!in || !scale || !out) { set_error("null tensor pointer"); return CT_E_ARG; }
    const GParams p = make_params(d, in, scale, zp, g_idx, out);
    switch (op) {
    case CT_OP_QUANTIZE:
    case CT_OP_DEQUANTIZE:
    case CT_OP_FAKE_QUANTIZE: {
#pragma omp parallel for schedule(static)
        for (int64_t r = 0; r < p.rows; ++r)
            for (int64_t c = 0; c < p.cols; ++c) {
                const int64_t i = r * p.cols + c;
                if (op == CT_OP_QUANTIZE) store_from_f32(p.out, i, p.q_dt, quant_at(p, r, c));
                else if (op == CT_OP_DEQUANTIZE) store_from_f32(p.out, i, p.out_dt, dequant_at(p, load_as_f32(p.in, i, p.q_dt), r, c));
                else store_from_f32(p.out, i, p.out_dt, dequant_at(p, quant_at(p, r, c), r, c));
            }
        return CT_OK;
    }
    case CT_OP_QUANTIZE_PACK:
        if (d.qtype != CT_Q_INT) { set_error("quantize_pack needs integer quantization"); return CT_E_DTYPE; }
        CPU_BITS_SWITCH(d.num_bits, (cpu_quantpack<B>(p)));
        return CT_OK;
    case CT_OP_UNPACK_DEQUANTIZE:
        CPU_BITS_SWITCH(d.num_bits, (cpu_unpackdeq<B>(p)));
        return CT_OK;
    }
    set_error("op %d has no CPU twin (device = -1 covers pack / unpack, quantize / dequantize / fake_quantize and the two fused compressor bodies)", op);
    return CT_E_UNSUPPORTED;
}

// ct_hadamard_transform on the host: the butterfly order of hadamard.cu (stage h = 1, 2, ..., 2^log2_n / 2), the core stage's sequential
// sums over a = 0 .. K - 1, the same conversions (hadamard.cuh)
template <class C, int DT>
static void cpu_hadamard_rows(const ct_hadamard_job& j) {
    using E = Elem<DT>;
    using T = typename E::T;
    const int64_t m = (int64_t)1 << j.log2_n;
    const int64_t K = j.core_order > 0 ? j.core_order : 1;
    const int64_t n = K * m;
    const bool mix = j.core_order > 0 && j.core != nullptr;
    const int64_t per_row = j.shape[3] / n;
    const int64_t rows = j.shape[0] * j.shape[1] * j.shape[2] * per_row;
    const C scale = (C)std::sqrt((double)n);
    const T* x = reinterpret_cast<const T*>(j.x);
    T* out = reinterpret_cast<T*>(j.out);
#pragma omp parallel
    {
        C* z = new C[n];
        C* y = new C[n];
#pragma omp for schedule(static)
        for (int64_t r = 0; r < rows; ++r) {
            const int64_t bhs = r / per_row, k = r % per_row;
            const int64_t s = bhs % j.shape[2], bh = bhs / j.shape[2];
            const int64_t h = bh % j.shape[1], b = bh / j.shape[1];
            const int64_t off = b * j.stride[0] + h * j.stride[1] + s * j.stride[2] + k * n;
            for (int64_t i = 0; i < n; ++i) {
                const int64_t q = j.perm ? j.perm[i] : i;
                C v = E::template load<C>(x[off + i]);
                if (j.sign && !j.inverse && j.sign[q] < 0) v = -v;
                z[q] = v;
            }
            for (int64_t hh = 1; hh < m; hh <<= 1)
                for (int64_t i = 0; i < n; ++i)
                    if (!(i & hh)) {
                        const C a = z[i], c = z[i + hh];
                        z[i] = a + c;
                        z[i + hh] = a - c;
                    }
            if (mix) {
                for (int64_t c = 0; c < K; ++c)
                    for (int64_t d = 0; d < m; ++d) {
                        C acc = 0;
                        for (int64_t a = 0; a < K; ++a) {
                            const bool neg = (j.inverse ? j.core[a * K + c] : j.core[c * K + a]) < 0;
                            const C v = z[a * m + d];
                            acc = a == 0 ? (neg ? -v : v) : (neg ? acc - v : acc + v);
                        }
                        y[c * m + d] = acc;
                    }
                std::memcpy(z, y, sizeof(C) * n);
            }
            for (int64_t i = 0; i < n; ++i) {
                const int64_t q = j.perm ? j.perm[i] : i;
                C v = z[q];
                if (j.sign && j.inverse && j.sign[q] < 0) v = -v;
                out[off + i] = E::store(v / scale);
            }
        }
        delete[] z;
        delete[] y;
    }
}

template <class C>
static void cpu_hadamard_dt(const ct_hadamard_job& j) {
    switch (j.dtype) {
    case CT_BF16: cpu_hadamard_rows<C, CT_BF16>(j); break;
    case CT_F16: cpu_hadamard_rows<C, CT_F16>(j); break;
    default: cpu_hadamard_rows<C, CT_F32>(j); break;
    }
}

void cpu_hadamard(const ct_hadamard_job& j) {
    if (j.precision == CT_F64) cpu_hadamard_dt<double>(j);
    else cpu_hadamard_dt<float>(j);
}

}  // namespace ctb

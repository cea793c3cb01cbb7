// convert.cu -- checkpoint-format conversions (SURVEY 8(f) rank 3): AutoAWQ GEMM int4 -> compressed-tensors pack-quantized.
//
// Reference: entrypoints/convert/converters/autoawq.py:179-262 (unpack_awq -> reverse_awq_order -> & 15 -> - 8 -> .T ->
// pack_to_int32).  AutoAWQ stores qweight as int32 [K, N/8]: word (k, w) holds the eight 4-bit codes of output channels
// 8w .. 8w+7 of input channel k, channel 8w + c in nibble REV[c], REV = [0, 4, 1, 5, 2, 6, 3, 7].  compressed-tensors wants
// weight_packed int32 [N, K/8] with nibble i of word (n, kw) = code(k = 8 kw + i, n) (the signed value - 8 is re-offset by + 8
// when packing, so the nibble itself never changes).  The whole chain is therefore an 8x8 nibble transpose per (8 k, 1 word)
// block with a fixed column permutation -- one pass, 0.5 B/elem in, 0.5 B/elem out, instead of the reference's six full-size
// int8 / int32 temporaries.
#include "engine.h"

namespace ctb {

// nibble j of w
__device__ __forceinline__ uint32_t nib(uint32_t w, int j) { return (w >> (4 * j)) & 0xfu; }

constexpr int AWQ_TK = 64;    // k rows per tile  (8 output words per row of the tile)
constexpr int AWQ_TW = 32;    // input words per tile row (256 output channels)

// grid: (ceil(N/8 / 32), ceil(K / 64)); block: 256 = 32 (word in tile) x 8 (k-octet in tile)
__global__ void __launch_bounds__(256) awq_repack_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                         int64_t K, int64_t NW /* N/8 */, int64_t KW /* ceil(K/8) */) {
    __shared__ uint32_t tile[8][AWQ_TW * 8 + 8];   // [k-octet][output channel in tile]
    const int wl = threadIdx.x & 31, kl = threadIdx.x >> 5;
    const int64_t w = (int64_t)blockIdx.x * AWQ_TW + wl;
    const int64_t k0 = (int64_t)blockIdx.y * AWQ_TK + kl * 8;
    uint32_t v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = (w < NW && k0 + i < K) ? __ldg(in + (k0 + i) * NW + w) : 0u;   // rows past K pack as raw 0 (helpers.py:62-70)
    // O_c nibble i = v[i] nibble REV[c]
    constexpr int REV[8] = {0, 4, 1, 5, 2, 6, 3, 7};
    uint32_t o[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        uint32_t acc = 0;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc |= nib(v[i], REV[c]) << (4 * i);
        o[c] = acc;
    }
    // two 16-byte shared stores per thread, linear in wl
    uint4* dst = reinterpret_cast<uint4*>(&tile[kl][wl * 8]);
    dst[0] = make_uint4(o[0], o[1], o[2], o[3]);
    dst[1] = make_uint4(o[4], o[5], o[6], o[7]);
    __syncthreads();
    // thread t owns output channel t of the tile: 8 consecutive words (one 32-byte sector) of its row
    const int nl = threadIdx.x;
    const int64_t n = (int64_t)blockIdx.x * AWQ_TW * 8 + nl;
    const int64_t kw0 = (int64_t)blockIdx.y * (AWQ_TK / 8);
    if (n < NW * 8) {
        uint32_t r[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = tile[j][nl];
        uint32_t* dst_row = out + n * KW + kw0;
        // uint4 stores need a 16-byte aligned row: KW % 4 == 0 aligns every row to the base, which must be aligned itself
        if (kw0 + 8 <= KW && (KW % 4) == 0 && (reinterpret_cast<uintptr_t>(out) & 15u) == 0) {
            reinterpret_cast<uint4*>(dst_row)[0] = make_uint4(r[0], r[1], r[2], r[3]);
            reinterpret_cast<uint4*>(dst_row)[1] = make_uint4(r[4], r[5], r[6], r[7]);
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                if (kw0 + j < KW) dst_row[j] = r[j];
        }
    }
}

// qzeros int32 [G, N/8] -> weight_zero_point int32 [N/8, G] (pack_to_int32(zp.T, packed_dim=0).contiguous(), autoawq.py:124-128):
// a word transpose with the nibble permutation applied inside each word.  Qparam-sized; one thread per output word.
__global__ void __launch_bounds__(256) awq_repack_zeros_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int64_t G, int64_t NW) {
    constexpr int REV[8] = {0, 4, 1, 5, 2, 6, 3, 7};
    const int64_t total = G * NW;
    for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t nw = t / G, g = t - nw * G;
        const uint32_t v = __ldg(in + g * NW + nw);
        uint32_t acc = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc |= nib(v, REV[j]) << (4 * j);
        out[t] = acc;
    }
}

}  // namespace ctb

using namespace ctb;

extern "C" {

int ct_awq_repack_int4(const int32_t* qweight, int32_t* weight_packed, int64_t K, int64_t N, int device, void* stream) {
    if (K < 0 || N < 0 || N % 8 != 0) { set_error("AutoAWQ qweight needs out_features %% 8 == 0"); return CT_E_SHAPE; }
    int rc = check_device(device);
    if (rc) return rc;
    if (K * N == 0) return CT_OK;
    if (!qweight || !weight_packed) { set_error("null tensor pointer"); return CT_E_ARG; }
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    const int64_t NW = N / 8, KW = (K + 7) / 8;
    const dim3 grid((unsigned)((NW + AWQ_TW - 1) / AWQ_TW), (unsigned)((K + AWQ_TK - 1) / AWQ_TK));
    if (grid.y > 65535u) { set_error("in_features too large for one launch"); return CT_E_SHAPE; }
    awq_repack_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const uint32_t*>(qweight),
                                                                                 reinterpret_cast<uint32_t*>(weight_packed), K, NW, KW);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

int ct_awq_repack_zeros_int4(const int32_t* qzeros, int32_t* zero_point_packed, int64_t G, int64_t N, int device, void* stream) {
    if (G < 0 || N < 0 || N % 8 != 0) { set_error("AutoAWQ qzeros needs out_features %% 8 == 0"); return CT_E_SHAPE; }
    int rc = check_device(device);
    if (rc) return rc;
    if (G * N == 0) return CT_OK;
    if (!qzeros || !zero_point_packed) { set_error("null tensor pointer"); return CT_E_ARG; }
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");
    const int64_t total = G * (N / 8);
    int64_t blocks = (total + 255) / 256;
    if (blocks > GRID_SMS * 32) blocks = GRID_SMS * 32;
    awq_repack_zeros_kernel<<<(unsigned)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const uint32_t*>(qzeros), reinterpret_cast<uint32_t*>(zero_point_packed), G, N / 8);
    count_launch();
    CT_CUDA_TRY(cudaGetLastError());
    return CT_OK;
}

}  // extern "C"

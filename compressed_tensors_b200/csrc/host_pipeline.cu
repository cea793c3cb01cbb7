// host_pipeline.cu -- ct_host_run_many: one op over host-resident tensors (one large CPU tensor, or a CPU-resident model),
// pipelined ACROSS tensors.  All row chunks of all tensors form one queue that is fed through NSLOT staging slots (own stream
// each: H2D chunk -> kernel -> D2H chunk), so that the upload of one chunk, the kernel of the one before and the download of the
// one before that overlap on the two copy engines and the SMs, and the H2D copy engine never drains between tensors.  Every
// tensor's scales / zero points are uploaded once into a per-call aux area and published to the other slots with an event.
// Device scratch is cached per device (grow-only) and serialised by a mutex.  Blocking: once anything is queued, the call returns
// only after every slot stream has drained, on error too, so no copy from or into the caller's buffers outlives the call.
//
// Test hook: CT_B200_HOST_CHUNK_MB (default 32) sets the streamed input per chunk; at 1 MiB small tensors span many chunks.
#include <cstdlib>
#include <mutex>
#include <vector>

#include "engine.h"

namespace ctb {

constexpr int NSLOT = 4;
static size_t host_chunk() { const char* v = getenv("CT_B200_HOST_CHUNK_MB"); int n = v ? atoi(v) : 32; return (size_t)(n < 1 ? 1 : (n > 512 ? 512 : n)) << 20; }

struct Scratch {
    std::mutex mu;
    void* in[NSLOT] = {};
    void* out[NSLOT] = {};
    size_t in_cap = 0, out_cap = 0;
    void* aux = nullptr;
    size_t aux_cap = 0;
    cudaStream_t st[NSLOT] = {};
    bool init = false;
};
static Scratch g_scratch[16];

// k buffers of at least `bytes` each; a failed allocation leaves cap = 0 (and no freed pointer behind), so the next call retries
static int grow(void** buf, int k, size_t& cap, size_t bytes) {
    if (bytes <= cap) return CT_OK;
    cap = 0;
    for (int i = 0; i < k; ++i) { if (buf[i]) cudaFree(buf[i]); buf[i] = nullptr; }
    for (int i = 0; i < k; ++i) CT_CUDA_TRY(cudaMalloc(&buf[i], bytes));
    cap = bytes;
    return CT_OK;
}

static size_t up256(size_t v) { return (v + 255) / 256 * 256; }

static int row_bytes(int op, const ct_quant_desc& d, size_t& in_row, size_t& out_row) {
    const int64_t nw = (d.cols * d.num_bits + 31) / 32;
    switch (op) {
    case CT_OP_QUANTIZE_PACK: in_row = (size_t)d.cols * dt_size(d.x_dtype); out_row = (size_t)nw * 4; break;
    case CT_OP_UNPACK_DEQUANTIZE: in_row = (size_t)nw * 4; out_row = (size_t)d.cols * dt_size(d.out_dtype); break;
    case CT_OP_QUANTIZE: in_row = (size_t)d.cols * dt_size(d.x_dtype); out_row = (size_t)d.cols * dt_size(d.q_dtype); break;
    case CT_OP_DEQUANTIZE: in_row = (size_t)d.cols * dt_size(d.q_dtype); out_row = (size_t)d.cols * dt_size(d.out_dtype); break;
    case CT_OP_FAKE_QUANTIZE: in_row = (size_t)d.cols * dt_size(d.x_dtype); out_row = (size_t)d.cols * dt_size(d.out_dtype); break;
    case CT_OP_QUANTIZE_PACK_FP4: in_row = (size_t)d.cols * dt_size(d.x_dtype); out_row = (size_t)d.cols / 2; break;
    case CT_OP_UNPACK_DEQUANTIZE_FP4: in_row = (size_t)d.cols / 2; out_row = (size_t)d.cols * dt_size(d.out_dtype); break;
    default: set_error("unknown op %d", op); return CT_E_ARG;
    }
    if (in_row == 0 || out_row == 0) { set_error("bad dtype in descriptor"); return CT_E_DTYPE; }
    return CT_OK;
}

static int64_t scale_count(const ct_quant_desc& d) {
    const bool row_scaled = (d.rdiv != CT_DIV_INF);
    const int64_t row_blocks = row_scaled ? (d.rows + d.rdiv - 1) / d.rdiv : 1;
    const int64_t per_row = (d.cdiv == CT_DIV_INF) ? 1 : (d.cols + d.cdiv - 1) / d.cdiv;
    return (row_scaled && d.s_row_stride > 0) ? row_blocks * d.s_row_stride : per_row;
}

}  // namespace ctb

extern "C" int ct_host_run_many(int op, int n, const ct_quant_desc* descs, const void* const* in, const void* const* scale,
                                const void* const* zp, void* const* out, int device) {
    using namespace ctb;
    if (n < 0 || (n > 0 && (!descs || !in || !scale || !out))) { set_error("null table"); return CT_E_ARG; }
    int rc = check_device(device);
    if (rc) return rc;
    if (device >= 16) { set_error("device index too large"); return CT_E_ARG; }
    if (n == 0) return CT_OK;
    DeviceGuard guard(device);
    if (!guard.ok) return cuda_fail(cudaGetLastError(), "cudaSetDevice");

    const size_t CHUNK = host_chunk();   // bytes of streamed input per chunk
    struct T { size_t in_row, out_row, s_off, z_off, s_bytes, z_bytes, g_off; int64_t rpc; };   // g_off: the tensor's global scale (HOST pointer in
                                                                                                // the descriptor of this entry point), uploaded to aux
    std::vector<T> ts((size_t)n);
    size_t aux_total = 0, max_in = 0, max_out = 0;
    for (int i = 0; i < n; ++i) {
        const ct_quant_desc& d = descs[i];
        T& t = ts[i];
        if (d.rows * d.cols == 0) { t = T{}; continue; }
        if (!in[i] || !scale[i] || !out[i]) { set_error("null tensor pointer (tensor %d)", i); return CT_E_ARG; }
        rc = row_bytes(op, d, t.in_row, t.out_row);
        if (rc) return rc;
        const int64_t ns = scale_count(d);
        t.s_bytes = (size_t)ns * dt_size(d.scale_dtype);
        t.z_bytes = (zp && zp[i]) ? (size_t)ns * dt_size(d.zp_dtype) : 0;
        t.s_off = aux_total; aux_total += up256(t.s_bytes);
        t.z_off = aux_total; aux_total += up256(t.z_bytes);
        t.g_off = aux_total; aux_total += d.global_scale ? 256 : 0;
        int64_t rpc = (int64_t)(CHUNK / t.in_row);
        if (rpc < 1) rpc = 1;
        if (d.rdiv != CT_DIV_INF && d.rdiv > 1) rpc = (rpc + d.rdiv - 1) / d.rdiv * d.rdiv;
        if (rpc > d.rows) rpc = d.rows;
        t.rpc = rpc;
        if ((size_t)rpc * t.in_row > max_in) max_in = (size_t)rpc * t.in_row;
        if ((size_t)rpc * t.out_row > max_out) max_out = (size_t)rpc * t.out_row;
    }

    Scratch& S = g_scratch[device];
    std::lock_guard<std::mutex> lk(S.mu);
    if (!S.init) {
        for (int i = 0; i < NSLOT; ++i) CT_CUDA_TRY(cudaStreamCreateWithFlags(&S.st[i], cudaStreamNonBlocking));
        S.init = true;
    }
    rc = grow(S.in, NSLOT, S.in_cap, max_in);
    if (!rc) rc = grow(S.out, NSLOT, S.out_cap, max_out);
    if (!rc) rc = grow(&S.aux, 1, S.aux_cap, aux_total);
    if (rc) return rc;
    uint8_t* aux = reinterpret_cast<uint8_t*>(S.aux);

    std::vector<cudaEvent_t> evs;
    auto enqueue = [&]() -> int {
        int slot = 0;
        for (int i = 0; i < n; ++i) {
            const ct_quant_desc& d = descs[i];
            const T& t = ts[i];
            if (d.rows * d.cols == 0) continue;
            // qparams of this tensor: uploaded on the slot of its first chunk, published to the others
            cudaStream_t s0 = S.st[slot];
            CT_CUDA_TRY(cudaMemcpyAsync(aux + t.s_off, scale[i], t.s_bytes, cudaMemcpyHostToDevice, s0));
            if (t.z_bytes) CT_CUDA_TRY(cudaMemcpyAsync(aux + t.z_off, zp[i], t.z_bytes, cudaMemcpyHostToDevice, s0));
            if (d.global_scale) CT_CUDA_TRY(cudaMemcpyAsync(aux + t.g_off, d.global_scale, sizeof(float), cudaMemcpyHostToDevice, s0));
            cudaEvent_t ev;
            CT_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            evs.push_back(ev);
            CT_CUDA_TRY(cudaEventRecord(ev, s0));
            const bool row_scaled = (d.rdiv != CT_DIV_INF);
            bool first = true;
            for (int64_t r0 = 0; r0 < d.rows; r0 += t.rpc, slot = (slot + 1) % NSLOT) {
                const int64_t nr = (d.rows - r0 < t.rpc) ? d.rows - r0 : t.rpc;
                cudaStream_t st = S.st[slot];
                if (!first) CT_CUDA_TRY(cudaStreamWaitEvent(st, ev, 0));
                first = false;
                CT_CUDA_TRY(cudaMemcpyAsync(S.in[slot], reinterpret_cast<const uint8_t*>(in[i]) + (size_t)r0 * t.in_row, (size_t)nr * t.in_row, cudaMemcpyHostToDevice, st));
                ct_quant_desc sub = d;
                sub.rows = nr;
                if (d.global_scale) sub.global_scale = aux + t.g_off;
                const int64_t sblock = row_scaled ? (r0 / d.rdiv) * d.s_row_stride : 0;
                const void* sc = aux + t.s_off + (size_t)sblock * dt_size(d.scale_dtype);
                const void* zz = t.z_bytes ? aux + t.z_off + (size_t)sblock * dt_size(d.zp_dtype) : nullptr;
                const void* ins[1] = {S.in[slot]};
                const void* scs[1] = {sc};
                const void* zps[1] = {zz};
                void* outs[1] = {S.out[slot]};
                const int r = run_batched(op, 1, &sub, ins, scs, zps, nullptr, outs, device, st);
                if (r) return r;
                CT_CUDA_TRY(cudaMemcpyAsync(reinterpret_cast<uint8_t*>(out[i]) + (size_t)r0 * t.out_row, S.out[slot], (size_t)nr * t.out_row, cudaMemcpyDeviceToHost, st));
            }
        }
        return CT_OK;
    };
    rc = enqueue();
    // the one exit once anything is queued: drain every slot (the first error is the one reported), then release the events
    for (int i = 0; i < NSLOT; ++i) {
        const cudaError_t e = cudaStreamSynchronize(S.st[i]);
        if (e != cudaSuccess && !rc) rc = cuda_fail(e, "cudaStreamSynchronize");
    }
    for (auto e : evs) cudaEventDestroy(e);
    return rc;
}

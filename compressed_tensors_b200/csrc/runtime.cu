// runtime.cu -- error strings, device checks, launch counter.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <mutex>

#include "engine.h"

namespace ctb {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
const char* last_error() { return g_err; }

int cuda_fail(cudaError_t e, const char* what) {
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    return CT_E_CUDA;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int64_t launch_count() { return g_launches.load(std::memory_order_relaxed); }

// ---- devices --------------------------------------------------------------------------------
static std::mutex g_dev_mu;
static int g_sms[64];
static int g_l2[64];
static int g_cc[64];
static bool g_dev_init[64];

static int dev_info(int device) {
    if (device < 0 || device >= 64) return -1;
    std::lock_guard<std::mutex> lk(g_dev_mu);
    if (!g_dev_init[device]) {
        int n = 0;
        if (cudaGetDeviceCount(&n) != cudaSuccess || device >= n) { cudaGetLastError(); return -1; }
        int sms = 0, major = 0, minor = 0;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device);
        cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device);
        g_sms[device] = sms;
        cudaDeviceGetAttribute(&g_l2[device], cudaDevAttrL2CacheSize, device);
        g_cc[device] = major * 10 + minor;
        g_dev_init[device] = true;
    }
    return 0;
}
int sm_count(int device) { return dev_info(device) == 0 ? g_sms[device] : GRID_SMS; }
int64_t l2_bytes(int device) { return dev_info(device) == 0 ? g_l2[device] : 0; }

// ---- launch scratch ---------------------------------------------------------------------------
// Job tables and tile counters come from a library-owned stream-ordered pool per device whose release
// threshold is "never": the default pool hands its memory back at every synchronisation, which made the
// first launch after a sync pay for a fresh physical allocation.
static cudaMemPool_t g_pool[64];
static bool g_pool_init[64];

int scratch_alloc(void** p, size_t bytes, int device, cudaStream_t stream) {
    if (device < 0 || device >= 64) { set_error("bad device %d", device); return CT_E_ARG; }
    cudaMemPool_t pool;
    {
        std::lock_guard<std::mutex> lk(g_dev_mu);
        if (!g_pool_init[device]) {
            cudaMemPoolProps props = {};
            props.allocType = cudaMemAllocationTypePinned;
            props.handleTypes = cudaMemHandleTypeNone;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = device;
            CT_CUDA_TRY(cudaMemPoolCreate(&g_pool[device], &props));
            uint64_t keep = ~0ull;
            CT_CUDA_TRY(cudaMemPoolSetAttribute(g_pool[device], cudaMemPoolAttrReleaseThreshold, &keep));
            g_pool_init[device] = true;
        }
        pool = g_pool[device];
    }
    CT_CUDA_TRY(cudaMallocFromPoolAsync(p, bytes, pool, stream));
    return CT_OK;
}

int check_device(int device) {
    if (dev_info(device) != 0) {
        set_error("no usable CUDA device %d: libct_b200 has no CPU path", device);
        return CT_E_NODEV;
    }
    if (g_cc[device] != 90) {
        set_error("device %d is sm_%d; libct_b200 is built for sm_90a (H100) only", device, g_cc[device]);
        return CT_E_NODEV;
    }
    return CT_OK;
}

}  // namespace ctb

// ---- C ABI: library / device -----------------------------------------------------------------
extern "C" {
const char* ct_version(void) { return "ct_b200 0.1.0 (sm_90a)"; }
const char* ct_last_error(void) { return ctb::last_error(); }
int ct_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
int ct_device_ok(int device) { return ctb::check_device(device) == CT_OK ? 1 : 0; }
int64_t ct_launch_count(void) { return ctb::launch_count(); }
}

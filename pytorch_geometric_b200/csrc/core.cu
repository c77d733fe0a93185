// core.cu -- version, error string, device info.
#include <cstdarg>
#include <cstring>

#include "common.cuh"

namespace b200mp {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace b200mp

extern "C" const char* b200mp_version(void) { return B200MP_VERSION; }
extern "C" const char* b200mp_last_error(void) { return b200mp::g_err; }

extern "C" int b200mp_device_info(int* sm_count, int* cc_major, int* cc_minor, int64_t* l2_bytes) {
    int dev = 0;
    B200MP_CUDA(cudaGetDevice(&dev));
    int v = 0;
    if (sm_count) {
        B200MP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
        *sm_count = v;
    }
    if (cc_major) {
        B200MP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev));
        *cc_major = v;
    }
    if (cc_minor) {
        B200MP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev));
        *cc_minor = v;
    }
    if (l2_bytes) {
        B200MP_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, dev));
        *l2_bytes = v;
    }
    return B200MP_OK;
}

// ---------------------------------------------------------------- runtime options
namespace b200mp {
static int g_spmm_impl = 0;
int get_option_spmm_impl() { return g_spmm_impl; }
static int g_spmm_tune = 0;
int get_option_spmm_tune() { return g_spmm_tune; }
static int g_attn_staged = 2;   // cp.async-staged attention sweeps (csrc/attention.cu): 2 = with one-warp CTAs, 1 = 4-warp CTAs, 0 = register-staged loop
int get_option_attn_staged() { return g_attn_staged; }
static int g_multi_tune = 6;    // multi_aggr.cu: 6 = one-warp CTAs for the row sweeps (default), 5 = the 128-thread form, kept for A/B
int get_option_multi_tune() { return g_multi_tune; }

// Work counters of the persistent kernels: a small device-resident pool, one slot per launch in
// round-robin order, zeroed on the launching stream right before the kernel (so concurrent
// launches on different streams never share a slot unless > kSlots launches are in flight).
constexpr int kSlots = 1024;
constexpr int kMaxDev = 16;
static unsigned long long* g_pool[kMaxDev] = {nullptr};
static unsigned int g_next = 0;
unsigned long long* tma_counter_slot(cudaStream_t stream) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDev) {
        set_error("tma_counter_slot: bad device");
        return nullptr;
    }
    if (!g_pool[dev]) {
        if (cudaMalloc(&g_pool[dev], sizeof(unsigned long long) * kSlots) != cudaSuccess) {
            set_error("tma_counter_slot: cudaMalloc failed");
            return nullptr;
        }
    }
    unsigned long long* slot = g_pool[dev] + (__atomic_fetch_add(&g_next, 1u, __ATOMIC_RELAXED) % kSlots);
    if (cudaMemsetAsync(slot, 0, sizeof(unsigned long long), stream) != cudaSuccess) {
        set_error("tma_counter_slot: memset failed");
        return nullptr;
    }
    return slot;
}
}  // namespace b200mp

extern "C" int b200mp_set_option(const char* name, int value) {
    if (!name) return B200MP_ERR_INVALID_ARG;
    if (strcmp(name, "spmm_impl") == 0) {
        if (value < 0 || value > 2) return B200MP_ERR_INVALID_ARG;
        b200mp::g_spmm_impl = value;
        return B200MP_OK;
    }
    if (strcmp(name, "spmm_tune") == 0) {
        b200mp::g_spmm_tune = value;
        return B200MP_OK;
    }
    if (strcmp(name, "multi_tune") == 0) {
        if (value != 5 && value != 6) return B200MP_ERR_INVALID_ARG;
        b200mp::g_multi_tune = value;
        return B200MP_OK;
    }
    if (strcmp(name, "attn_staged") == 0) {
        if (value < 0 || value > 2) return B200MP_ERR_INVALID_ARG;      // 2: staged + one-warp CTAs (forward, source sweep)
        b200mp::g_attn_staged = value;
        return B200MP_OK;
    }
    // GEMM knobs: validated and accepted so that existing callers keep working, but the sm_90a wgmma GEMM
    // (csrc/gemm_tf32x3.cu) has one configuration, so they do not change what runs
    if (strcmp(name, "gemm_prefetch") == 0) return (value < 0 || value > 64) ? B200MP_ERR_INVALID_ARG : B200MP_OK;
    if (strcmp(name, "gemm_debug") == 0) return B200MP_OK;
    if (strcmp(name, "gemm_mode") == 0) return (value != 0 && value != 1) ? B200MP_ERR_INVALID_ARG : B200MP_OK;
    if (strcmp(name, "gemm_bk") == 0) return (value != 16 && value != 32) ? B200MP_ERR_INVALID_ARG : B200MP_OK;
    b200mp::set_error("unknown option %s", name);
    return B200MP_ERR_INVALID_ARG;
}

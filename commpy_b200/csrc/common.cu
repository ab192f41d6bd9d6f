// Status strings, device properties, scratch allocation (host-side plumbing of libcommpy_b200.so).
#include <atomic>
#include <mutex>
#include <unordered_map>

#include "common.cuh"

namespace cpb {

thread_local char g_cuda_err[256] = "";

static std::atomic<int> g_options[CPB_OPT_COUNT];
int option(int id) { return (id >= 0 && id < CPB_OPT_COUNT) ? g_options[id].load(std::memory_order_relaxed) : 0; }
int set_option(int id, int v)
{
    if (id < 0 || id >= CPB_OPT_COUNT) return CPB_EINVAL;
    g_options[id].store(v, std::memory_order_relaxed);
    return CPB_OK;
}

int record_cuda_error(cudaError_t e, const char *what, const char *file, int line)
{
    snprintf(g_cuda_err, sizeof(g_cuda_err), "%s at %s:%d: %s", what, file, line, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? CPB_ENOMEM : CPB_ECUDA;
}

const DeviceProps &device_props()
{
    static thread_local DeviceProps cache[64];
    static thread_local bool have[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    if (!have[dev]) {
        DeviceProps p{};
        int v = 0;
        cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev); p.sm_count = v;
        cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, dev); p.cc_major = v;
        cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, dev); p.cc_minor = v;
        cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev); p.smem_optin = (size_t)v;
        // keep stream-ordered scratch cached in the default pool instead of returning it to the OS at every sync
        cudaMemPool_t pool = nullptr;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess && pool) {
            unsigned long long thr = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
        }
        size_t fr = 0, tot = 0;
        cudaMemGetInfo(&fr, &tot);
        p.global_mem = tot;
        cache[dev] = p;
        have[dev] = true;
    }
    return cache[dev];
}

int ensure_dyn_smem(const void *kernel, size_t bytes, bool max_carveout)
{
    static std::mutex mu;
    static std::unordered_map<unsigned long long, size_t> done;      // (kernel, device) -> largest size opted in
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long key = (unsigned long long)(uintptr_t)kernel * 131ull + (unsigned long long)dev;
    std::lock_guard<std::mutex> lock(mu);
    auto it = done.find(key);
    if (it != done.end() && it->second >= bytes) return CPB_OK;
    CPB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    // kernels that get nothing from L1 ask for the largest shared-memory carve-out, so that the driver's own choice of
    // carve-out cannot hold the step-major MAP kernel below the 12 CTAs per SM its registers allow.  (Not for kernels that
    // re-read the other half of a 32-byte sector from L1, like the frame-major MAP kernel: they need the L1.)
    if (max_carveout)
        CPB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    done[key] = bytes;
    return CPB_OK;
}

static std::mutex g_pool_mu;
static std::unordered_map<int, cudaMemPool_t> g_pools;      // device -> the library's scratch pool

int release_scratch_pool()
{
    int dev = 0;
    CPB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(g_pool_mu);
    auto it = g_pools.find(dev);
    if (it != g_pools.end()) CPB_CUDA(cudaMemPoolTrimTo(it->second, 0));
    return CPB_OK;
}

int Scratch::acquire(void *user, size_t user_bytes, size_t need, cudaStream_t s)
{
    stream = s;
    if (need == 0) { ptr = nullptr; owned = false; return CPB_OK; }
    if (user != nullptr) {
        if (user_bytes < need) return CPB_EINVAL;
        ptr = user; owned = false;
        return CPB_OK;
    }
    // the library's own stream-ordered pool (one per device), which keeps what it has been given: with the default pool's
    // release threshold of 0 every synchronisation returned the scratch to the driver and the next call paid for gigabytes
    // of fresh physical memory (the host-buffer pipelines synchronise once per call)
    int dev = 0;
    CPB_CUDA(cudaGetDevice(&dev));
    cudaMemPool_t pool = nullptr;
    {
        std::lock_guard<std::mutex> lock(g_pool_mu);
        auto &pools = g_pools;
        auto it = pools.find(dev);
        if (it == pools.end()) {
            cudaMemPoolProps props{};
            props.allocType = cudaMemAllocationTypePinned;
            props.handleTypes = cudaMemHandleTypeNone;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = dev;
            CPB_CUDA(cudaMemPoolCreate(&pool, &props));
            uint64_t keep = UINT64_MAX;
            CPB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
            pools[dev] = pool;
        } else {
            pool = it->second;
        }
    }
    CPB_CUDA(cudaMallocFromPoolAsync(&ptr, need, pool, s));
    owned = true;
    return CPB_OK;
}

void Scratch::release()
{
    if (owned && ptr) cudaFreeAsync(ptr, stream);
    ptr = nullptr; owned = false;
}

}  // namespace cpb

extern "C" {

const char *cpb_strerror(int status)
{
    switch (status) {
    case CPB_OK: return "ok";
    case CPB_EINVAL: return "invalid argument";
    case CPB_EUNSUPPORTED: return "configuration not supported by the H100 path";
    case CPB_ECUDA: return "CUDA runtime error (see cpb_last_cuda_error)";
    case CPB_ENOMEM: return "out of device memory";
    case CPB_ETRELLIS: return "trellis state without exactly 2^k predecessors";
    default: return "unknown status";
    }
}

const char *cpb_last_cuda_error(void) { return cpb::g_cuda_err; }

int cpb_version(void) { return 200; }

int cpb_set_option(int option_id, int value) { return cpb::set_option(option_id, value); }
int cpb_get_option(int option_id, int *value)
{
    if (!value || option_id < 0 || option_id >= CPB_OPT_COUNT) return CPB_EINVAL;
    *value = cpb::option(option_id);
    return CPB_OK;
}

int cpb_release_scratch(void) { return cpb::release_scratch_pool(); }

int cpb_device_info(int *sm_count, int *cc_major, int *cc_minor, size_t *global_mem_bytes)
{
    int n = 0;
    CPB_CUDA(cudaGetDeviceCount(&n));
    if (n <= 0) return CPB_ECUDA;
    const cpb::DeviceProps &p = cpb::device_props();
    if (sm_count) *sm_count = p.sm_count;
    if (cc_major) *cc_major = p.cc_major;
    if (cc_minor) *cc_minor = p.cc_minor;
    if (global_mem_bytes) *global_mem_bytes = p.global_mem;
    return CPB_OK;
}

}  // extern "C"

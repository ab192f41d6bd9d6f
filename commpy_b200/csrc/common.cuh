// Shared helpers for the commpy_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/commpy_b200.h"

namespace cpb {

// last CUDA error text, per host thread (returned by cpb_last_cuda_error()).
extern thread_local char g_cuda_err[256];
int record_cuda_error(cudaError_t e, const char *what, const char *file, int line);

#define CPB_CUDA(call)                                                              \
    do {                                                                            \
        cudaError_t e__ = (call);                                                   \
        if (e__ != cudaSuccess) return cpb::record_cuda_error(e__, #call, __FILE__, __LINE__); \
    } while (0)

#define CPB_LAUNCH_CHECK() CPB_CUDA(cudaGetLastError())

struct DeviceProps {
    int sm_count;
    int cc_major, cc_minor;
    size_t smem_optin;   // max dynamic shared memory per block (opt-in)
    size_t global_mem;
};
const DeviceProps &device_props();   // cached for the current device

// Stream-ordered scratch that falls back to a caller-supplied workspace.
struct Scratch {
    void *ptr = nullptr;
    bool owned = false;
    cudaStream_t stream = nullptr;
    int acquire(void *user, size_t user_bytes, size_t need, cudaStream_t s);
    void release();
};

// the decoders' scratch comes from a library-owned stream-ordered pool (one per device) that keeps what it has been given;
// this hands the unused part back to the driver (cpb_release_scratch)
int release_scratch_pool();

// cudaFuncAttributeMaxDynamicSharedMemorySize opt-in, made once per (kernel, device) and size: launches do not pay for it
int ensure_dyn_smem(const void *kernel, size_t bytes, bool max_carveout = false);

// explicit test / experiment switches (cpb_set_option); read with relaxed atomics, never from the environment
int option(int id);

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

}  // namespace cpb

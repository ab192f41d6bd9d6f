// Opaque handle bodies shared between translation units, and the host-buffer pipeline context a handle owns.
#pragma once
#include <functional>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace cpb {

// H2D(chunk i+1) || kernels(chunk i) || D2H(chunk i-1) on three internal streams with persistent device buffers.
// One context per HANDLE (trellis / LDPC code / modem), created on first use and freed with the handle: no global
// state; calls on the same handle serialise on the handle's own mutex, calls on different handles run concurrently.
struct PipeCtx {
    static constexpr int NS = 3;
    std::mutex mu;
    bool ready = false;
    int device = -1;
    cudaStream_t st[NS] = {nullptr, nullptr, nullptr};
    void *din[NS] = {nullptr, nullptr, nullptr};
    void *dout[NS] = {nullptr, nullptr, nullptr};
    size_t cap_in = 0, cap_out = 0;
    ~PipeCtx();
};

struct HostSeg {            // one per-frame array of a batched call
    const void *in;         // host source (inputs) ...
    void *out;              // ... or host destination (outputs)
    size_t stride;          // bytes per frame
};

// Runs `launch(din, dout, first_frame, n_frames, stream)` over chunks of `chunk` frames; din[k] / dout[k] are the
// device copies of ins[k] / outs[k] for that chunk.  Returns after every output host buffer is complete.
using PipeLaunch = std::function<int(const std::vector<void *> &, const std::vector<void *> &, int64_t, int64_t, cudaStream_t)>;
int pipe_run(PipeCtx &c, const std::vector<HostSeg> &ins, const std::vector<HostSeg> &outs, int64_t batch, int64_t chunk,
             const PipeLaunch &launch);
int64_t pipe_chunk(int64_t batch, int64_t min_chunk, int64_t multiple);

}  // namespace cpb

struct cpbTrellis {
    int k, n, M, S, I;
    std::vector<int32_t> next_state, output;   // host copies, S x I
    int32_t *pred_dev = nullptr;               // S*I entries: prev_state | input<<8 | output<<16, (p asc, u asc)
    int32_t *next_dev = nullptr, *out_dev = nullptr;   // S x I tables on the device (BCJR)
    int fast_id = 0;
    int device = 0;
    cpb::PipeCtx pipe;                         // host-buffer pipeline of cpb_*_host calls made with this handle
};

namespace cpb {

// Systematic LDPC encoder plans of one code (ldpclink.cu), built on first use: [0] peeled, [1] dense.  status < 0: not
// built yet, else the cpb status the build returned (a singular code is refused on every call without redoing the work).
struct LdpcEncPlan;
struct LdpcEncCache {
    std::mutex mu;
    LdpcEncPlan *plan[2] = {nullptr, nullptr};
    int status[2] = {-1, -1};
    ~LdpcEncCache();
};

}  // namespace cpb

struct cpbLdpc {
    cpb::PipeCtx pipe;                                  // host-buffer pipeline of cpb_ldpc_*_host calls made with this handle
    int m, n, nnz;
    int max_row_deg, max_col_deg;
    int32_t *row_ptr = nullptr, *col_idx = nullptr;     // CSR
    int32_t *col_ptr = nullptr, *col_edge = nullptr;    // CSC: edge ids (CSR positions) of a column, ascending check
    std::vector<int32_t> host_row_ptr, host_col_idx;    // host copy of the CSR, for the encoder plan
    cpb::LdpcEncCache enc;
};

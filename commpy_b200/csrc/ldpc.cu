// LDPC min-sum belief propagation on sm_90a -- replaces the per-edge Python loop of
// commpy/channelcoding/ldpc.py:229-238 (MSA check-node update), :243-248 (variable-node update) and the
// early-stop test of :205, for a batch of blocks at once (the reference walks blocks sequentially, :197).
//
// Formulation.  Only the check-to-variable messages R (one per edge, CSR order) and the posteriors
// post_j = sum_i R_ij + llr_j are stored; the variable-to-check message the reference keeps explicitly,
// Q_ij = (tot_j + llr_j) - R_ij (:243-245), is recomputed as post_j - R_ij when the check node needs it:
// the same fp operation on the same operands, so nothing changes numerically.  Per iteration
//   check pass (one thread per check x frame group): gather post_j of the row, syndrome parity from
//        signbit(post_j) (:205 -- evaluated on the previous iteration's posteriors, i.e. BEFORE this
//        iteration, like the reference), two-minimum + sign parity, write R_ij = prod sign(others) * min|others|;
//   variable pass (one thread per variable x frame group): tot_j = sum_i R_ij in ascending check index
//        (the reference's summation order), post_j = tot_j + llr_j.  Frames whose syndrome was already zero
//        are frozen here: their posteriors stay those of the previous iteration, exactly the reference's break.
// Layout: frames are the innermost dimension of every array ([chunk][edge][frame], [variable][frame]), so each
// access is a coalesced 16-byte vector (float4 = 4 frames, double2 = 2 frames) whatever the edge index,
// and the CSR/CSC index reads are warp-uniform.  For batches of >= 128 frames the min-sum check pass is
// bulk::cn_bulk_kernel, which stages whole rows through shared memory with the bulk-copy engine (see below).  Algorithmic HBM traffic per frame-iteration: 12*E + 8*n bytes
// in fp32 (read R + write R in the check pass, read R in the variable pass, read llr + write post).
//
// CPB_LDPC_FP64 runs the same kernels in double: min-sum is only abs/min/negate/add/sub, the adds happen in
// the reference's order and no multiply exists to be contracted into an FMA, so decisions, iteration counts
// and out_llrs equal the float64 reference bit for bit.
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "common.cuh"
#include "handles.cuh"

using namespace cpb;

cpb::PipeCtx &cpb_ldpc_pipe(cpbLdpc *h) { return h->pipe; }
void cpb_ldpc_dims(const cpbLdpc *h, int *m, int *n) { *m = h->m; *n = h->n; }

namespace ldpc {

template <typename T> struct VecOf;
template <> struct VecOf<float> { static constexpr int V = 4; struct alignas(16) type { float v[4]; }; };
template <> struct VecOf<double> { static constexpr int V = 2; struct alignas(16) type { double v[2]; }; };

// R (check-to-variable messages) is stored chunk-major: [frame chunk][edge][RS frames], RS = frames per chunk
// (RS = F, one chunk, unless the bulk-copy check pass is in use), so that the rows of one check node and one
// chunk are contiguous.
struct RLayout {
    int RS;                // frames per chunk (row stride)
    int64_t chunk_elems;   // nnz * RS
    template <typename T> __device__ __forceinline__ T *at(T *R, int64_t f) const { return R + (f / RS) * chunk_elems + (f % RS); }
};

struct State {
    int32_t *unsat_iter;   // [F] last iteration (1-based) at which an unsatisfied check was seen
    int32_t *done;         // [F]
    int32_t *iters;        // [F]
};

// llr[f][j] (clipped in place, ldpc.py:186) -> llrT[j][F], post[j][F]; padded frames get +1 (a codeword)
template <typename T>
__global__ void __launch_bounds__(256) load_kernel(T *__restrict__ llr, int64_t batch, int n, int64_t F,
                                                   T *__restrict__ llrT, T *__restrict__ post)
{
    __shared__ T tile[32][33];
    const int64_t f0 = (int64_t)blockIdx.y * 32;
    const int j0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
    for (int r = ty; r < 32; r += 8) {
        const int64_t f = f0 + r;
        const int j = j0 + tx;
        T v = (T)1;
        if (f < batch && j < n) {
            v = llr[f * n + j];
            v = v > (T)500 ? (T)500 : (v < (T)-500 ? (T)-500 : v);
            llr[f * n + j] = v;
        }
        tile[r][tx] = v;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int j = j0 + r;
        const int64_t f = f0 + tx;
        if (j < n && f < F) {
            const T v = tile[tx][r];
            llrT[(int64_t)j * F + f] = v;
            post[(int64_t)j * F + f] = v;
        }
    }
}

template <typename T>
__global__ void __launch_bounds__(256) store_kernel(const T *__restrict__ post, int64_t batch, int n, int64_t F,
                                                    uint8_t *__restrict__ dec, T *__restrict__ out_llr)
{
    __shared__ T tile[32][33];
    const int64_t f0 = (int64_t)blockIdx.y * 32;
    const int j0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int r = ty; r < 32; r += 8) {
        const int j = j0 + r;
        const int64_t f = f0 + tx;
        tile[r][tx] = (j < n && f < F) ? post[(int64_t)j * F + f] : (T)0;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int64_t f = f0 + r;
        const int j = j0 + tx;
        if (f < batch && j < n) {
            const T v = tile[tx][r];
            dec[f * n + j] = (uint8_t)(signbit(v) ? 1 : 0);       // ldpc.py:193,248 (-0.0 -> 1)
            if (out_llr) out_llr[f * n + j] = v;
        }
    }
}

__global__ void finish_iters_kernel(const State st, int64_t batch, int n_iters, int32_t *iters_out)
{
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f < batch) iters_out[f] = st.done[f] ? st.iters[f] : n_iters;
}

// DEGMAX > 0: rows of degree <= DEGMAX keep their variable-to-check messages in registers between the two passes
// (one read of R and post per edge); DEGMAX == 0: any degree, messages are recomputed in the second pass.
template <typename T, int DEGMAX>
__global__ void __launch_bounds__(256) cn_kernel(const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ col_idx,
                                                 int m, int64_t F, int iter, const T *__restrict__ post,
                                                 T *__restrict__ Rbase, const State st, const RLayout rl)
{
    using VT = typename VecOf<T>::type;
    constexpr int V = VecOf<T>::V;
    constexpr int QN = (DEGMAX > 0) ? DEGMAX : 1;
    const int64_t G = F / V;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)m * G) return;
    const int i = (int)(gid / G);
    const int64_t f = (gid - (int64_t)i * G) * V;
    T *const Rf = rl.at(Rbase, f);
    const int64_t RS = rl.RS;
    bool act[V];
    bool any = false;
#pragma unroll
    for (int v = 0; v < V; ++v) { act[v] = st.done[f + v] == 0; any |= act[v]; }
    if (!any) return;
    const int e0 = __ldg(&row_ptr[i]), e1 = __ldg(&row_ptr[i + 1]);
    T min1[V], min2[V];
    int arg[V], neg[V], par[V];
#pragma unroll
    for (int v = 0; v < V; ++v) { min1[v] = (T)INFINITY; min2[v] = (T)INFINITY; arg[v] = -1; neg[v] = 0; par[v] = 0; }
    VT q[QN];
    const int deg = e1 - e0;
    if (DEGMAX > 0) {
        // issue every load of the row before the first use (edges past the row's degree re-read its last edge, so
        // no load is predicated and the memory system sees 2*DEGMAX independent 16-byte requests per thread)
        int cix[QN];
#pragma unroll
        for (int k = 0; k < QN; ++k) cix[k] = __ldg(&col_idx[min(e0 + k, e1 - 1)]);
        VT pv[QN];
#pragma unroll
        for (int k = 0; k < QN; ++k) {
            pv[k] = *reinterpret_cast<const VT *>(post + (int64_t)cix[k] * F + f);
            q[k] = *reinterpret_cast<const VT *>(Rf + (int64_t)min(e0 + k, e1 - 1) * RS);
        }
#pragma unroll
        for (int k = 0; k < QN; ++k) {
            if (k < deg) {
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    par[v] ^= signbit(pv[k].v[v]) ? 1 : 0;
                    const T x = pv[k].v[v] - q[k].v[v];       // Q_ij = (tot_j + llr_j) - R_ij, ldpc.py:244-245
                    q[k].v[v] = x;
                    const T a = fabs(x);
                    neg[v] += (x < (T)0) ? 1 : 0;
                    // (a branch-free fmin/fmax form needs fewer instructions, but ptxas then sinks the post loads next
                    // to their uses, which exposes their latency)
                    if (a < min1[v]) { min2[v] = min1[v]; min1[v] = a; arg[v] = k; }
                    else if (a < min2[v]) min2[v] = a;
                }
            }
        }
    } else {
        for (int e = e0; e < e1; ++e) {
            const int c = __ldg(&col_idx[e]);
            const VT p = *reinterpret_cast<const VT *>(post + (int64_t)c * F + f);
            const VT r = *reinterpret_cast<const VT *>(Rf + (int64_t)e * RS);
#pragma unroll
            for (int v = 0; v < V; ++v) {
                par[v] ^= signbit(p.v[v]) ? 1 : 0;
                const T x = p.v[v] - r.v[v];
                const T a = fabs(x);
                neg[v] += (x < (T)0) ? 1 : 0;
                if (a < min1[v]) { min2[v] = min1[v]; min1[v] = a; arg[v] = e - e0; }
                else if (a < min2[v]) min2[v] = a;
            }
        }
    }
    // benign race: every writer stores the same value; test first so ~m writers per frame do not all hit one word
#pragma unroll
    for (int v = 0; v < V; ++v)
        if (act[v] && par[v] && st.unsat_iter[f + v] != iter + 1) st.unsat_iter[f + v] = iter + 1;
    if (DEGMAX > 0) {
#pragma unroll
        for (int k = 0; k < QN; ++k) {
            const int e = e0 + k;
            if (e < e1) {
                VT r;
                bool all = true;
#pragma unroll
                for (int v = 0; v < V; ++v) all &= act[v];
                if (!all) r = *reinterpret_cast<const VT *>(Rf + (int64_t)e * RS);     // keep finished frames' messages
#pragma unroll
                for (int v = 0; v < V; ++v) {
                    const T x = q[k].v[v];
                    const T mag = (k == arg[v]) ? min2[v] : min1[v];          // min over the OTHER edges (:238)
                    const int ng = neg[v] - ((x < (T)0) ? 1 : 0);
                    const T val = (ng & 1) ? -mag : mag;                      // prod of sign(others)
                    if (act[v]) r.v[v] = val;
                }
                *reinterpret_cast<VT *>(Rf + (int64_t)e * RS) = r;
            }
        }
    } else {
        for (int e = e0; e < e1; ++e) {
            const int c = __ldg(&col_idx[e]);
            const VT p = *reinterpret_cast<const VT *>(post + (int64_t)c * F + f);
            VT r = *reinterpret_cast<const VT *>(Rf + (int64_t)e * RS);
#pragma unroll
            for (int v = 0; v < V; ++v) {
                const T x = p.v[v] - r.v[v];
                const T mag = ((e - e0) == arg[v]) ? min2[v] : min1[v];
                const int ng = neg[v] - ((x < (T)0) ? 1 : 0);
                const T val = (ng & 1) ? -mag : mag;
                if (act[v]) r.v[v] = val;
            }
            *reinterpret_cast<VT *>(Rf + (int64_t)e * RS) = r;
        }
    }
}

// ---- check pass staged through shared memory by the bulk-copy engine (TMA, cp.async.bulk) -------------------------------
// With frames innermost, the messages of one edge for a chunk of FT frames are ONE contiguous row of FT*sizeof(T) bytes
// (1 KB at FT = 256 floats), and so is the posterior row the edge gathers.  A persistent CTA therefore walks tiles
// (check node i, frame chunk c): warp 0 asks the copy engine for the 2*deg rows of a tile (lane k <-> edge k) and an
// mbarrier counts the bytes as they land; FT threads (one frame each) run the two-minimum update on the staged rows in
// place; warp 0 hands the R rows back to the copy engine (bulk store).  NSTAGE tiles rotate, loads run NSTAGE-2 tiles
// ahead, so the memory system always holds several KB per CTA in flight without a register being spent on it -- in the
// register-staged kernel above, loads, math and stores share the same 16 warps per SM, which limits the bytes in flight.
// Same arithmetic, same order: results are bit-identical to cn_kernel.
namespace bulk {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *b, int count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *b, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *b)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *b, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void load_row(void *dst_smem, const void *src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void store_row(void *dst, const void *src_smem, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

constexpr int MAXDEG = 32;      // lane k of the producer warp owns edge k
constexpr int NSTAGE = 6;       // tiles resident in shared memory
constexpr int LAG = 4;          // a tile's rows are stored LAG tiles after its loads were issued

// Min-sum update of one staged row for one frame: rs[k*FT] = R_ik (in/out), ps[k*FT] = posterior of the edge's variable.
// Same operations in the same order as cn_kernel (Q = post - R; first minimum keeps the lowest edge index; a message's
// sign is the parity of the strictly negative OTHER Q's), written without data-dependent branches.
// Returns the syndrome parity of the row (signbit of the posteriors, ldpc.py:193,205).
template <typename T, int DEG>
__device__ __forceinline__ int consume_row(T *rs, const T *ps, int FT, bool act)
{
    T x[DEG];
    T min1 = (T)INFINITY, min2 = (T)INFINITY;
    int arg = -1, par = 0;
    unsigned negmask = 0;
#pragma unroll
    for (int k = 0; k < DEG; ++k) {
        const T p = ps[(size_t)k * FT];
        par ^= signbit(p) ? 1 : 0;
        x[k] = p - rs[(size_t)k * FT];                       // Q_ij = (tot_j + llr_j) - R_ij, ldpc.py:244-245
    }
#pragma unroll
    for (int k = 0; k < DEG; ++k) {
        const T a = fabs(x[k]);
        if (x[k] < (T)0) negmask |= 1u << k;
        const bool lt = a < min1;
        min2 = fmin(min2, fmax(a, min1));
        min1 = fmin(min1, a);
        arg = lt ? k : arg;
    }
    if (act) {
        const unsigned flip = (__popc(negmask) & 1) ? ~negmask : negmask;   // bit k: odd number of negative OTHER messages
#pragma unroll
        for (int k = 0; k < DEG; ++k) {
            const T mag = (k == arg) ? min2 : min1;              // min over the OTHER edges (:238)
            rs[(size_t)k * FT] = ((flip >> k) & 1u) ? -mag : mag;   // prod of sign(others)
        }
    }
    return par;
}

template <typename T>
__device__ __forceinline__ int consume_row_any(T *rs, const T *ps, int FT, int deg, bool act)
{
    T min1 = (T)INFINITY, min2 = (T)INFINITY;
    int arg = -1, neg = 0, par = 0;
    for (int k = 0; k < deg; ++k) {
        const T p = ps[(size_t)k * FT];
        par ^= signbit(p) ? 1 : 0;
        const T x = p - rs[(size_t)k * FT];
        const T a = fabs(x);
        neg += (x < (T)0) ? 1 : 0;
        if (a < min1) { min2 = min1; min1 = a; arg = k; }
        else if (a < min2) min2 = a;
    }
    if (act) {
        for (int k = 0; k < deg; ++k) {
            const T x = ps[(size_t)k * FT] - rs[(size_t)k * FT];
            const T mag = (k == arg) ? min2 : min1;
            const int ng = neg - ((x < (T)0) ? 1 : 0);
            rs[(size_t)k * FT] = (ng & 1) ? -mag : mag;
        }
    }
    return par;
}

// CTA = FT consumer threads (one frame each) + one producer warp.  A CTA owns one frame chunk and every
// (gridDim.x / nchunks)-th check node.  Producer step t:  wait until the consumers are done with tile t-LAG, bulk-store
// its R rows;  wait until the stores of tile t-NSTAGE have left shared memory, bulk-load tile t into that stage.
// Consumers: wait for the bytes of tile t, update the rows in place, signal the producer.  No block-wide barrier.
template <typename T>
__global__ void __launch_bounds__(288) cn_bulk_kernel(const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ col_idx,
                                                      int m, int64_t F, int iter, const T *__restrict__ post,
                                                      T *__restrict__ R, const State st, int nchunks, int maxdeg, int64_t nnz)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int FT = blockDim.x - 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ncw = FT >> 5;                                     // consumer warps
    const size_t stage_elems = (size_t)2 * maxdeg * FT;
    T *tiles = reinterpret_cast<T *>(smem_raw);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + (size_t)NSTAGE * stage_elems * sizeof(T));
    uint64_t *comp = full + NSTAGE;
    int *info = reinterpret_cast<int *>(comp + NSTAGE);          // [NSTAGE][2]: degree, first edge
    const int c = (int)(blockIdx.x % nchunks);                   // frame chunk of this CTA
    const int i0 = (int)(blockIdx.x / nchunks), istride = (int)(gridDim.x / nchunks);
    const int mine = (i0 < m) ? (m - i0 + istride - 1) / istride : 0;
    const int64_t f0 = (int64_t)c * FT;
    const int nfr = (int)min((int64_t)FT, F - f0);
    const uint32_t row_bytes = (uint32_t)nfr * (uint32_t)sizeof(T);
    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&comp[s], ncw); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // frames that already satisfied their syndrome are frozen (ldpc.py:205): a chunk without a live frame is skipped
    bool act = false;
    if (tid < nfr) act = st.done[f0 + tid] == 0;
    const int any_live = __syncthreads_or(act ? 1 : 0);
    if (!any_live || mine == 0) return;

    if (warp == ncw) {
        // ------------------------------------------------ producer warp
        // R is chunk-major, so the deg rows of a tile are one contiguous block: one bulk load and one bulk store per tile
        // (lane 0), plus one bulk load per gathered posterior row (lane k <-> edge k).
        T *const Rc = R + (int64_t)c * nnz * FT;
        // index prefetch: row_ptr two tiles ahead, col_idx one tile ahead, so no step waits on a dependent load
        int e0_n, e1_n, col_n, e0_nn = 0, e1_nn = 0;
        e0_n = __ldg(&row_ptr[i0]); e1_n = __ldg(&row_ptr[i0 + 1]);
        col_n = (lane < e1_n - e0_n) ? __ldg(&col_idx[e0_n + lane]) : 0;
        if (mine > 1) { e0_nn = __ldg(&row_ptr[i0 + istride]); e1_nn = __ldg(&row_ptr[i0 + istride + 1]); }
        for (int t = 0; t < mine + LAG; ++t) {
            const int u = t - LAG;
            if (u >= 0) {                                        // store tile u
                const int su = u % NSTAGE;
                mbar_wait(&comp[su], (uint32_t)((u / NSTAGE) & 1));
                if (lane == 0) {
                    const int deg = info[su * 2 + 0], e0 = info[su * 2 + 1];
                    store_row(Rc + (int64_t)e0 * FT, tiles + (size_t)su * stage_elems, (uint32_t)deg * row_bytes);
                }
                commit_group();
            }
            if (t < mine) {                                      // load tile t
                const int s = t % NSTAGE;
                const int e0 = e0_n, deg = e1_n - e0_n, col = col_n;
                if (t + 1 < mine) {
                    e0_n = e0_nn; e1_n = e1_nn;
                    col_n = (lane < e1_n - e0_n) ? __ldg(&col_idx[e0_n + lane]) : 0;
                    if (t + 2 < mine) {
                        const int i = i0 + (t + 2) * istride;
                        e0_nn = __ldg(&row_ptr[i]); e1_nn = __ldg(&row_ptr[i + 1]);
                    }
                }
                wait_group_read<NSTAGE - LAG>();                 // stores of tile t-NSTAGE have been read out of this stage
                T *rs = tiles + (size_t)s * stage_elems;
                if (lane == 0) {
                    info[s * 2 + 0] = deg; info[s * 2 + 1] = e0;
                    mbar_expect_tx(&full[s], 2u * (uint32_t)deg * row_bytes);
                    load_row(rs, Rc + (int64_t)e0 * FT, (uint32_t)deg * row_bytes, &full[s]);
                }
                __syncwarp();
                if (lane < deg)
                    load_row(rs + (size_t)(maxdeg + lane) * FT, post + (int64_t)col * F + f0, row_bytes, &full[s]);
            }
        }
        wait_group_read<0>();               // shared memory must outlive the last stores
        return;
    }

    // ---------------------------------------------------- consumers: thread <-> frame f0 + tid
    const bool valid = tid < nfr;
    const int64_t f = f0 + tid;
    int unsat = 0;
    for (int t = 0; t < mine; ++t) {
        const int s = t % NSTAGE;
        mbar_wait(&full[s], (uint32_t)((t / NSTAGE) & 1));
        const int deg = info[s * 2 + 0];
        T *rs = tiles + (size_t)s * stage_elems + tid;
        const T *ps = rs + (size_t)maxdeg * FT;
        if (valid) {
            int par;
            switch (deg) {                      // warp-uniform: fully unrolled bodies for the common short rows
            case 2: par = consume_row<T, 2>(rs, ps, FT, act); break;
            case 3: par = consume_row<T, 3>(rs, ps, FT, act); break;
            case 4: par = consume_row<T, 4>(rs, ps, FT, act); break;
            case 5: par = consume_row<T, 5>(rs, ps, FT, act); break;
            case 6: par = consume_row<T, 6>(rs, ps, FT, act); break;
            case 7: par = consume_row<T, 7>(rs, ps, FT, act); break;
            case 8: par = consume_row<T, 8>(rs, ps, FT, act); break;
            default: par = consume_row_any<T>(rs, ps, FT, deg, act); break;
            }
            unsat |= par;
        }
        fence_proxy_async();                // the copy engine must see the rows just written
        __syncwarp();
        if (lane == 0) mbar_arrive(&comp[s]);
    }
    // one flag store per frame and CTA (every writer stores the same value)
    if (valid && act && unsat && st.unsat_iter[f] != iter + 1) st.unsat_iter[f] = iter + 1;
}

template <typename T>
static size_t smem_bytes(int maxdeg, int FT)
{
    return (size_t)NSTAGE * 2 * maxdeg * FT * sizeof(T) + (size_t)NSTAGE * (2 * sizeof(uint64_t) + 2 * sizeof(int));
}

}  // namespace bulk

// The NaN an x86 CPU produces for 0 * inf (sign bit set), and the quiet NaN with a clear sign bit.
template <typename T> __device__ __forceinline__ T x86_default_nan();
template <> __device__ __forceinline__ float x86_default_nan<float>() { return __int_as_float(0xffc00000u); }
template <> __device__ __forceinline__ double x86_default_nan<double>() { return __longlong_as_double(0xfff8000000000000ull); }
template <typename T> __device__ __forceinline__ T positive_nan();
template <> __device__ __forceinline__ float positive_nan<float>() { return __int_as_float(0x7fc00000u); }
template <> __device__ __forceinline__ double positive_nan<double>() { return __longlong_as_double(0x7ff8000000000000ull); }

// Sum-product check node (ldpc.py:209-227): t = tanh(Q/2), R_ij = 2 atanh(clip((prod_row t) / t_ij, -1, 1)) clipped to
// +-500.  Same formula as the reference (product of the whole row divided by the edge's own factor); the product is
// formed directly instead of through exp2(sum(log2(complex))).  Q_ij is formed in the message type T, everything after
// it in double whatever T is, and R is rounded to T once: an fp32 message can then take any value up to the reference's
// saturation knee 2 atanh(1 - 2^-53) ~ 37.4 (in float the knee would be 2 atanh(1 - 2^-24) ~ 17.3, and every message
// between 17.3 and 37.4 would jump to 500).  Conditioning: with x = prod/t_ij computed to a relative error rho
// (~3 deg eps here, eps = 2^-53, plus the reference's own log2/exp2 error), |dR| <= 2 atanh(|x|(1+rho)) - 2 atanh(|x|)
// ~ 2 rho |x| cosh^2(R/2), so a message near the knee may legitimately come out as ~37 in one and 500 in the other.
// Exact zeros: tanh(+-0) = +-0 makes the product +-0 (sign = parity of the sign bits, as the reference's complex log
// counts arg(-0) = pi) and the zero edge's own message (1/+-0) * +-0 = NaN.  On x86 that NaN has its sign bit set, which
// the reference's decision signbit() turns into a 1; the kernel writes the same NaN, and vn_spa_kernel keeps its sign.
// A NaN that enters through Q has passed numpy's tanh, whose NaN is positive: the kernel writes a positive NaN then.
template <typename T>
__global__ void __launch_bounds__(256) cn_spa_kernel(const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ col_idx,
                                                     int m, int64_t F, int iter, const T *__restrict__ post,
                                                     T *__restrict__ Rbase, const State st, const RLayout rl)
{
    using VT = typename VecOf<T>::type;
    constexpr int V = VecOf<T>::V;
    const int64_t G = F / V;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)m * G) return;
    const int i = (int)(gid / G);
    const int64_t f = (gid - (int64_t)i * G) * V;
    T *const Rf = rl.at(Rbase, f);
    const int64_t RS = rl.RS;
    bool act[V];
    bool any = false;
#pragma unroll
    for (int v = 0; v < V; ++v) { act[v] = st.done[f + v] == 0; any |= act[v]; }
    if (!any) return;
    const int e0 = __ldg(&row_ptr[i]), e1 = __ldg(&row_ptr[i + 1]);
    double prod[V];
    int par[V];
#pragma unroll
    for (int v = 0; v < V; ++v) { prod[v] = 1.0; par[v] = 0; }
    for (int e = e0; e < e1; ++e) {
        const int c = __ldg(&col_idx[e]);
        const VT p = *reinterpret_cast<const VT *>(post + (int64_t)c * F + f);
        const VT r = *reinterpret_cast<const VT *>(Rf + (int64_t)e * RS);
#pragma unroll
        for (int v = 0; v < V; ++v) {
            par[v] ^= signbit(p.v[v]) ? 1 : 0;
            const T q = p.v[v] - r.v[v];                                 // Q_ij, ldpc.py:244-245
            prod[v] *= tanh((double)q * 0.5);
        }
    }
#pragma unroll
    for (int v = 0; v < V; ++v)
        if (act[v] && par[v] && st.unsat_iter[f + v] != iter + 1) st.unsat_iter[f + v] = iter + 1;
    for (int e = e0; e < e1; ++e) {
        const int c = __ldg(&col_idx[e]);
        const VT p = *reinterpret_cast<const VT *>(post + (int64_t)c * F + f);
        VT r = *reinterpret_cast<const VT *>(Rf + (int64_t)e * RS);
#pragma unroll
        for (int v = 0; v < V; ++v) {
            const T q = p.v[v] - r.v[v];
            const double t = tanh((double)q * 0.5);
            double x = (1.0 / t) * prod[v];
            x = x > 1.0 ? 1.0 : (x < -1.0 ? -1.0 : x);               // NaN passes through, as in numpy
            x = atanh(x) * 2.0;
            x = x > 500.0 ? 500.0 : (x < -500.0 ? -500.0 : x);
            // a NaN made here ((1/+-0) * +-0) has the sign bit set, one that came in through Q has it clear, whatever
            // sign the device's tanh/atanh pass on (its tanh keeps the sign of a NaN argument, numpy's does not)
            const T y = isnan(x) ? (isnan(prod[v]) ? positive_nan<T>() : x86_default_nan<T>()) : (T)x;
            if (act[v]) r.v[v] = y;
        }
        *reinterpret_cast<VT *>(Rf + (int64_t)e * RS) = r;
    }
}

// NAN_SIGN: a posterior that is NaN takes the sign bit of the first NaN message of the column, as x86 addition passes
// a NaN operand through unchanged (the GPU's add returns its own NaN).  Only the sum-product decoder makes NaN messages.
template <typename T, bool NAN_SIGN>
__device__ __forceinline__ void vn_body(const int32_t *__restrict__ col_ptr, const int32_t *__restrict__ col_edge,
                                        int n, int64_t F, int iter, const T *__restrict__ llrT,
                                        const T *__restrict__ Rbase, T *__restrict__ post, const State st,
                                        const RLayout rl)
{
    using VT = typename VecOf<T>::type;
    constexpr int V = VecOf<T>::V;
    const int64_t G = F / V;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)n * G) return;
    const int j = (int)(gid / G);
    const int64_t f = (gid - (int64_t)j * G) * V;
    const T *const Rf = rl.at(Rbase, f);
    const int64_t RS = rl.RS;
    bool act[V];
    bool any = false;
#pragma unroll
    for (int v = 0; v < V; ++v) {
        const bool dn = st.done[f + v] != 0;
        const bool unsat = st.unsat_iter[f + v] == iter + 1;
        act[v] = !dn && unsat;
        any |= act[v];
        if (j == 0 && !dn && !unsat) {          // syndrome was zero before this iteration: the reference breaks (:205)
            st.done[f + v] = 1;
            st.iters[f + v] = iter;
        }
    }
    if (!any) return;
    const int c0 = __ldg(&col_ptr[j]), c1 = __ldg(&col_ptr[j + 1]);
    T tot[V];
    int nan_sign[V];                            // -1: no NaN message yet, else the sign bit of the first one
#pragma unroll
    for (int v = 0; v < V; ++v) { tot[v] = (T)0; nan_sign[v] = -1; }
    for (int q = c0; q < c1; ++q) {             // ascending check index = the reference's summation order
        const int e = __ldg(&col_edge[q]);
        const VT r = *reinterpret_cast<const VT *>(Rf + (int64_t)e * RS);
#pragma unroll
        for (int v = 0; v < V; ++v) {
            tot[v] += r.v[v];
            if (NAN_SIGN && nan_sign[v] < 0 && isnan(r.v[v])) nan_sign[v] = signbit(r.v[v]) ? 1 : 0;
        }
    }
    const VT l = *reinterpret_cast<const VT *>(llrT + (int64_t)j * F + f);
    VT p = *reinterpret_cast<const VT *>(post + (int64_t)j * F + f);
#pragma unroll
    for (int v = 0; v < V; ++v) {
        T x = tot[v] + l.v[v];                                          // ldpc.py:247
        if (NAN_SIGN && nan_sign[v] >= 0) x = copysign(x, nan_sign[v] ? (T)-1 : (T)1);
        if (act[v]) p.v[v] = x;
    }
    *reinterpret_cast<VT *>(post + (int64_t)j * F + f) = p;
}

template <typename T>
__global__ void __launch_bounds__(256) vn_kernel(const int32_t *__restrict__ col_ptr, const int32_t *__restrict__ col_edge,
                                                 int n, int64_t F, int iter, const T *__restrict__ llrT,
                                                 const T *__restrict__ Rbase, T *__restrict__ post, const State st,
                                                 const RLayout rl)
{
    vn_body<T, false>(col_ptr, col_edge, n, F, iter, llrT, Rbase, post, st, rl);
}

template <typename T>
__global__ void __launch_bounds__(256) vn_spa_kernel(const int32_t *__restrict__ col_ptr, const int32_t *__restrict__ col_edge,
                                                     int n, int64_t F, int iter, const T *__restrict__ llrT,
                                                     const T *__restrict__ Rbase, T *__restrict__ post, const State st,
                                                     const RLayout rl)
{
    vn_body<T, true>(col_ptr, col_edge, n, F, iter, llrT, Rbase, post, st, rl);
}

static size_t state_bytes(int64_t F) { return (size_t)F * sizeof(int32_t) * 3; }

template <typename T>
static size_t ws_bytes(const cpbLdpc *h, int64_t F)
{
    return ((size_t)h->nnz + 2 * (size_t)h->n) * F * sizeof(T) + state_bytes(F) + 256;
}

static int64_t pad_frames(int64_t batch) { return ceil_div(batch, 32) * 32; }

// frames per pass so that the workspace stays under ~6 GB
template <typename T>
static int64_t chunk_frames(const cpbLdpc *h, int64_t batch)
{
    const double per = ((double)h->nnz + 2.0 * h->n) * sizeof(T) + 12.0;
    int64_t c = (int64_t)(6.0e9 / per);
    c = (c / 32) * 32;
    if (c < 32) c = 32;
    return std::min<int64_t>(c, pad_frames(batch));
}

template <typename T>
static int run(const cpbLdpc *h, T *llr, int64_t batch, int n_iters, int spa, uint8_t *dec, T *out_llr, int32_t *iters_out,
               void *workspace, size_t workspace_bytes, cudaStream_t st)
{
    constexpr int V = VecOf<T>::V;
    const int64_t Fc = chunk_frames<T>(h, batch);
    Scratch ws;
    int rc = ws.acquire(workspace, workspace_bytes, ws_bytes<T>(h, Fc), st);
    if (rc) return rc;
    char *base = reinterpret_cast<char *>(ws.ptr);
    T *R = reinterpret_cast<T *>(base);
    T *post = R + (size_t)h->nnz * Fc;
    T *llrT = post + (size_t)h->n * Fc;
    State s;
    s.unsat_iter = reinterpret_cast<int32_t *>(llrT + (size_t)h->n * Fc);
    s.done = s.unsat_iter + Fc;
    s.iters = s.done + Fc;
    for (int64_t f0 = 0; f0 < batch; f0 += Fc) {
        const int64_t nb = std::min<int64_t>(Fc, batch - f0);
        const int64_t F = pad_frames(nb);
        cudaError_t e = cudaMemsetAsync(R, 0, (size_t)h->nnz * F * sizeof(T), st);
        if (e == cudaSuccess) e = cudaMemsetAsync(s.unsat_iter, 0, state_bytes(Fc), st);
        if (e != cudaSuccess) { ws.release(); return record_cuda_error(e, "cudaMemsetAsync", __FILE__, __LINE__); }
        // note: R/post/llrT use stride F (<= Fc) inside this chunk
        dim3 tgrid((unsigned)ceil_div(h->n, 32), (unsigned)(F / 32));
        load_kernel<T><<<tgrid, 256, 0, st>>>(llr + f0 * h->n, nb, h->n, F, llrT, post);
        const int64_t G = F / V;
        const unsigned cn_blocks = (unsigned)ceil_div((int64_t)h->m * G, 256);
        const unsigned vn_blocks = (unsigned)ceil_div((int64_t)h->n * G, 256);
        // bulk-copy staged check pass: min-sum, row degree <= 32, frame chunks of 256 or 128
        // (CPB_LDPC_NO_BULK=1 forces the register-staged kernels: used by the test that compares the two paths)
        bool use_bulk = !spa && h->max_row_deg <= bulk::MAXDEG && !option(CPB_OPT_LDPC_NO_BULK);
        int FT = (F % 256 == 0) ? 256 : ((F % 128 == 0) ? 128 : 0);
        int nchunks = 0, bulk_grid = 0;
        size_t bulk_smem = 0;
        if (FT == 0) use_bulk = false;
        if (use_bulk) {
            nchunks = (int)(F / FT);
            bulk_smem = bulk::smem_bytes<T>(h->max_row_deg, FT);
            if (bulk_smem > 200 * 1024) {
                use_bulk = false;
            } else {
                { const int rc_ = ensure_dyn_smem(reinterpret_cast<const void *>(bulk::cn_bulk_kernel<T>), bulk_smem); if (rc_) { ws.release(); return rc_; } }
                const DeviceProps &dp = device_props();
                const int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (size_t)(220 * 1024) / (bulk_smem + 1024)));
                int64_t want = (int64_t)(dp.sm_count > 0 ? dp.sm_count : 132) * per_sm;
                want = std::max<int64_t>(nchunks, (want / nchunks) * nchunks);        // a multiple of nchunks
                bulk_grid = (int)std::min<int64_t>((int64_t)h->m * nchunks, want);
            }
        }
        RLayout rl;
        rl.RS = use_bulk ? FT : (int)F;
        rl.chunk_elems = (int64_t)h->nnz * rl.RS;
        for (int it = 0; it < n_iters; ++it) {
            if (use_bulk)
                bulk::cn_bulk_kernel<T><<<bulk_grid, FT + 32, bulk_smem, st>>>(h->row_ptr, h->col_idx, h->m, F, it, post, R, s, nchunks,
                                                                             h->max_row_deg, (int64_t)h->nnz);
            else if (spa) cn_spa_kernel<T><<<cn_blocks, 256, 0, st>>>(h->row_ptr, h->col_idx, h->m, F, it, post, R, s, rl);
            else if (h->max_row_deg <= 8) cn_kernel<T, 8><<<cn_blocks, 256, 0, st>>>(h->row_ptr, h->col_idx, h->m, F, it, post, R, s, rl);
            else cn_kernel<T, 0><<<cn_blocks, 256, 0, st>>>(h->row_ptr, h->col_idx, h->m, F, it, post, R, s, rl);
            if (spa) vn_spa_kernel<T><<<vn_blocks, 256, 0, st>>>(h->col_ptr, h->col_edge, h->n, F, it, llrT, R, post, s, rl);
            else vn_kernel<T><<<vn_blocks, 256, 0, st>>>(h->col_ptr, h->col_edge, h->n, F, it, llrT, R, post, s, rl);
        }
        store_kernel<T><<<tgrid, 256, 0, st>>>(post, nb, h->n, F, dec + f0 * h->n, out_llr ? out_llr + f0 * h->n : nullptr);
        if (iters_out)
            finish_iters_kernel<<<(unsigned)ceil_div(nb, 256), 256, 0, st>>>(s, nb, n_iters, iters_out + f0);
        e = cudaGetLastError();
        if (e != cudaSuccess) { ws.release(); return record_cuda_error(e, "ldpc kernels", __FILE__, __LINE__); }
    }
    ws.release();
    return CPB_OK;
}

}  // namespace ldpc

extern "C" {

int cpb_ldpc_create(const int32_t *row_ptr, const int32_t *col_idx, int m, int n, cpbLdpc **out)
{
    if (!row_ptr || !col_idx || !out || m < 1 || n < 1) return CPB_EINVAL;
    const int nnz = row_ptr[m];
    if (row_ptr[0] != 0 || nnz < 1) return CPB_EINVAL;
    cpbLdpc *h = new cpbLdpc();
    h->m = m; h->n = n; h->nnz = nnz;
    std::vector<int32_t> col_ptr(n + 1, 0), col_edge(nnz), fill(n, 0);
    int maxr = 0;
    for (int i = 0; i < m; ++i) {
        const int deg = row_ptr[i + 1] - row_ptr[i];
        if (deg < 2) { delete h; return CPB_EINVAL; }         // the reference's min over an empty set raises
        maxr = std::max(maxr, deg);
        for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
            if (col_idx[e] < 0 || col_idx[e] >= n) { delete h; return CPB_EINVAL; }
            col_ptr[col_idx[e] + 1]++;
        }
    }
    int maxc = 0;
    for (int j = 0; j < n; ++j) { maxc = std::max(maxc, col_ptr[j + 1]); col_ptr[j + 1] += col_ptr[j]; }
    for (int i = 0; i < m; ++i)                                // rows ascending => edges of a column in ascending check index
        for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
            const int j = col_idx[e];
            col_edge[col_ptr[j] + fill[j]++] = e;
        }
    h->max_row_deg = maxr; h->max_col_deg = maxc;
    h->host_row_ptr.assign(row_ptr, row_ptr + m + 1);
    h->host_col_idx.assign(col_idx, col_idx + nnz);
    cudaError_t e = cudaMalloc(&h->row_ptr, sizeof(int32_t) * (m + 1));
    if (e == cudaSuccess) e = cudaMalloc(&h->col_idx, sizeof(int32_t) * nnz);
    if (e == cudaSuccess) e = cudaMalloc(&h->col_ptr, sizeof(int32_t) * (n + 1));
    if (e == cudaSuccess) e = cudaMalloc(&h->col_edge, sizeof(int32_t) * nnz);
    if (e == cudaSuccess) e = cudaMemcpy(h->row_ptr, row_ptr, sizeof(int32_t) * (m + 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(h->col_idx, col_idx, sizeof(int32_t) * nnz, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(h->col_ptr, col_ptr.data(), sizeof(int32_t) * (n + 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(h->col_edge, col_edge.data(), sizeof(int32_t) * nnz, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        record_cuda_error(e, "ldpc handle upload", __FILE__, __LINE__);
        cpb_ldpc_destroy(h);
        return CPB_ECUDA;
    }
    *out = h;
    return CPB_OK;
}

int cpb_ldpc_destroy(cpbLdpc *h)
{
    if (!h) return CPB_OK;
    if (h->row_ptr) cudaFree(h->row_ptr);
    if (h->col_idx) cudaFree(h->col_idx);
    if (h->col_ptr) cudaFree(h->col_ptr);
    if (h->col_edge) cudaFree(h->col_edge);
    delete h;
    return CPB_OK;
}

int cpb_ldpc_workspace_bytes(const cpbLdpc *h, int64_t batch, int precision, size_t *bytes)
{
    if (!h || !bytes || batch < 0) return CPB_EINVAL;
    if (precision == CPB_LDPC_FP64) *bytes = ldpc::ws_bytes<double>(h, ldpc::chunk_frames<double>(h, batch));
    else *bytes = ldpc::ws_bytes<float>(h, ldpc::chunk_frames<float>(h, batch));
    return CPB_OK;
}

static int ldpc_dispatch(const cpbLdpc *h, void *llr_dev, int precision, int64_t batch, int n_iters, int spa,
                         uint8_t *dec_dev, void *out_llr_dev, int32_t *iters_dev, void *workspace_dev,
                         size_t workspace_bytes, void *stream)
{
    if (h && batch == 0) return CPB_OK;
    if (!h || !llr_dev || !dec_dev || batch < 0 || n_iters < 0) return CPB_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    if (precision == CPB_LDPC_FP64)
        return ldpc::run<double>(h, reinterpret_cast<double *>(llr_dev), batch, n_iters, spa, dec_dev,
                                 reinterpret_cast<double *>(out_llr_dev), iters_dev, workspace_dev, workspace_bytes, st);
    if (precision == CPB_LDPC_FP32)
        return ldpc::run<float>(h, reinterpret_cast<float *>(llr_dev), batch, n_iters, spa, dec_dev,
                                reinterpret_cast<float *>(out_llr_dev), iters_dev, workspace_dev, workspace_bytes, st);
    return CPB_EINVAL;
}

int cpb_ldpc_minsum(const cpbLdpc *h, void *llr_dev, int precision, int64_t batch, int n_iters, uint8_t *dec_dev,
                    void *out_llr_dev, int32_t *iters_dev, void *workspace_dev, size_t workspace_bytes, void *stream)
{
    return ldpc_dispatch(h, llr_dev, precision, batch, n_iters, 0, dec_dev, out_llr_dev, iters_dev, workspace_dev,
                         workspace_bytes, stream);
}

int cpb_ldpc_sumproduct(const cpbLdpc *h, void *llr_dev, int precision, int64_t batch, int n_iters, uint8_t *dec_dev,
                        void *out_llr_dev, int32_t *iters_dev, void *workspace_dev, size_t workspace_bytes, void *stream)
{
    return ldpc_dispatch(h, llr_dev, precision, batch, n_iters, 1, dec_dev, out_llr_dev, iters_dev, workspace_dev,
                         workspace_bytes, stream);
}

}  // extern "C"

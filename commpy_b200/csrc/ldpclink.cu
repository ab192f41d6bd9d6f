// Systematic LDPC encoding from the parity-check matrix, and the transmit side of an LDPC-coded link generated on the
// device (SURVEY 8(f) row 3): what LinkModel.link_performance does per frame with an LDPC code on the host,
//     msg = randint(0, 2, send_chunk)                                  commpy/links.py:318
//     coded = triang_ldpc_systematic_encode(msg, params)               commpy/channelcoding/ldpc.py:302-354
//     symbols = modem.modulate(coded)                                  commpy/modulation.py:79-98 (MSB-first index)
//     y = h * symbols + noise                                          commpy/channels.py:176-221
// for a batch of frames at once.
//
// Code word layout (the reference's): c = [message (k = n - m bits) | parity (m bits)] with H c = 0 over GF(2).  With
// H = [H_s | H_p] (H_s the first k columns) the parity is p = H_p^-1 H_s msg.  The plan (built on the host from the
// CSR H, once per handle and form) takes one of two forms:
//   * peeled: H_p peels completely -- a row order r_0 .. r_{m-1} in which row r_t has exactly one parity bit, pivot_t,
//     not solved by an earlier row.  The device computes s_t = (H_s msg)[r_t] (sparse, parallel over steps and frames)
//     and then pivot_t = s_t ^ (the other parity bits of row r_t), in step order.  A staircase H_p (each row's only
//     other parity bit is the previous step's) makes this a prefix XOR carried in a register.
//   * dense: H_p invertible over GF(2) and k m <= 2^26 bits.  The host computes P = H_p^-1 H_s by Gauss-Jordan
//     elimination on bit-packed rows; parity bit i is the XOR of the message bits that row i of P selects.
// A singular H_p is CPB_EINVAL; a code that does not peel and exceeds the dense bound is CPB_EUNSUPPORTED.
// CPB_OPT_LDPC_ENC_FORCE_DENSE makes a peelable code that fits the bound use the dense form (the cross-check).
//
// Bit-slicing: every device array of the encoder holds 32 frames per uint32 word, [bit][W] with W = frames / 32
// words per bit (bit f of word w = frame 32 w + f), so one XOR processes 32 frames and every access of a warp is a
// contiguous run of words.  Algorithmic bytes per frame: k message bytes read (encode) or written (TX), k / 8 bytes of
// packed message written, then read once per edge of H_s (peeled: 4 E_s / 32 bytes per frame, mostly from L2), m / 8
// bytes of syndrome and of parity written and read, m parity bytes written.
//
// TX randomness is the conv link's (philox.cuh): message bits from counter word 0, symbol s's noise from word 1 and its
// flat-fading gain from word 5 (box_muller of the pair (x, y) for even s, (z, w) for odd s of counter s / 2), drawn by the
// shared code-word modulator (codeword_tx.cu).
#include <algorithm>
#include <cmath>
#include <deque>
#include <vector>

#include "codeword_tx.cuh"
#include "common.cuh"
#include "handles.cuh"
#include "philox.cuh"

using namespace cpb;

struct cpbModem;
void cpb_modem_info(const cpbModem *m, int *M, int *nb, const float **cst_dev);

namespace cpb {

enum { ENC_PEELED = 0, ENC_DENSE = 1 };
constexpr int64_t DENSE_MAX_BITS = (int64_t)1 << 26;     // k m of the dense form's P
constexpr int64_t CHUNK_FRAMES = 8192;                   // frames per pass: bounds the scratch (a multiple of 32)

struct LdpcEncPlan {
    int form, m, n, k;
    // peeled: step t solves parity bit steps[t].x from row order[t]; its other parity bits are the previous step's
    // (steps[t].w = 1) and dep[steps[t].y .. steps[t].z); hs_ptr / hs_col: the message columns of row order[t]
    int4 *steps = nullptr;
    int32_t *dep = nullptr, *hs_ptr = nullptr, *hs_col = nullptr;
    // dense: P bit-packed, m rows of kw words (bit j of row i = word j / 32, bit j % 32)
    uint32_t *P = nullptr;
    int kw = 0;
    void *dev = nullptr;                                 // one device allocation holding the arrays above
};

LdpcEncCache::~LdpcEncCache()
{
    for (LdpcEncPlan *p : plan)
        if (p) {
            if (p->dev) cudaFree(p->dev);
            delete p;
        }
}

}  // namespace cpb

namespace ldpclink {

// ---- host: the plan -----------------------------------------------------------------------------------------------
struct HostPlan {
    int form = ENC_PEELED;
    std::vector<int32_t> order, pivot;                   // peeled: row and parity bit of each step
    std::vector<uint32_t> P;                             // dense: m x kw words
    int kw = 0;
};

// Peeling: rows whose parity part has one unsolved bit are queued in ascending row order (FIFO); popping one solves that
// bit, which may leave other rows with one unsolved bit.  True when all m parity bits were solved.
static bool peel(const int32_t *row_ptr, const int32_t *col_idx, int m, int k, HostPlan &hp)
{
    std::vector<int32_t> cnt(m, 0), pcol_ptr(m + 1, 0), pcol_row;
    for (int i = 0; i < m; ++i)
        for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e)
            if (col_idx[e] >= k) { ++cnt[i]; ++pcol_ptr[col_idx[e] - k + 1]; }
    for (int j = 0; j < m; ++j) pcol_ptr[j + 1] += pcol_ptr[j];
    pcol_row.resize(pcol_ptr[m]);
    std::vector<int32_t> fill(pcol_ptr.begin(), pcol_ptr.end() - 1);
    for (int i = 0; i < m; ++i)
        for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e)
            if (col_idx[e] >= k) pcol_row[fill[col_idx[e] - k]++] = i;
    std::vector<char> solved(m, 0), used(m, 0);
    std::deque<int32_t> q;
    for (int i = 0; i < m; ++i)
        if (cnt[i] == 1) q.push_back(i);
    hp.order.clear(); hp.pivot.clear();
    while (!q.empty()) {
        const int i = q.front();
        q.pop_front();
        if (used[i] || cnt[i] != 1) continue;
        int j = -1;
        for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e)
            if (col_idx[e] >= k && !solved[col_idx[e] - k]) j = col_idx[e] - k;
        used[i] = 1; solved[j] = 1;
        hp.order.push_back(i); hp.pivot.push_back(j);
        for (int e = pcol_ptr[j]; e < pcol_ptr[j + 1]; ++e)
            if (--cnt[pcol_row[e]] == 1 && !used[pcol_row[e]]) q.push_back(pcol_row[e]);
    }
    return (int)hp.order.size() == m;
}

// Gauss-Jordan elimination of [H_p | H_s] over GF(2) on 64-bit words: [I | P] when H_p is invertible.
static int dense(const int32_t *row_ptr, const int32_t *col_idx, int m, int k, HostPlan &hp)
{
    const int64_t words = (m + (int64_t)k + 63) / 64;
    std::vector<uint64_t> A((size_t)m * words, 0);
    for (int i = 0; i < m; ++i)
        for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
            const int c = col_idx[e];
            const int64_t b = c >= k ? c - k : m + (int64_t)c;     // parity part first, then the message part
            A[(size_t)i * words + b / 64] ^= 1ull << (b % 64);
        }
    for (int c = 0; c < m; ++c) {
        const int64_t cw = c / 64;
        const uint64_t bit = 1ull << (c % 64);
        int r = c;
        while (r < m && !(A[(size_t)r * words + cw] & bit)) ++r;
        if (r == m) return CPB_EINVAL;                                  // H_p singular over GF(2)
        if (r != c)
            std::swap_ranges(A.begin() + (size_t)r * words, A.begin() + (size_t)(r + 1) * words, A.begin() + (size_t)c * words);
        const uint64_t *pc = &A[(size_t)c * words];
        for (int i = 0; i < m; ++i) {
            if (i == c || !(A[(size_t)i * words + cw] & bit)) continue;
            uint64_t *pi = &A[(size_t)i * words];
            for (int64_t w = cw; w < words; ++w) pi[w] ^= pc[w];
        }
    }
    hp.form = ENC_DENSE;
    hp.kw = (k + 31) / 32;
    hp.P.assign((size_t)m * hp.kw, 0u);
    for (int i = 0; i < m; ++i)
        for (int j = 0; j < k; ++j) {
            const int64_t b = m + (int64_t)j;
            if ((A[(size_t)i * words + b / 64] >> (b % 64)) & 1ull) hp.P[(size_t)i * hp.kw + j / 32] |= 1u << (j % 32);
        }
    hp.order.resize(m); hp.pivot.resize(m);
    for (int i = 0; i < m; ++i) hp.order[i] = hp.pivot[i] = i;
    return CPB_OK;
}

static int build_host_plan(const int32_t *row_ptr, const int32_t *col_idx, int m, int n, bool force_dense, HostPlan &hp)
{
    const int k = n - m;
    if (k < 1) return CPB_EINVAL;
    const bool fits = (int64_t)k * m <= DENSE_MAX_BITS;
    if (!(force_dense && fits) && peel(row_ptr, col_idx, m, k, hp)) {
        hp.form = ENC_PEELED;
        return CPB_OK;
    }
    if (!fits) return CPB_EUNSUPPORTED;
    return dense(row_ptr, col_idx, m, k, hp);
}

static int upload(const cpbLdpc *h, const HostPlan &hp, LdpcEncPlan *p)
{
    const int m = h->m, k = h->n - h->m;
    const int32_t *row_ptr = h->host_row_ptr.data(), *col_idx = h->host_col_idx.data();
    p->form = hp.form; p->m = m; p->n = h->n; p->k = k;
    std::vector<int4> steps;
    std::vector<int32_t> dep, hs_ptr, hs_col;
    if (hp.form == ENC_PEELED) {
        steps.resize(m);
        hs_ptr.assign(1, 0);
        for (int t = 0; t < m; ++t) {
            const int i = hp.order[t];
            int4 s = make_int4(hp.pivot[t], (int)dep.size(), 0, 0);
            for (int e = row_ptr[i]; e < row_ptr[i + 1]; ++e) {
                const int c = col_idx[e];
                if (c < k) hs_col.push_back(c);
                else if (c - k == hp.pivot[t]) continue;
                else if (t > 0 && c - k == hp.pivot[t - 1]) s.w = 1;
                else dep.push_back(c - k);
            }
            s.z = (int)dep.size();
            steps[t] = s;
            hs_ptr.push_back((int32_t)hs_col.size());
        }
    }
    const size_t b_steps = steps.size() * sizeof(int4), b_dep = dep.size() * 4, b_ptr = hs_ptr.size() * 4,
                 b_col = hs_col.size() * 4, b_P = hp.P.size() * 4;
    const size_t total = b_steps + b_dep + b_ptr + b_col + b_P + 64;
    CPB_CUDA(cudaMalloc(&p->dev, total));
    char *at = reinterpret_cast<char *>(p->dev);
    cudaError_t e = cudaSuccess;
    const void *srcs[5] = {steps.data(), dep.data(), hs_ptr.data(), hs_col.data(), hp.P.data()};
    const size_t sizes[5] = {b_steps, b_dep, b_ptr, b_col, b_P};
    char *dst[5];
    for (int a = 0; a < 5; ++a) {
        dst[a] = at;
        if (sizes[a] && e == cudaSuccess) e = cudaMemcpy(at, srcs[a], sizes[a], cudaMemcpyHostToDevice);
        at += (sizes[a] + 15) & ~(size_t)15;
    }
    if (e != cudaSuccess) return record_cuda_error(e, "ldpc encoder plan upload", __FILE__, __LINE__);
    p->steps = reinterpret_cast<int4 *>(dst[0]);
    p->dep = reinterpret_cast<int32_t *>(dst[1]);
    p->hs_ptr = reinterpret_cast<int32_t *>(dst[2]);
    p->hs_col = reinterpret_cast<int32_t *>(dst[3]);
    p->P = reinterpret_cast<uint32_t *>(dst[4]);
    p->kw = hp.kw;
    return CPB_OK;
}

// the handle's plan of the form the option selects (the dense one when forced and the code fits the bound)
static int get_plan(const cpbLdpc *hc, const LdpcEncPlan **out)
{
    cpbLdpc *h = const_cast<cpbLdpc *>(hc);
    const int k = h->n - h->m;
    const bool dense_wanted = option(CPB_OPT_LDPC_ENC_FORCE_DENSE) && k >= 1 && (int64_t)k * h->m <= DENSE_MAX_BITS;
    const int slot = dense_wanted ? 1 : 0;
    std::lock_guard<std::mutex> lock(h->enc.mu);
    if (h->enc.status[slot] < 0) {
        HostPlan hp;
        int rc = build_host_plan(h->host_row_ptr.data(), h->host_col_idx.data(), h->m, h->n, dense_wanted, hp);
        if (rc == CPB_OK) {
            LdpcEncPlan *p = new LdpcEncPlan();
            rc = upload(h, hp, p);
            if (rc != CPB_OK) {
                if (p->dev) cudaFree(p->dev);
                delete p;
                return rc;                                   // a CUDA failure is not cached
            }
            h->enc.plan[slot] = p;
        }
        h->enc.status[slot] = rc;
    }
    *out = h->enc.plan[slot];
    return h->enc.status[slot];
}

// ---- device: encoder ----------------------------------------------------------------------------------------------
// Packs message bits [32 q, 32 q + 32) of the 32 frames of word w into M[bit][W] (one warp per (w, q)).  GEN: the bits
// are Philox counter word 0 of each frame and are also written to msg as bytes; otherwise they are read from msg
// (a nonzero byte is a 1).
template <bool GEN>
__global__ void __launch_bounds__(256) pack_kernel(uint8_t *__restrict__ msg, int64_t frames, int k, int64_t W, int64_t nq,
                                                   int64_t first_frame, uint32_t seed_lo, uint32_t seed_hi,
                                                   uint32_t *__restrict__ M)
{
    const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= W * nq) return;                                // warp-uniform
    const int64_t w = warp / nq, q = warp - w * nq;
    const int64_t f = w * 32 + lane;
    const bool valid = f < frames;
    const int j0 = (int)(q * 32);
    const int nj = min(32, k - j0);
    uint8_t *row = msg + f * k + j0;
    uint32_t bits = 0;
    if (valid) {
        if (GEN) {
            const uint64_t fg = (uint64_t)(first_frame + f);
            const uint4 r = philox4x32_10(make_uint4((uint32_t)fg, (uint32_t)(fg >> 32), (uint32_t)(q >> 2), 0u), seed_lo, seed_hi);
            const uint32_t c = q & 3;
            bits = (c == 0) ? r.x : (c == 1) ? r.y : (c == 2) ? r.z : r.w;
            if (nj < 32) bits &= (1u << nj) - 1u;
            for (int j = 0; j < nj; ++j) row[j] = (uint8_t)((bits >> j) & 1u);
        } else {
            for (int j = 0; j < nj; ++j) bits |= (row[j] != 0 ? 1u : 0u) << j;
        }
    }
    uint32_t mine = 0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const uint32_t b = __ballot_sync(0xffffffffu, (bits >> j) & 1u);
        if (lane == j) mine = b;
    }
    if (lane < nj) M[(int64_t)(j0 + lane) * W + w] = mine;
}

// peeled, first half: S[t][w] = XOR of the message bits of row order[t] (its H_s part)
__global__ void __launch_bounds__(256) peel_syndrome_kernel(const int32_t *__restrict__ hs_ptr, const int32_t *__restrict__ hs_col,
                                                            int m, int64_t W, const uint32_t *__restrict__ M,
                                                            uint32_t *__restrict__ S)
{
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)m * W) return;
    const int t = (int)(gid / W);
    const int64_t w = gid - (int64_t)t * W;
    uint32_t v = 0;
    const int e1 = __ldg(&hs_ptr[t + 1]);
    for (int e = __ldg(&hs_ptr[t]); e < e1; ++e) v ^= __ldg(&M[(int64_t)__ldg(&hs_col[e]) * W + w]);
    S[gid] = v;
}

// peeled, second half: the steps in order, one thread per word of 32 frames; the previous step's bit stays in a register
// (a staircase needs nothing else), any other parity bit is read back from P, which this thread wrote earlier
__global__ void __launch_bounds__(128) peel_solve_kernel(const int4 *__restrict__ steps, const int32_t *__restrict__ dep, int m,
                                                         int64_t W, const uint32_t *__restrict__ S, uint32_t *P)
{
    const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= W) return;
    uint32_t last = 0;
#pragma unroll 4
    for (int t = 0; t < m; ++t) {
        const int4 s = __ldg(&steps[t]);
        uint32_t v = __ldg(&S[(int64_t)t * W + w]);
        if (s.w) v ^= last;
        for (int e = s.y; e < s.z; ++e) v ^= P[(int64_t)__ldg(&dep[e]) * W + w];
        P[(int64_t)s.x * W + w] = v;
        last = v;
    }
}

// dense: P_out[i][w] = XOR over the set bits j of row i of P of M[j][w]
__global__ void __launch_bounds__(256) dense_parity_kernel(const uint32_t *__restrict__ P, int kw, int m, int64_t W,
                                                           const uint32_t *__restrict__ M, uint32_t *__restrict__ out)
{
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= (int64_t)m * W) return;
    const int i = (int)(gid / W);
    const int64_t w = gid - (int64_t)i * W;
    uint32_t v = 0;
    for (int q = 0; q < kw; ++q) {
        uint32_t bits = __ldg(&P[(int64_t)i * kw + q]);
        while (bits) {
            const int j = __ffs(bits) - 1;
            bits &= bits - 1u;
            v ^= __ldg(&M[(int64_t)(q * 32 + j) * W + w]);
        }
    }
    out[gid] = v;
}

// parity words [m][W] -> bytes dst[f * ld + i]; a 32 x 8 block moves 32 parity bits of the 32 frames of word w
__global__ void __launch_bounds__(256) unpack_parity_kernel(const uint32_t *__restrict__ Pw, int m, int64_t W, int64_t frames,
                                                            uint8_t *__restrict__ dst, int64_t ld)
{
    __shared__ uint32_t s[32];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int i = blockIdx.x * 32 + tx;
    const int64_t w = blockIdx.y;
    if (ty == 0) s[tx] = (i < m) ? Pw[(int64_t)i * W + w] : 0u;
    __syncthreads();
    if (i >= m) return;
    for (int r = ty; r < 32; r += 8) {
        const int64_t f = w * 32 + r;
        if (f < frames) dst[f * ld + i] = (uint8_t)((s[tx] >> r) & 1u);
    }
}

// ---- host: launches -----------------------------------------------------------------------------------------------
static unsigned blocks(int64_t threads, int per) { return (unsigned)ceil_div(threads, per); }

// parity of `frames` (<= CHUNK_FRAMES) frames whose packed message is M: into Pw ([m][W] words); S is the peeled form's
// syndrome scratch
static void encode_words(const LdpcEncPlan *p, int64_t W, const uint32_t *M, uint32_t *S, uint32_t *Pw, cudaStream_t st)
{
    if (p->form == ENC_PEELED) {
        peel_syndrome_kernel<<<blocks((int64_t)p->m * W, 256), 256, 0, st>>>(p->hs_ptr, p->hs_col, p->m, W, M, S);
        peel_solve_kernel<<<blocks(W, 128), 128, 0, st>>>(p->steps, p->dep, p->m, W, S, Pw);
    } else {
        dense_parity_kernel<<<blocks((int64_t)p->m * W, 256), 256, 0, st>>>(p->P, p->kw, p->m, W, M, Pw);
    }
}

static size_t scratch_words(const LdpcEncPlan *p, int64_t W) { return (size_t)W * ((size_t)p->k + 2 * (size_t)p->m); }

// h_dev == nullptr: AWGN
static int link_tx(const cpbLdpc *h, const cpbModem *md, int64_t frames, uint64_t seed, int64_t first_frame, float sigma,
                   uint8_t *msg_dev, float *y_dev, float *h_dev, float mean_re, float mean_im, float nlos, void *stream)
{
    if (!h || !md || frames < 0 || first_frame < 0) return CPB_EINVAL;
    if (h_dev && !(nlos >= 0.0f && std::isfinite(nlos) && std::isfinite(mean_re) && std::isfinite(mean_im))) return CPB_EINVAL;
    int Mc, nb;
    const float *cst;
    cpb_modem_info(md, &Mc, &nb, &cst);
    if (nb < 1 || nb > 16 || h->n % nb) return CPB_EINVAL;           // the code word must fill whole symbols
    if (frames == 0) return CPB_OK;
    if (!msg_dev || !y_dev) return CPB_EINVAL;
    const LdpcEncPlan *p;
    int rc = get_plan(h, &p);
    if (rc) return rc;
    const int64_t Fc = std::min<int64_t>(CHUNK_FRAMES, ceil_div(frames, 32) * 32), Wc = Fc / 32;
    const size_t words = scratch_words(p, Wc);
    Scratch ws;
    cudaStream_t st = (cudaStream_t)stream;
    rc = ws.acquire(nullptr, 0, words * 4 + (size_t)Fc * p->m, st);
    if (rc) return rc;
    uint32_t *M = reinterpret_cast<uint32_t *>(ws.ptr), *S = M + (size_t)Wc * p->k, *Pw = S + (size_t)Wc * p->m;
    uint8_t *par = reinterpret_cast<uint8_t *>(Pw + (size_t)Wc * p->m);
    cwtx::TxParams tp;
    memset(&tp, 0, sizeof(tp));
    tp.nsym = h->n / nb; tp.npairs = (tp.nsym + 1) / 2;
    tp.k = p->k; tp.m = p->m; tp.nb = nb;
    tp.seed_lo = (uint32_t)seed; tp.seed_hi = (uint32_t)(seed >> 32);
    tp.sigma = sigma;
    tp.mean_re = mean_re; tp.mean_im = mean_im; tp.nlos_std = (float)std::sqrt(0.5 * (double)nlos);
    tp.cst = reinterpret_cast<const float2 *>(cst);
    tp.par = par;
    const int64_t nq = ceil_div(p->k, 32);
    for (int64_t f0 = 0; f0 < frames; f0 += Fc) {
        const int64_t nf = std::min(Fc, frames - f0), W = ceil_div(nf, 32);
        uint8_t *msg = msg_dev + f0 * p->k;
        pack_kernel<true><<<blocks(W * nq * 32, 256), 256, 0, st>>>(msg, nf, p->k, W, nq, first_frame + f0, tp.seed_lo,
                                                                     tp.seed_hi, M);
        encode_words(p, W, M, S, Pw, st);
        unpack_parity_kernel<<<dim3((unsigned)ceil_div(p->m, 32), (unsigned)W), 256, 0, st>>>(Pw, p->m, W, nf, par, p->m);
        tp.frames = nf; tp.first_frame = first_frame + f0;
        tp.msg = msg;
        tp.y = reinterpret_cast<float2 *>(y_dev) + f0 * tp.nsym;
        tp.h = h_dev ? reinterpret_cast<float2 *>(h_dev) + f0 * tp.nsym : nullptr;
        cwtx::launch_modulate(tp, h_dev != nullptr, st);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { ws.release(); return record_cuda_error(e, "ldpc link tx kernels", __FILE__, __LINE__); }
    }
    ws.release();
    return CPB_OK;
}

}  // namespace ldpclink

extern "C" {

int cpb_ldpc_encoder_plan(const int32_t *row_ptr, const int32_t *col_idx, int m, int n, int force_dense, int *form,
                          int32_t *order_host, int32_t *pivot_host, uint32_t *P_host)
{
    if (!row_ptr || !col_idx || !form || m < 1 || n <= m || row_ptr[0] != 0) return CPB_EINVAL;
    for (int i = 0; i < m; ++i)
        if (row_ptr[i + 1] < row_ptr[i]) return CPB_EINVAL;
    for (int e = 0; e < row_ptr[m]; ++e)
        if (col_idx[e] < 0 || col_idx[e] >= n) return CPB_EINVAL;
    ldpclink::HostPlan hp;
    const int rc = ldpclink::build_host_plan(row_ptr, col_idx, m, n, force_dense != 0, hp);
    if (rc) return rc;
    *form = hp.form;
    if (order_host) std::copy(hp.order.begin(), hp.order.end(), order_host);
    if (pivot_host) std::copy(hp.pivot.begin(), hp.pivot.end(), pivot_host);
    if (P_host && hp.form == cpb::ENC_DENSE) std::copy(hp.P.begin(), hp.P.end(), P_host);
    return CPB_OK;
}

int cpb_ldpc_encode(const cpbLdpc *h, const uint8_t *msg_dev, int64_t batch, uint8_t *cw_dev, void *stream)
{
    using namespace ldpclink;
    if (!h || batch < 0) return CPB_EINVAL;
    if (batch == 0) return CPB_OK;
    if (!msg_dev || !cw_dev) return CPB_EINVAL;
    const LdpcEncPlan *p;
    int rc = get_plan(h, &p);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t Fc = std::min<int64_t>(CHUNK_FRAMES, ceil_div(batch, 32) * 32), Wc = Fc / 32;
    Scratch ws;
    rc = ws.acquire(nullptr, 0, scratch_words(p, Wc) * 4, st);
    if (rc) return rc;
    uint32_t *M = reinterpret_cast<uint32_t *>(ws.ptr), *S = M + (size_t)Wc * p->k, *Pw = S + (size_t)Wc * p->m;
    const int64_t nq = ceil_div(p->k, 32);
    cudaError_t e = cudaMemcpy2DAsync(cw_dev, (size_t)p->n, msg_dev, (size_t)p->k, (size_t)p->k, (size_t)batch,
                                      cudaMemcpyDeviceToDevice, st);
    for (int64_t f0 = 0; f0 < batch && e == cudaSuccess; f0 += Fc) {
        const int64_t nf = std::min(Fc, batch - f0), W = ceil_div(nf, 32);
        pack_kernel<false><<<blocks(W * nq * 32, 256), 256, 0, st>>>(const_cast<uint8_t *>(msg_dev) + f0 * p->k, nf, p->k, W,
                                                                      nq, 0, 0u, 0u, M);
        encode_words(p, W, M, S, Pw, st);
        unpack_parity_kernel<<<dim3((unsigned)ceil_div(p->m, 32), (unsigned)W), 256, 0, st>>>(Pw, p->m, W, nf,
                                                                                             cw_dev + f0 * p->n + p->k, p->n);
        e = cudaGetLastError();
    }
    ws.release();
    if (e != cudaSuccess) return record_cuda_error(e, "ldpc encode", __FILE__, __LINE__);
    return CPB_OK;
}

int cpb_ldpc_link_tx(const cpbLdpc *h, const cpbModem *modem, int64_t frames, uint64_t seed, int64_t first_frame,
                     float noise_sigma, uint8_t *msg_dev, float *y_dev, void *stream)
{
    return ldpclink::link_tx(h, modem, frames, seed, first_frame, noise_sigma, msg_dev, y_dev, nullptr, 0.0f, 0.0f, 0.0f,
                             stream);
}

int cpb_ldpc_link_tx_fading(const cpbLdpc *h, const cpbModem *modem, int64_t frames, uint64_t seed, int64_t first_frame,
                            float noise_sigma, float mean_re, float mean_im, float nlos, uint8_t *msg_dev, float *y_dev,
                            float *h_dev, void *stream)
{
    if (!h_dev && frames > 0) return CPB_EINVAL;
    return ldpclink::link_tx(h, modem, frames, seed, first_frame, noise_sigma, msg_dev, y_dev, h_dev, mean_re, mean_im,
                             nlos, stream);
}

}  // extern "C"

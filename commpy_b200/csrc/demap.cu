// PSK/QAM demapper on sm_90a -- replaces the triple loop of commpy/modulation.py:127-137
// (Modem.demodulate, 'soft') and the argmin of :121-123 ('hard').
//
//   LLR(bit b) = log sum_{k: bit b of k = 1} exp(-|y-c_k|^2/nv) - log sum_{k: bit b = 0} exp(-|y-c_k|^2/nv)
//
// exact log-sum-exp (not max-log), written MSB first per symbol, positive favours bit 1.  The reference sums
// raw exponentials and so returns +-inf/NaN once they underflow; here the smallest exponent is subtracted
// first, which is the same number wherever the reference is finite.
//
// Two kernels, one thread per symbol (coalesced 8-byte loads, 16-byte LLR stores; the separable kernel reads its
// axis levels as constant-bank operands, the general one from a shared-memory copy of the constellation):
//   demod_soft_separable  Gray-labelled square QAM, c[k] = pamI[k_hi] + j*pamQ[k_lo] (modulation.py:242-262
//                         + the Gray reorder of :68-77): the sums factor per axis, 2*sqrt(M) exponentials
//                         instead of M*log2(M) (32 instead of 2048 at 256-QAM).
//   demod_soft_general    any constellation (PSK, custom Modem): M exponentials per symbol from a
//                         shared-memory copy of the constellation.
#include <cmath>
#include <vector>

#include "common.cuh"
#include "handles.cuh"

using namespace cpb;

struct cpbModem {
    cpb::PipeCtx pipe;             // host-buffer pipeline of cpb_demod_*_host calls made with this handle
    int M, nb;
    float2 *cst_dev = nullptr;     // M points
    int separable = 0;
    int r = 0;                     // sqrt(M) when separable
    float pam_i[64], pam_q[64];    // axis levels indexed by k_hi / k_lo
};

namespace demap {

constexpr float LOG2E = 1.4426950408889634f;
constexpr float LN2 = 0.6931471805599453f;

struct SepTables {
    float pi[64];
    float pq[64];
};

// log2 of a group sum is off + log2(sum).  Sums are accumulated relative to the GLOBAL nearest point (off = -dmin);
// when a whole group lies more than ~100 octaves further away its fp32 sum underflows, and only then it is
// re-accumulated relative to the group's own nearest point (rare: |LLR| > 69).
constexpr float TINY = 7.8886e-31f;     // 2^-100

// raw MUFU.EX2 (ex2a() adds range handling for denormal results that the sums below do not need)
__device__ __forceinline__ float ex2a(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// one axis of a separable constellation: R levels, HB = log2(R) bits; out[h] = LLR of axis bit h (LSB = 0).
// lev[i] is the level of axis label i.  Per level: y - lev, square, one FMA against the nearest level's distance,
// one MUFU.EX2.  The 2*HB group sums share a binary tree over the label bits (R-2 + 2(R-HB-1) adds instead of
// HB*R): s_l[j] = sum of the 2^l labels j*2^l .. (j+1)*2^l-1, and bit h splits level h into odd / even j.
template <int HB>
__device__ __forceinline__ void axis_llr(float y, const float (&lev)[64], float inv_nv_log2e, float (&out)[HB])
{
    constexpr int R = 1 << HB;
    float tt[R];
    float tmin = 3.0e38f;
#pragma unroll
    for (int i = 0; i < R; ++i) {
        const float t = y - lev[i];
        tt[i] = t * t;
        tmin = fminf(tmin, tt[i]);
    }
    const float dmin = tmin * inv_nv_log2e;
    float s[R];                                     // in-place tree: after level l, s[j << l] holds s_l[j]
#pragma unroll
    for (int i = 0; i < R; ++i) s[i] = ex2a(fmaf(tt[i], -inv_nv_log2e, dmin));
    float num[HB], den[HB];
#pragma unroll
    for (int h = 0; h < HB; ++h) {
        const int step = 1 << h;                    // entries of level h sit at multiples of step
        float n = s[step], d = s[0];
#pragma unroll
        for (int j = 2; j < (R >> h); j += 2) { d += s[j * step]; n += s[(j + 1) * step]; }
        num[h] = n; den[h] = d;
        if (h + 1 < HB) {
#pragma unroll
            for (int j = 0; j < (R >> h); j += 2) s[j * step] += s[(j + 1) * step];
        }
    }
#pragma unroll
    for (int h = 0; h < HB; ++h) {
        float l1 = __log2f(num[h]), l0 = __log2f(den[h]);
        if (fminf(num[h], den[h]) < TINY) {
            // a whole group underflowed against the global nearest level: redo it against its own nearest level
#pragma unroll
            for (int g = 0; g < 2; ++g) {
                if ((g ? num[h] : den[h]) >= TINY) continue;
                float tg = 3.0e38f, sg = 0.0f;
#pragma unroll
                for (int i = 0; i < R; ++i)
                    if (((i >> h) & 1) == g) tg = fminf(tg, tt[i]);
                const float dg = tg * inv_nv_log2e;
#pragma unroll
                for (int i = 0; i < R; ++i)
                    if (((i >> h) & 1) == g) sg += ex2a(fmaf(tt[i], -inv_nv_log2e, dg));
                const float l = (dmin - dg) + __log2f(sg);
                if (g) l1 = l; else l0 = l;
            }
        }
        out[h] = (l1 - l0) * LN2;
    }
}

template <int HB>
__global__ void __launch_bounds__(256) demod_soft_separable(const float2 *__restrict__ y, int64_t nsym,
                                                            const SepTables tab, float inv_nv_log2e,
                                                            float *__restrict__ llr)
{
    // the levels are read straight from the kernel parameters (constant bank operands of the FADDs)
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nsym) return;
    const float2 v = __ldg(&y[i]);
    float li[HB], lq[HB];
    axis_llr<HB>(v.x, tab.pi, inv_nv_log2e, li);     // high half of the index bits
    axis_llr<HB>(v.y, tab.pq, inv_nv_log2e, lq);     // low half
    // output position nb-1-b for bit b (modulation.py:137): MSB first = axis I bits (high) then axis Q bits
    float o[2 * HB];
#pragma unroll
    for (int h = 0; h < HB; ++h) {
        o[HB - 1 - h] = li[h];
        o[2 * HB - 1 - h] = lq[h];
    }
    float *dst = llr + i * (2 * HB);
    if ((2 * HB) % 4 == 0) {
#pragma unroll
        for (int j = 0; j < 2 * HB; j += 4)
            *reinterpret_cast<float4 *>(dst + j) = make_float4(o[j], o[j + 1], o[j + 2], o[j + 3]);
    } else {
#pragma unroll
        for (int j = 0; j < 2 * HB; j += 2) *reinterpret_cast<float2 *>(dst + j) = make_float2(o[j], o[j + 1]);
    }
}

template <int NB>
__global__ void __launch_bounds__(256) demod_soft_general(const float2 *__restrict__ y, int64_t nsym,
                                                          const float2 *__restrict__ cst, int M, float inv_nv_log2e,
                                                          float *__restrict__ llr)
{
    extern __shared__ float2 sc[];
    for (int k = threadIdx.x; k < M; k += blockDim.x) sc[k] = cst[k];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nsym) return;
    const float2 v = __ldg(&y[i]);
    float dmin = 3.0e38f;
    for (int k = 0; k < M; ++k) {
        const float a = v.x - sc[k].x, b = v.y - sc[k].y;
        dmin = fminf(dmin, (a * a + b * b) * inv_nv_log2e);
    }
    float num[NB], den[NB];
#pragma unroll
    for (int b = 0; b < NB; ++b) { num[b] = 0.0f; den[b] = 0.0f; }
    for (int k = 0; k < M; ++k) {
        const float a = v.x - sc[k].x, b2 = v.y - sc[k].y;
        const float e = ex2a(dmin - (a * a + b2 * b2) * inv_nv_log2e);
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            if ((k >> b) & 1) num[b] += e; else den[b] += e;
        }
    }
    float *dst = llr + i * NB;
#pragma unroll
    for (int b = 0; b < NB; ++b) {
        float l1 = __log2f(num[b]), l0 = __log2f(den[b]);
        if (fminf(num[b], den[b]) < TINY) {          // a whole group underflowed: redo it against its own nearest point
            for (int g = 0; g < 2; ++g) {
                if ((g ? num[b] : den[b]) >= TINY) continue;
                float dg = 3.0e38f, sg = 0.0f;
                for (int k = 0; k < M; ++k)
                    if (((k >> b) & 1) == g) {
                        const float a = v.x - sc[k].x, b2 = v.y - sc[k].y;
                        dg = fminf(dg, (a * a + b2 * b2) * inv_nv_log2e);
                    }
                for (int k = 0; k < M; ++k)
                    if (((k >> b) & 1) == g) {
                        const float a = v.x - sc[k].x, b2 = v.y - sc[k].y;
                        sg += ex2a(dg - (a * a + b2 * b2) * inv_nv_log2e);
                    }
                const float l = (dmin - dg) + __log2f(sg);
                if (g) l1 = l; else l0 = l;
            }
        }
        dst[NB - 1 - b] = (l1 - l0) * LN2;
    }
}

__global__ void __launch_bounds__(256) demod_hard_kernel(const float2 *__restrict__ y, int64_t nsym,
                                                         const float2 *__restrict__ cst, int M, int nb,
                                                         uint8_t *__restrict__ bits)
{
    extern __shared__ float2 sc[];
    for (int k = threadIdx.x; k < M; k += blockDim.x) sc[k] = cst[k];
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nsym) return;
    const float2 v = __ldg(&y[i]);
    float best = 3.0e38f;
    int arg = 0;
    for (int k = 0; k < M; ++k) {            // first minimum (argmin, modulation.py:122)
        const float a = v.x - sc[k].x, b = v.y - sc[k].y;
        const float d = a * a + b * b;
        if (d < best) { best = d; arg = k; }
    }
    uint8_t *dst = bits + i * nb;
    for (int b = 0; b < nb; ++b) dst[b] = (uint8_t)((arg >> (nb - 1 - b)) & 1);      // MSB first
}

}  // namespace demap

// accessor for the other translation units (not part of the C-ABI)
cpb::PipeCtx &cpb_modem_pipe(cpbModem *m) { return m->pipe; }

void cpb_modem_info(const cpbModem *m, int *M, int *nb, const float **cst_dev)
{
    *M = m->M; *nb = m->nb; *cst_dev = reinterpret_cast<const float *>(m->cst_dev);
}

extern "C" {

int cpb_modem_create(const double *constellation, int M, cpbModem **out)
{
    if (!constellation || !out || M < 2 || M > 4096) return CPB_EINVAL;
    int nb = 0;
    while ((1 << nb) < M) ++nb;
    if ((1 << nb) != M) return CPB_EINVAL;            // ValueError of modulation.py:163-164
    cpbModem *m = new cpbModem();
    m->M = M; m->nb = nb;
    std::vector<float2> c(M);
    for (int k = 0; k < M; ++k) c[k] = make_float2((float)constellation[2 * k], (float)constellation[2 * k + 1]);
    // separable: c[k_hi*r + k_lo] = pamI[k_hi] + j*pamQ[k_lo] with r = sqrt(M)
    if (nb % 2 == 0 && nb >= 2 && nb <= 12) {
        const int r = 1 << (nb / 2);
        bool ok = true;
        for (int hi = 0; hi < r && ok; ++hi)
            for (int lo = 0; lo < r && ok; ++lo) {
                const double re = constellation[2 * (hi * r + lo)], im = constellation[2 * (hi * r + lo) + 1];
                if (re != constellation[2 * (hi * r)] || im != constellation[2 * lo + 1]) ok = false;
            }
        if (ok) {
            m->separable = 1; m->r = r;
            for (int i = 0; i < r; ++i) {
                m->pam_i[i] = (float)constellation[2 * (i * r)];
                m->pam_q[i] = (float)constellation[2 * i + 1];
            }
        }
    }
    if (cudaMalloc(&m->cst_dev, sizeof(float2) * M) != cudaSuccess ||
        cudaMemcpy(m->cst_dev, c.data(), sizeof(float2) * M, cudaMemcpyHostToDevice) != cudaSuccess) {
        record_cuda_error(cudaGetLastError(), "modem constellation upload", __FILE__, __LINE__);
        cpb_modem_destroy(m);
        return CPB_ECUDA;
    }
    *out = m;
    return CPB_OK;
}

int cpb_modem_destroy(cpbModem *m)
{
    if (!m) return CPB_OK;
    if (m->cst_dev) cudaFree(m->cst_dev);
    delete m;
    return CPB_OK;
}

int cpb_modem_is_separable(const cpbModem *m) { return m ? m->separable : 0; }

int cpb_demod_soft(const cpbModem *m, const float *y_dev, int64_t n_sym, float noise_var, float *llr_dev, void *stream)
{
    if (m && n_sym == 0) return CPB_OK;            // nothing to do: empty tensors carry null pointers
    if (!m || !y_dev || !llr_dev || n_sym < 0) return CPB_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const float inv = demap::LOG2E / noise_var;
    const unsigned grid = (unsigned)ceil_div(n_sym, 256);
    const float2 *y = reinterpret_cast<const float2 *>(y_dev);
    if (m->separable && m->r <= 64) {
        demap::SepTables tab;
        memset(&tab, 0, sizeof(tab));
        for (int i = 0; i < m->r; ++i) { tab.pi[i] = m->pam_i[i]; tab.pq[i] = m->pam_q[i]; }
        switch (m->nb / 2) {
        case 1: demap::demod_soft_separable<1><<<grid, 256, 0, st>>>(y, n_sym, tab, inv, llr_dev); break;
        case 2: demap::demod_soft_separable<2><<<grid, 256, 0, st>>>(y, n_sym, tab, inv, llr_dev); break;
        case 3: demap::demod_soft_separable<3><<<grid, 256, 0, st>>>(y, n_sym, tab, inv, llr_dev); break;
        case 4: demap::demod_soft_separable<4><<<grid, 256, 0, st>>>(y, n_sym, tab, inv, llr_dev); break;
        case 5: demap::demod_soft_separable<5><<<grid, 256, 0, st>>>(y, n_sym, tab, inv, llr_dev); break;
        default: return CPB_EUNSUPPORTED;
        }
        CPB_LAUNCH_CHECK();
        return CPB_OK;
    }
    const size_t smem = sizeof(float2) * m->M;
#define CPB_GEN(NB) case NB: demap::demod_soft_general<NB><<<grid, 256, smem, st>>>(y, n_sym, m->cst_dev, m->M, inv, llr_dev); break;
    switch (m->nb) {
        CPB_GEN(1) CPB_GEN(2) CPB_GEN(3) CPB_GEN(4) CPB_GEN(5) CPB_GEN(6)
        CPB_GEN(7) CPB_GEN(8) CPB_GEN(9) CPB_GEN(10) CPB_GEN(11) CPB_GEN(12)
    default: return CPB_EUNSUPPORTED;
    }
#undef CPB_GEN
    CPB_LAUNCH_CHECK();
    return CPB_OK;
}

int cpb_demod_hard(const cpbModem *m, const float *y_dev, int64_t n_sym, uint8_t *bits_dev, void *stream)
{
    if (m && n_sym == 0) return CPB_OK;
    if (!m || !y_dev || !bits_dev || n_sym < 0) return CPB_EINVAL;
    const unsigned grid = (unsigned)ceil_div(n_sym, 256);
    demap::demod_hard_kernel<<<grid, 256, sizeof(float2) * m->M, (cudaStream_t)stream>>>(
        reinterpret_cast<const float2 *>(y_dev), n_sym, m->cst_dev, m->M, m->nb, bits_dev);
    CPB_LAUNCH_CHECK();
    return CPB_OK;
}

}  // extern "C"

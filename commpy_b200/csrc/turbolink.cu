// Transmit side of a turbo-coded BPSK-AWGN link, generated on the device -- SURVEY 8(f) row 4: what
// commpy/channelcoding/turbo.py:14-59 (turbo_encode) + a BPSK mapper + AWGN do per frame on the host, for a batch:
//     sys  = msg                                     (turbo.py:47-49: conv_encode(msg, trellis, 'rsc')[::2], tail cut :55)
//     par1 = parity stream of the component code over msg          (:50, :56)
//     par2 = parity stream of the component code over msg[p_array] (:52-54, :57)
//     y_x  = (2 x - 1) + sigma * N(0,1)              for x in (sys, par1, par2)
// The reference's termination='rsc' pads ZERO INPUT bits (convcode.py:505-527), which does not drive a recursive encoder
// back to state 0, and the tails are cut off again: the three streams are those of an unterminated encoder started in
// state 0 -- exactly what map_decode assumes (beta_N = 1 for every state, turbo.py:225-226).
//
// Randomness is counter based (Philox4x32-10, same keying as txlink.cu), so nothing depends on the batch split: the
// message, noise and gain streams are the counter words of philox.cuh.
//
// Flat fading (FADING = true, cpb_turbo_link_tx_fading; SISOFlatChannel, commpy/channels.py:176-221): each value
// x = 2 bit - 1 of each stream is received as y = h x + sigma (n_re + j n_im), n_re the AWGN link's noise and
// h = mean + sqrt(nlos / 2) (g.x + j g.y).  y_re = fmaf(sigma, n_re, h_re x), so the message and Re(y) at h = 1 + 0j are
// the AWGN link's bit for bit.
//
// Receiver (cpb_bpsk_combine): s = Re(conj(h) y) = |h|^2 x + N(0, sigma^2 |h|^2), whose exact LLR 2 s / sigma^2 is the
// channel term the MAP / turbo kernels form from a symbol s at noise variance sigma^2: the decoder takes s unchanged.
//
// With a modem (cpb_turbo_link_tx_modem[_fading]): the code word c = [sys | par1 | par2] (3N bits, the three streams above,
// sys = msg) is mapped MSB first by Modem.modulate's rule, with no channel interleaver.  msg_kernel draws the message,
// parity_kernel writes [par1 | par2] (frames x 2N bytes) and the shared code-word modulator (codeword_tx.cu, k = N,
// m = 2N) maps c and adds the conv link's noise (counter word 1) and gains (word 5), one draw per symbol pair.
#include <algorithm>
#include <cmath>
#include <vector>

#include "codeword_tx.cuh"
#include "common.cuh"
#include "philox.cuh"

using namespace cpb;

struct cpbTrellis;
void cpb_trellis_dims(const cpbTrellis *t, int *k, int *n, int *S);
void cpb_trellis_host_tables(const cpbTrellis *t, const int32_t **next, const int32_t **out);
struct cpbModem;
void cpb_modem_info(const cpbModem *m, int *M, int *nb, const float **cst_dev);

namespace turbolink {

struct Params {
    int64_t frames, N, first_frame;
    uint32_t seed_lo, seed_hi;
    float sigma;
    const int32_t *perm;
    uint32_t next_bits[2];    // next state of (s, u) packed 5 bits each: S <= 8 -> 16 entries x 3 bits ... kept generic below
    uint8_t next_tab[64], par_tab[64];   // S <= 32: [2 s + u]
    int S;
    uint8_t *msg;
    float *ysys, *ypar1, *ypar2;
    float2 *y, *h;            // fading: [3][frames][N] complex64, stream-major
    float mean_re, mean_im;   // fading: mean gain and per-component std of its scattered part
    float nlos_std;
};

// imaginary noise (counter word 5 + j) and gains (8 + j) of values 4q .. 4q+3 of stream j
__device__ __forceinline__ void fading_draws(const Params &p, uint32_t f_lo, uint32_t f_hi, uint32_t q, uint32_t j, float ni[4],
                                             float2 hh[4])
{
    const uint4 r = philox4x32_10(make_uint4(f_lo, f_hi, q, 5u + j), p.seed_lo, p.seed_hi);
    const float2 a = box_muller(r.x, r.y), b = box_muller(r.z, r.w);
    ni[0] = a.x; ni[1] = a.y; ni[2] = b.x; ni[3] = b.y;
    const uint4 g0 = philox4x32_10(make_uint4(f_lo, f_hi, 2u * q, 8u + j), p.seed_lo, p.seed_hi);
    const uint4 g1 = philox4x32_10(make_uint4(f_lo, f_hi, 2u * q + 1u, 8u + j), p.seed_lo, p.seed_hi);
    hh[0] = fading_gain(p.nlos_std, p.mean_re, p.mean_im, box_muller(g0.x, g0.y));
    hh[1] = fading_gain(p.nlos_std, p.mean_re, p.mean_im, box_muller(g0.z, g0.w));
    hh[2] = fading_gain(p.nlos_std, p.mean_re, p.mean_im, box_muller(g1.x, g1.y));
    hh[3] = fading_gain(p.nlos_std, p.mean_re, p.mean_im, box_muller(g1.z, g1.w));
}

// message bits: one thread per 128 bits
__global__ void __launch_bounds__(256) msg_kernel(const Params p)
{
    const int64_t blocks = (p.N + 127) >> 7;
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= p.frames * blocks) return;
    const int64_t fl = gid / blocks, b = gid - fl * blocks;
    const uint64_t fg = (uint64_t)(p.first_frame + fl);
    const uint4 r = philox4x32_10(make_uint4((uint32_t)fg, (uint32_t)(fg >> 32), (uint32_t)b, 0u), p.seed_lo, p.seed_hi);
    const uint32_t w[4] = {r.x, r.y, r.z, r.w};
    uint8_t *m = p.msg + fl * p.N + (b << 7);
    const int64_t cnt = min((int64_t)128, p.N - (b << 7));
    for (int64_t i = 0; i < cnt; ++i) m[i] = (uint8_t)((w[i >> 5] >> (i & 31)) & 1u);
}

// one thread per (frame, component encoder): encoder 0 walks msg in natural order (and emits the systematic stream),
// encoder 1 walks msg[p_array].  FADING: complex outputs y and gains h instead of the real streams.
template <bool FADING>
__global__ void __launch_bounds__(128) encode_kernel(const Params p)
{
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= 2 * p.frames) return;
    const int64_t fl = gid >> 1;
    const int enc = (int)(gid & 1);
    const uint64_t fg = (uint64_t)(p.first_frame + fl);
    const uint32_t f_lo = (uint32_t)fg, f_hi = (uint32_t)(fg >> 32);
    const uint8_t *m = p.msg + fl * p.N;
    float *ypar = FADING ? nullptr : (enc ? p.ypar2 : p.ypar1) + fl * p.N;
    float *ysys = FADING ? nullptr : p.ysys + fl * p.N;
    const int64_t plane = p.frames * p.N;                // fading: one stream of y / h
    float2 *cpar = FADING ? p.y + (1 + enc) * plane + fl * p.N : nullptr;
    float2 *hpar = FADING ? p.h + (1 + enc) * plane + fl * p.N : nullptr;
    float2 *csys = FADING ? p.y + fl * p.N : nullptr;
    float2 *hsys = FADING ? p.h + fl * p.N : nullptr;
    int state = 0;                                       // the encoder starts in state 0 (convcode.py:529)
    for (int64_t q = 0; q < p.N; q += 4) {
        const uint4 rp = philox4x32_10(make_uint4(f_lo, f_hi, (uint32_t)(q >> 2), 3u + (uint32_t)enc), p.seed_lo, p.seed_hi);
        const float2 a = box_muller(rp.x, rp.y), b = box_muller(rp.z, rp.w);
        const float nz[4] = {a.x, a.y, b.x, b.y};
        float ns[4] = {0.f, 0.f, 0.f, 0.f};
        if (enc == 0) {
            const uint4 rs = philox4x32_10(make_uint4(f_lo, f_hi, (uint32_t)(q >> 2), 2u), p.seed_lo, p.seed_hi);
            const float2 c = box_muller(rs.x, rs.y), d = box_muller(rs.z, rs.w);
            ns[0] = c.x; ns[1] = c.y; ns[2] = d.x; ns[3] = d.y;
        }
        float nzi[4], nsi[4];
        float2 hp[4], hs[4];
        if (FADING) {
            fading_draws(p, f_lo, f_hi, (uint32_t)(q >> 2), 1u + (uint32_t)enc, nzi, hp);
            if (enc == 0) fading_draws(p, f_lo, f_hi, (uint32_t)(q >> 2), 0u, nsi, hs);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int64_t t = q + i;
            if (t >= p.N) break;
            const int u = enc ? (int)m[__ldg(p.perm + t)] : (int)m[t];
            const int e = 2 * state + u;
            const int par = p.par_tab[e];
            state = p.next_tab[e];
            if (FADING) {
                const float xp = par ? 1.0f : -1.0f, xs = u ? 1.0f : -1.0f;
                cpar[t] = make_float2(fmaf(p.sigma, nz[i], hp[i].x * xp), fmaf(p.sigma, nzi[i], hp[i].y * xp));
                hpar[t] = hp[i];
                if (enc == 0) {
                    csys[t] = make_float2(fmaf(p.sigma, ns[i], hs[i].x * xs), fmaf(p.sigma, nsi[i], hs[i].y * xs));
                    hsys[t] = hs[i];
                }
            } else {
                ypar[t] = fmaf(p.sigma, nz[i], par ? 1.0f : -1.0f);
                if (enc == 0) ysys[t] = fmaf(p.sigma, ns[i], u ? 1.0f : -1.0f);
            }
        }
    }
}

// coherent BPSK combining: s = Re(conj(h) y) = h_re y_re + h_im y_im.  vec: y and h 16-byte aligned, s 16-byte aligned --
// threads [0, n/4) take four values each (two 16-byte loads of y and of h, one 16-byte store), the next n % 4 threads one.
__device__ __forceinline__ float combine1(float2 y, float2 h) { return fmaf(h.y, y.y, h.x * y.x); }

__global__ void __launch_bounds__(256) bpsk_combine_kernel(const float2 *__restrict__ y, const float2 *__restrict__ h, int64_t n,
                                                           float *__restrict__ s, int vec)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (vec) {
        const int64_t n4 = n >> 2;
        if (i < n4) {
            const float4 y0 = reinterpret_cast<const float4 *>(y)[2 * i], y1 = reinterpret_cast<const float4 *>(y)[2 * i + 1];
            const float4 h0 = reinterpret_cast<const float4 *>(h)[2 * i], h1 = reinterpret_cast<const float4 *>(h)[2 * i + 1];
            reinterpret_cast<float4 *>(s)[i] = make_float4(combine1(make_float2(y0.x, y0.y), make_float2(h0.x, h0.y)),
                                                           combine1(make_float2(y0.z, y0.w), make_float2(h0.z, h0.w)),
                                                           combine1(make_float2(y1.x, y1.y), make_float2(h1.x, h1.y)),
                                                           combine1(make_float2(y1.z, y1.w), make_float2(h1.z, h1.w)));
            return;
        }
        const int64_t t = 4 * n4 + (i - n4);             // scalar tail
        if (t < n) s[t] = combine1(y[t], h[t]);
    } else if (i < n) {
        s[i] = combine1(y[i], h[i]);
    }
}


// parity streams of the modem TX: one thread per (frame, component encoder), encoder 0 over msg, encoder 1 over
// msg[p_array]; threads [0, frames) run encoder 0 and [frames, 2 frames) encoder 1, so a warp walks one encoder.
// par: frames x 2N bytes, row f = [par1 | par2].  vec (N % 16 == 0, msg, perm and par 16-byte aligned): 16 steps at a
// time -- their 16 input bits are loaded first (one 16-byte load of msg, or four of perm and 16 gathers), then the
// state walks the table and the 16 parity bits leave in one 16-byte store.  The table is read from shared memory: the lanes
// of a warp look up different entries, which the constant cache would serve one address at a time.
struct ParityParams {
    int64_t frames, N;
    const int32_t *perm;
    const uint8_t *msg;
    uint8_t *par;
    uint8_t tab[64];          // S <= 32: [2 s + u] = (next state << 1) | parity bit; copied to shared memory per block
    int vec;
};

__global__ void __launch_bounds__(128) parity_kernel(const __grid_constant__ ParityParams p)
{
    __shared__ uint8_t tab[64];
    if (threadIdx.x < 64) tab[threadIdx.x] = p.tab[threadIdx.x];
    __syncthreads();
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= 2 * p.frames) return;
    const int enc = gid >= p.frames ? 1 : 0;
    const int64_t fl = gid - enc * p.frames;
    const uint8_t *m = p.msg + fl * p.N;
    uint8_t *out = p.par + (2 * fl + enc) * p.N;
    uint32_t state = 0;                                  // the encoder starts in state 0 (convcode.py:529)
    if (p.vec) {
        for (int64_t t = 0; t < p.N; t += 16) {
            uint32_t u[16];
            if (enc == 0) {
                const uint4 v = *reinterpret_cast<const uint4 *>(m + t);
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int i = 0; i < 16; ++i) u[i] = (w[i >> 2] >> (8 * (i & 3))) & 0xffu;
            } else {
                const int4 *pv = reinterpret_cast<const int4 *>(p.perm + t);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int4 q = __ldg(pv + j);
                    u[4 * j] = m[q.x]; u[4 * j + 1] = m[q.y]; u[4 * j + 2] = m[q.z]; u[4 * j + 3] = m[q.w];
                }
            }
            uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const uint32_t e = tab[2 * state + u[i]];
                w[i >> 2] |= (e & 1u) << (8 * (i & 3));
                state = e >> 1;
            }
            *reinterpret_cast<uint4 *>(out + t) = make_uint4(w[0], w[1], w[2], w[3]);
        }
    } else {
        for (int64_t t = 0; t < p.N; ++t) {
            const uint32_t u = enc ? (uint32_t)m[__ldg(p.perm + t)] : (uint32_t)m[t];
            const uint32_t e = tab[2 * state + u];
            out[t] = (uint8_t)(e & 1u);
            state = e >> 1;
        }
    }
}

}  // namespace turbolink

// the component trellis as the TX kernels take it: next state and parity bit of (s, u) at [2 s + u]; CPB_EUNSUPPORTED
// unless k = 1, n = 2, S <= 32 and systematic (MSB of the output symbol = input)
static int turbo_tables(const cpbTrellis *t, uint8_t next_tab[64], uint8_t par_tab[64], int *S_out)
{
    int k, n, S;
    cpb_trellis_dims(t, &k, &n, &S);
    if (k != 1 || n != 2 || S > 32) return CPB_EUNSUPPORTED;
    const int32_t *nst, *otab;
    cpb_trellis_host_tables(t, &nst, &otab);
    for (int s = 0; s < S; ++s)
        for (int u = 0; u < 2; ++u) {
            if (((otab[s * 2 + u] >> 1) & 1) != u) return CPB_EUNSUPPORTED;
            next_tab[2 * s + u] = (uint8_t)nst[s * 2 + u];
            par_tab[2 * s + u] = (uint8_t)(otab[s * 2 + u] & 1);
        }
    *S_out = S;
    return CPB_OK;
}

// fading == false: AWGN into sys / par1 / par2; otherwise flat fading into y / h ([3][frames][N] complex64)
static int turbo_link_tx_impl(const cpbTrellis *t, const int32_t *perm_dev, int64_t frames, int64_t N, uint64_t seed,
                              int64_t first_frame, float noise_sigma, bool fading, float mean_re, float mean_im, float nlos,
                              uint8_t *msg_dev, float *sys_dev, float *par1_dev, float *par2_dev, float *y_dev, float *h_dev,
                              void *stream)
{
    if (!t || frames < 0 || N < 1 || first_frame < 0) return CPB_EINVAL;
    if (fading && !(nlos >= 0.0f && std::isfinite(nlos) && std::isfinite(mean_re) && std::isfinite(mean_im) &&
                    std::isfinite(noise_sigma)))
        return CPB_EINVAL;
    if (frames == 0) return CPB_OK;
    if (!perm_dev || !msg_dev) return CPB_EINVAL;
    if (fading ? (!y_dev || !h_dev) : (!sys_dev || !par1_dev || !par2_dev)) return CPB_EINVAL;
    turbolink::Params p;
    memset(&p, 0, sizeof(p));
    const int rc = turbo_tables(t, p.next_tab, p.par_tab, &p.S);
    if (rc) return rc;
    p.frames = frames; p.N = N; p.first_frame = first_frame;
    p.seed_lo = (uint32_t)seed; p.seed_hi = (uint32_t)(seed >> 32);
    p.sigma = noise_sigma; p.perm = perm_dev;
    p.msg = msg_dev; p.ysys = sys_dev; p.ypar1 = par1_dev; p.ypar2 = par2_dev;
    p.y = reinterpret_cast<float2 *>(y_dev); p.h = reinterpret_cast<float2 *>(h_dev);
    p.mean_re = mean_re; p.mean_im = mean_im;
    p.nlos_std = (float)std::sqrt(0.5 * (double)nlos);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t blocks = (N + 127) >> 7;
    turbolink::msg_kernel<<<(unsigned)ceil_div(frames * blocks, 256), 256, 0, st>>>(p);
    if (fading) turbolink::encode_kernel<true><<<(unsigned)ceil_div(2 * frames, 128), 128, 0, st>>>(p);
    else turbolink::encode_kernel<false><<<(unsigned)ceil_div(2 * frames, 128), 128, 0, st>>>(p);
    CPB_LAUNCH_CHECK();
    return CPB_OK;
}

extern "C" int cpb_turbo_link_tx(const cpbTrellis *t, const int32_t *perm_dev, int64_t frames, int64_t N, uint64_t seed,
                                 int64_t first_frame, float noise_sigma, uint8_t *msg_dev, float *sys_dev, float *par1_dev,
                                 float *par2_dev, void *stream)
{
    return turbo_link_tx_impl(t, perm_dev, frames, N, seed, first_frame, noise_sigma, false, 0.0f, 0.0f, 0.0f, msg_dev, sys_dev,
                              par1_dev, par2_dev, nullptr, nullptr, stream);
}

extern "C" int cpb_turbo_link_tx_fading(const cpbTrellis *t, const int32_t *perm_dev, int64_t frames, int64_t N, uint64_t seed,
                                        int64_t first_frame, float noise_sigma, float mean_re, float mean_im, float nlos,
                                        uint8_t *msg_dev, float *y_dev, float *h_dev, void *stream)
{
    return turbo_link_tx_impl(t, perm_dev, frames, N, seed, first_frame, noise_sigma, true, mean_re, mean_im, nlos, msg_dev,
                              nullptr, nullptr, nullptr, y_dev, h_dev, stream);
}

// frames per pass of the modem TX: bounds the parity scratch (frames x 2N bytes) to 256 MiB
static const int64_t MODEM_CHUNK_FRAMES = 8192, MODEM_SCRATCH_BYTES = (int64_t)1 << 28;

// h_dev == nullptr: AWGN
static int turbo_link_tx_modem_impl(const cpbTrellis *t, const cpbModem *md, const int32_t *perm_dev, int64_t frames, int64_t N,
                                    uint64_t seed, int64_t first_frame, float noise_sigma, bool fading, float mean_re,
                                    float mean_im, float nlos, uint8_t *msg_dev, float *y_dev, float *h_dev, void *stream)
{
    if (!t || !md || frames < 0 || N < 1 || first_frame < 0) return CPB_EINVAL;
    if (fading && !(nlos >= 0.0f && std::isfinite(nlos) && std::isfinite(mean_re) && std::isfinite(mean_im) &&
                    std::isfinite(noise_sigma)))
        return CPB_EINVAL;
    int Mc, nb;
    const float *cst;
    cpb_modem_info(md, &Mc, &nb, &cst);
    if (nb < 1 || nb > 16 || (3 * N) % nb) return CPB_EINVAL;          // the code word must fill whole symbols
    if (frames == 0) return CPB_OK;
    if (!perm_dev || !msg_dev || !y_dev || (fading && !h_dev)) return CPB_EINVAL;
    if (N > ((int64_t)1 << 29)) return CPB_EUNSUPPORTED;                // 3N bits of a code word index with int
    turbolink::Params p;
    memset(&p, 0, sizeof(p));
    turbolink::ParityParams pp;
    memset(&pp, 0, sizeof(pp));
    int rc = turbo_tables(t, p.next_tab, p.par_tab, &p.S);
    if (rc) return rc;
    for (int e = 0; e < 2 * p.S; ++e) pp.tab[e] = (uint8_t)((p.next_tab[e] << 1) | p.par_tab[e]);
    const int64_t Fc = std::max<int64_t>(1, std::min<int64_t>({frames, MODEM_CHUNK_FRAMES, MODEM_SCRATCH_BYTES / (2 * N)}));
    cudaStream_t st = (cudaStream_t)stream;
    Scratch ws;
    rc = ws.acquire(nullptr, 0, (size_t)Fc * 2 * (size_t)N, st);
    if (rc) return rc;
    uint8_t *par = reinterpret_cast<uint8_t *>(ws.ptr);
    p.N = N;
    p.seed_lo = (uint32_t)seed; p.seed_hi = (uint32_t)(seed >> 32);
    pp.N = N; pp.perm = perm_dev; pp.par = par;
    cwtx::TxParams tp;
    memset(&tp, 0, sizeof(tp));
    tp.nsym = 3 * N / nb; tp.npairs = (tp.nsym + 1) / 2;
    tp.k = (int)N; tp.m = (int)(2 * N); tp.nb = nb;
    tp.seed_lo = p.seed_lo; tp.seed_hi = p.seed_hi;
    tp.sigma = noise_sigma;
    tp.mean_re = mean_re; tp.mean_im = mean_im; tp.nlos_std = (float)std::sqrt(0.5 * (double)nlos);
    tp.cst = reinterpret_cast<const float2 *>(cst);
    tp.par = par;
    const int64_t blocks = (N + 127) >> 7;
    for (int64_t f0 = 0; f0 < frames; f0 += Fc) {
        const int64_t nf = std::min(Fc, frames - f0);
        uint8_t *msg = msg_dev + f0 * N;
        p.frames = nf; p.first_frame = first_frame + f0; p.msg = msg;
        turbolink::msg_kernel<<<(unsigned)ceil_div(nf * blocks, 256), 256, 0, st>>>(p);
        pp.frames = nf; pp.msg = msg;
        pp.vec = (N % 16 == 0 && ((reinterpret_cast<uintptr_t>(msg) | reinterpret_cast<uintptr_t>(par) |
                               reinterpret_cast<uintptr_t>(perm_dev)) & 15) == 0) ? 1 : 0;
        turbolink::parity_kernel<<<(unsigned)ceil_div(2 * nf, 128), 128, 0, st>>>(pp);
        tp.frames = nf; tp.first_frame = first_frame + f0;
        tp.msg = msg;
        tp.y = reinterpret_cast<float2 *>(y_dev) + f0 * tp.nsym;
        tp.h = fading ? reinterpret_cast<float2 *>(h_dev) + f0 * tp.nsym : nullptr;
        cwtx::launch_modulate(tp, fading, st);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { ws.release(); return record_cuda_error(e, "turbo link modem tx kernels", __FILE__, __LINE__); }
    }
    ws.release();
    return CPB_OK;
}

extern "C" int cpb_turbo_link_tx_modem(const cpbTrellis *t, const cpbModem *modem, const int32_t *perm_dev, int64_t frames,
                                       int64_t N, uint64_t seed, int64_t first_frame, float noise_sigma, uint8_t *msg_dev,
                                       float *y_dev, void *stream)
{
    return turbo_link_tx_modem_impl(t, modem, perm_dev, frames, N, seed, first_frame, noise_sigma, false, 0.0f, 0.0f, 0.0f,
                                    msg_dev, y_dev, nullptr, stream);
}

extern "C" int cpb_turbo_link_tx_modem_fading(const cpbTrellis *t, const cpbModem *modem, const int32_t *perm_dev,
                                              int64_t frames, int64_t N, uint64_t seed, int64_t first_frame, float noise_sigma,
                                              float mean_re, float mean_im, float nlos, uint8_t *msg_dev, float *y_dev,
                                              float *h_dev, void *stream)
{
    return turbo_link_tx_modem_impl(t, modem, perm_dev, frames, N, seed, first_frame, noise_sigma, true, mean_re, mean_im, nlos,
                                    msg_dev, y_dev, h_dev, stream);
}

extern "C" int cpb_bpsk_combine(const float *y_dev, const float *h_dev, int64_t n, float *s_dev, void *stream)
{
    if (n < 0) return CPB_EINVAL;
    if (n == 0) return CPB_OK;
    if (!y_dev || !h_dev || !s_dev) return CPB_EINVAL;
    const bool vec = ((reinterpret_cast<uintptr_t>(y_dev) | reinterpret_cast<uintptr_t>(h_dev) |
                       reinterpret_cast<uintptr_t>(s_dev)) & 15) == 0;
    const int64_t threads = vec ? (n >> 2) + (n & 3) : n;
    turbolink::bpsk_combine_kernel<<<(unsigned)ceil_div(threads, 256), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float2 *>(y_dev), reinterpret_cast<const float2 *>(h_dev), n, s_dev, vec ? 1 : 0);
    CPB_LAUNCH_CHECK();
    return CPB_OK;
}

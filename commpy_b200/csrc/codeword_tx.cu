// Modulation and channel of a code word built on the device (codeword_tx.cuh): the LDPC TX (c = [message | parity]) and the
// turbo TX with a modem (c = [sys | par1 | par2], a = msg, b = the two parity streams).
#include "codeword_tx.cuh"
#include "common.cuh"
#include "philox.cuh"

using namespace cpb;

namespace cwtx {

// h * c; exact at h = 1 + 0j
__device__ __forceinline__ float2 cmul(float2 h, float2 c)
{
    return make_float2(h.x * c.x - h.y * c.y, h.x * c.y + h.y * c.x);
}

// one thread per (frame, symbol pair): the pair shares a Philox call of the noise (and of the gains)
template <bool FADING>
__global__ void __launch_bounds__(256) modulate_kernel(const TxParams p)
{
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= p.frames * p.npairs) return;
    const int64_t fl = gid / p.npairs;
    const int64_t q = gid - fl * p.npairs;
    const uint64_t fg = (uint64_t)(p.first_frame + fl);
    const uint32_t f_lo = (uint32_t)fg, f_hi = (uint32_t)(fg >> 32);
    const uint4 r = philox4x32_10(make_uint4(f_lo, f_hi, (uint32_t)q, 1u), p.seed_lo, p.seed_hi);
    const float2 nz[2] = {box_muller(r.x, r.y), box_muller(r.z, r.w)};
    float2 g[2];
    if (FADING) {
        const uint4 rh = philox4x32_10(make_uint4(f_lo, f_hi, (uint32_t)q, 5u), p.seed_lo, p.seed_hi);
        g[0] = fading_gain(p.nlos_std, p.mean_re, p.mean_im, box_muller(rh.x, rh.y));
        g[1] = fading_gain(p.nlos_std, p.mean_re, p.mean_im, box_muller(rh.z, rh.w));
    }
    const uint8_t *msg = p.msg + fl * p.k;
    const uint8_t *par = p.par + fl * p.m;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int64_t s = 2 * q + u;
        if (s >= p.nsym) break;
        uint32_t idx = 0;
        for (int b = 0; b < p.nb; ++b) {                 // first code bit of the symbol = MSB (modulation.py:93-96)
            const int64_t c = s * p.nb + b;
            idx = (idx << 1) | (uint32_t)(c < p.k ? msg[c] : par[c - p.k]);
        }
        float2 c = __ldg(&p.cst[idx]);
        if (FADING) {
            p.h[fl * p.nsym + s] = g[u];
            c = cmul(g[u], c);
        }
        p.y[fl * p.nsym + s] = make_float2(fmaf(p.sigma, nz[u].x, c.x), fmaf(p.sigma, nz[u].y, c.y));
    }
}

void launch_modulate(const TxParams &p, bool fading, cudaStream_t st)
{
    const unsigned grid = (unsigned)ceil_div(p.frames * p.npairs, 256);
    if (fading) modulate_kernel<true><<<grid, 256, 0, st>>>(p);
    else modulate_kernel<false><<<grid, 256, 0, st>>>(p);
}

}  // namespace cwtx

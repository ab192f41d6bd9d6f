// Counter-based random streams of the device TX chains (txlink.cu, turbolink.cu, ldpclink.cu, codeword_tx.cu).
//
// Every random value of global frame f is drawn from Philox4x32-10 with key = seed (lo, hi) and counter
// (f_lo, f_hi, index, word).  A value depends only on (seed, f, index, word), never on the launch geometry, the batch
// split or the number of GPUs (each rank passes its own first_frame).  The counter word names the stream; turbo stream j
// is 0 = sys, 1 = par1, 2 = par2:
//
//     word    stream                   index   values of one Philox call
//     0       message bits             b       bits 128 b .. 128 b + 127 (LSB first in x, y, z, w)
//     1       conv noise               q       symbols 2q, 2q+1 (box_muller(x, y), box_muller(z, w))
//     2 + j   turbo real noise         q       values 4q .. 4q+3 (Re, Im of box_muller(x, y), then of (z, w))
//     5       conv gains               q       symbols 2q, 2q+1, as the conv noise
//     5 + j   turbo imaginary noise    q       values 4q .. 4q+3, as the real noise
//     8 + j   turbo gains              c       values 2c, 2c+1 (one complex gain per box_muller)
//     0, 1, 5 LDPC link and turbo link over a modem: message bits, noise and gains as the conv link's words 0, 1 and 5
//             (the noise and gains drawn by the shared code-word modulator, codeword_tx.cu)
//
// The links share words 0 and 5; word 5 is a different stream in the BPSK turbo link, as no link draws from another's.
#pragma once
#include <stdint.h>

namespace cpb {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1)
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c;
}

// two uint32 -> two standard normals (Box-Muller); u1 in (0, 1]
__device__ __forceinline__ float2 box_muller(uint32_t a, uint32_t b)
{
    const float u1 = fmaf((float)a, 2.3283064365386963e-10f, 1.1641532182693481e-10f);
    const float u2 = (float)b * 2.3283064365386963e-10f;
    const float r = sqrtf(-2.0f * __logf(u1));
    float sn, cs;
    __sincosf(6.283185307179586f * u2, &sn, &cs);
    return make_float2(r * cs, r * sn);
}

// flat-fading gain from two standard normals g: mean + nlos_std (g.x + j g.y), nlos_std = sqrt(nlos / 2)
__device__ __forceinline__ float2 fading_gain(float nlos_std, float mean_re, float mean_im, float2 g)
{
    return make_float2(fmaf(nlos_std, g.x, mean_re), fmaf(nlos_std, g.y, mean_im));
}

}  // namespace cpb

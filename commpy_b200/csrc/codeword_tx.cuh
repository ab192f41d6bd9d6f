// Code-word modulator shared by the device TX chains whose code words are built before modulation (ldpclink.cu,
// turbolink.cu): c = [a (k bytes) | b (m bytes)] per frame, mapped nb bits at a time MSB first (Modem.modulate), times
// a flat-fading gain when FADING, plus noise.  Symbol s's noise is Philox counter word 1 and its gain word 5 of the conv
// link (philox.cuh): box_muller of the pair (x, y) for even s, (z, w) for odd s of counter s / 2.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cwtx {

struct TxParams {
    int64_t frames, nsym, npairs, first_frame;
    int k, m, nb;
    uint32_t seed_lo, seed_hi;
    float sigma;
    float mean_re, mean_im, nlos_std;
    const float2 *cst;
    const uint8_t *msg, *par;                            // frames x k, frames x m: code word c = [msg | par]
    float2 *y, *h;                                       // frames x nsym complex64; h only when fading
};

// modulate_kernel<fading> over p.frames frames, one thread per (frame, symbol pair)
void launch_modulate(const TxParams &p, bool fading, cudaStream_t st);

}  // namespace cwtx

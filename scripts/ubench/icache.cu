// Micro-benchmark: does a long straight-line loop body (like the unrolled add-compare-select block) run at full issue
// rate, or does instruction fetch limit it?  Body = N pairs (VIADDMNMX + IMAD) over 16 independent chains.
#include <cstdio>
#include <vector>
#include <cstdint>
#include <cuda_runtime.h>

template <int NPAIR>
__global__ void k(uint32_t *out, long long *cyc, uint32_t seed, int iters)
{
    uint32_t x[8], y[8];
    for (int i = 0; i < 8; ++i) { x[i] = seed + i * 77 + threadIdx.x; y[i] = seed * 5 + i; }
    uint32_t b = seed * 3 + 1, c = seed ^ 0x55aa;
    long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int r = 0; r < NPAIR / 8; ++r)
#pragma unroll
            for (int i = 0; i < 8; ++i) { x[i] = __viaddmin_u16x2(x[i], b, c); y[i] = y[i] * b + c; }
    }
    long long t1 = clock64();
    uint32_t s = 0;
    for (int i = 0; i < 8; ++i) s ^= x[i] ^ y[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int NPAIR>
void run(uint32_t *out, long long *cyc, int nsm)
{
    for (int warps : {1, 4, 8}) {
        const int iters = 65536 / NPAIR;
        k<NPAIR><<<nsm, 32 * warps>>>(out, cyc, 12345, iters);          // one CTA per SM
        std::vector<long long> h(nsm);
        cudaMemcpy(h.data(), cyc, sizeof(long long) * nsm, cudaMemcpyDeviceToHost);
        double m = 0; for (int i = 0; i < nsm; ++i) m += (double)h[i];
        m /= nsm;
        printf("body %5d instr (%6.1f KB): warps/SM %d: %.3f cycles per instruction per warp, %.3f IPC per SMSP\n", 2 * NPAIR, 2 * NPAIR * 16 / 1024.0,
               warps, m / ((double)iters * 2 * NPAIR), (warps >= 4 ? warps / 4.0 : 1.0) * (double)iters * 2 * NPAIR / m);
    }
}

int main()
{
    uint32_t *out; long long *cyc;
    int nsm = 0;
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&out, 1 << 22); cudaMalloc(&cyc, sizeof(long long) * nsm);
    run<64>(out, cyc, nsm); run<128>(out, cyc, nsm); run<256>(out, cyc, nsm); run<384>(out, cyc, nsm); run<512>(out, cyc, nsm);
    run<768>(out, cyc, nsm); run<1024>(out, cyc, nsm); run<2048>(out, cyc, nsm); run<4096>(out, cyc, nsm);
    return 0;
}

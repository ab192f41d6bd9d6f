// Micro-benchmark: issue rate and latency of the integer min/add-min instructions the Viterbi kernels use (sm_90a).
// One warp per CTA, one CTA per SM sub-partition is enough: cycles per warp instruction = rt of the pipe.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

#define REP 256
template <int OP>
__device__ __forceinline__ uint32_t op(uint32_t a, uint32_t b, uint32_t c)
{
    if (OP == 0) return __viaddmin_u16x2(a, b, c);
    if (OP == 1) return __viaddmin_u32(a, b, c);
    if (OP == 2) return __vimin3_u16x2(a, b, c);
    if (OP == 3) return __vimin3_u32(a, b, c);
    if (OP == 4) return __vminu2(a, b) + c * 0;          // 2-input packed min
    if (OP == 5) return min(a, b) ^ c;                   // 2-input 32-bit min + xor (2 instr)
    if (OP == 6) return (a & b) | c;                     // LOP3
    if (OP == 7) return a + b + c;                       // IADD3
    if (OP == 8) return a * b + c;                       // IMAD
    if (OP == 9) return __vaddus2(a, b) | c;             // packed add (saturating)
    if (OP == 10) return __vadd2(a, b) | c;
    if (OP == 11) return __viaddmax_u16x2(a, b, c);
    if (OP == 12) return __vimin_s16x2_relu(a, b) | c;
    return 0;
}

template <int OP, int CHAINS>
__global__ void k(uint32_t *out, long long *cyc, uint32_t seed)
{
    uint32_t x[CHAINS];
    for (int i = 0; i < CHAINS; ++i) x[i] = seed + i * 77 + threadIdx.x;
    uint32_t b = seed * 3 + 1, c = seed ^ 0x55aa;
    long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < 64; ++it) {
#pragma unroll
        for (int r = 0; r < REP / CHAINS; ++r)
#pragma unroll
            for (int i = 0; i < CHAINS; ++i) x[i] = op<OP>(x[i], b, c);
    }
    long long t1 = clock64();
    uint32_t s = 0;
    for (int i = 0; i < CHAINS; ++i) s ^= x[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}

// mixed: alternate add-min (ALU) with IMAD (FMA): can they issue back to back?
template <int CHAINS>
__global__ void kmix(uint32_t *out, long long *cyc, uint32_t seed)
{
    uint32_t x[CHAINS], y[CHAINS];
    for (int i = 0; i < CHAINS; ++i) { x[i] = seed + i * 77 + threadIdx.x; y[i] = seed * 5 + i; }
    uint32_t b = seed * 3 + 1, c = seed ^ 0x55aa;
    long long t0 = clock64();
#pragma unroll 1
    for (int it = 0; it < 64; ++it) {
#pragma unroll
        for (int r = 0; r < REP / CHAINS; ++r)
#pragma unroll
            for (int i = 0; i < CHAINS; ++i) { x[i] = __viaddmin_u16x2(x[i], b, c); y[i] = y[i] * b + c; }
    }
    long long t1 = clock64();
    uint32_t s = 0;
    for (int i = 0; i < CHAINS; ++i) s ^= x[i] ^ y[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) *cyc = t1 - t0;
}

template <int OP>
void run(const char *name, uint32_t *out, long long *cyc, int warps)
{
    long long h1, h8;
    k<OP, 1><<<1, 32 * warps>>>(out, cyc, 12345); cudaMemcpy(&h1, cyc, 8, cudaMemcpyDeviceToHost);
    k<OP, 8><<<1, 32 * warps>>>(out, cyc, 12345); cudaMemcpy(&h8, cyc, 8, cudaMemcpyDeviceToHost);
    printf("%-22s warps/CTA %d: dependent %.2f cyc/op, 8 chains %.2f cyc/op (per warp-instr: x%d warps on the SM)\n", name, warps,
           (double)h1 / (64.0 * REP), (double)h8 / (64.0 * REP), warps);
}

int main()
{
    uint32_t *out; long long *cyc;
    cudaMalloc(&out, 1 << 20); cudaMalloc(&cyc, 8);
    for (int warps : {1, 4, 8}) {
        run<0>("VIADDMNMX.U16x2", out, cyc, warps);
        run<1>("VIADDMNMX.U32", out, cyc, warps);
        run<2>("VIMNMX3.U16x2", out, cyc, warps);
        run<3>("VIMNMX3.U32", out, cyc, warps);
        run<4>("VIMNMX.U16x2 (2-in)", out, cyc, warps);
        run<5>("IMNMX.U32+LOP", out, cyc, warps);
        run<6>("LOP3", out, cyc, warps);
        run<7>("IADD3", out, cyc, warps);
        run<8>("IMAD", out, cyc, warps);
        run<9>("vaddus2|", out, cyc, warps);
        run<10>("vadd2|", out, cyc, warps);
        run<11>("VIADDMNMX(max).U16x2", out, cyc, warps);
        long long h;
        kmix<8><<<1, 32 * warps>>>(out, cyc, 12345); cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        printf("mixed addmin+IMAD pairs warps %d: %.2f cyc per pair\n", warps, (double)h / (64.0 * REP));
    }
    return 0;
}

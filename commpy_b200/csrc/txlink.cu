// Transmit side of a coded AWGN link, generated on the device -- the caller of the hot path, SURVEY 8(f) row 1.
// One kernel replaces, for a batch of frames, what LinkModel.link_performance does per frame on the host:
//     msg = randint(0, 2, send_chunk)                         commpy/links.py:318
//     coded = conv_encode(msg, trellis, 'cont')               commpy/channelcoding/convcode.py:475-558 (loop :535-540)
//     symbols = modem.modulate(coded)                         commpy/modulation.py:79-98 (MSB-first index, :93-96)
//     y = symbols + noise                                     commpy/channels.py:181-221, noise scale :53,:74
// so that 1e8-symbol BER points (BASELINE config 5) never touch the host.  Nothing here is on the parity path: the
// message bits are returned, and the receiver (cpb_demod_soft -> cpb_viterbi_decode -> cpb_count_errors) is what is
// checked against the oracle.
//
// Randomness is counter based (Philox4x32-10): message bit i of global frame f is bit (i & 127) of
// Philox(counter = (f_lo, f_hi, i >> 7, 0), key = seed); the noise of symbols 2q, 2q+1 of frame f comes from
// Philox(counter = (f_lo, f_hi, q, 1), key = seed) through Box-Muller.  Results therefore do not depend on the launch
// geometry, the batch split or the number of GPUs (each rank passes its own first_frame), SURVEY 8(e).
//
// Encoder: k = 1 feed-forward shift register; tap mask g_j bit b multiplies the input delayed by b (bit 0 = current
// input) -- derived on the host from the Trellis tables and verified against every (state, input) entry.
#include <cmath>
#include <vector>

#include "common.cuh"

using namespace cpb;

struct cpbTrellis;
struct cpbModem;
void cpb_trellis_dims(const cpbTrellis *t, int *k, int *n, int *S);
void cpb_trellis_host_tables(const cpbTrellis *t, const int32_t **next, const int32_t **out);
void cpb_modem_info(const cpbModem *m, int *M, int *nb, const float **cst_dev);

namespace txlink {

struct Params {
    uint32_t g[8];            // tap masks, n <= 8
    int n, mem;               // outputs per input bit, memory M
    int nb, Mc;               // bits per symbol, constellation size
    int64_t frames, frame_bits, nsym;   // per frame: information bits, symbols
    int64_t first_frame;
    uint32_t seed_lo, seed_hi;
    float sigma;              // per real component
    int spt;                  // symbols per thread
    uint32_t punct_mask;      // puncturing pattern over the coded stream (bit c mod punct_len set = keep), convcode.py:752-774
    int punct_len, punct_ones;
    int64_t chunks;           // threads per frame
    const float2 *cst;
    uint8_t *msg;
    float2 *y;
};

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

__global__ void __launch_bounds__(128) conv_link_tx_kernel(const Params p)
{
    extern __shared__ float2 s_cst[];
    for (int k = threadIdx.x; k < p.Mc; k += blockDim.x) s_cst[k] = p.cst[k];
    __syncthreads();
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= p.frames * p.chunks) return;
    const int64_t fl = gid / p.chunks;                       // frame within this call
    const int64_t ch = gid - fl * p.chunks;
    const uint64_t fg = (uint64_t)(p.first_frame + fl);      // global frame id
    const uint32_t f_lo = (uint32_t)fg, f_hi = (uint32_t)(fg >> 32);
    const int64_t s0 = ch * p.spt;
    const int64_t s1 = min(s0 + (int64_t)p.spt, p.nsym);
    // first information bit: s0 * nb kept bits are whole puncturing periods (punct_ones kept out of punct_len coded bits)
    int64_t i = (s0 * p.nb / p.punct_ones) * p.punct_len / p.n;
    int cpos = 0;

    uint32_t blk_id = 0xffffffffu;
    uint4 blk = make_uint4(0, 0, 0, 0);
    auto get_bit = [&](int64_t idx) -> uint32_t {
        const uint32_t b = (uint32_t)(idx >> 7);
        if (b != blk_id) { blk = philox4x32_10(make_uint4(f_lo, f_hi, b, 0u), p.seed_lo, p.seed_hi); blk_id = b; }
        const uint32_t w = (uint32_t)(idx >> 5) & 3u;
        const uint32_t word = (w == 0) ? blk.x : (w == 1) ? blk.y : (w == 2) ? blk.z : blk.w;
        return (word >> ((uint32_t)idx & 31u)) & 1u;
    };

    // shift register before bit i: bit b = u_{i-1-b}; the encoder starts in state 0 (convcode.py:529)
    uint32_t reg = 0;
    for (int b = 0; b < p.mem; ++b)
        if (i - 1 - b >= 0) reg |= get_bit(i - 1 - b) << b;
    const uint32_t regmask = (2u << p.mem) - 1u;

    uint8_t *msg = p.msg + fl * p.frame_bits;
    float2 *y = p.y + fl * p.nsym;
    const bool pack4 = ((p.frame_bits & 3) == 0) && ((i & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.msg) & 3) == 0);
    uint32_t mword = 0;
    uint64_t acc = 0;
    int nacc = 0;
    int64_t sym = s0;
    float2 spare = make_float2(0.f, 0.f);
    while (sym < s1) {
        const uint32_t u = get_bit(i);
        reg = ((reg << 1) | u) & regmask;
        if (pack4) {
            mword |= u << (8 * ((uint32_t)i & 3u));
            if (((uint32_t)i & 3u) == 3u) { *reinterpret_cast<uint32_t *>(msg + (i - 3)) = mword; mword = 0; }
        } else {
            msg[i] = (uint8_t)u;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (j < p.n) {
                if ((p.punct_mask >> cpos) & 1u) { acc = (acc << 1) | (uint64_t)(__popc(reg & p.g[j]) & 1); ++nacc; }
                cpos = (cpos + 1 == p.punct_len) ? 0 : cpos + 1;
            }
        ++i;
        while (nacc >= p.nb && sym < s1) {
            nacc -= p.nb;
            const uint32_t idx = (uint32_t)(acc >> nacc) & (uint32_t)(p.Mc - 1);      // first coded bit = MSB (modulation.py:93-96)
            float2 nz;
            if ((sym & 1) == 0) {
                const uint4 r = philox4x32_10(make_uint4(f_lo, f_hi, (uint32_t)(sym >> 1), 1u), p.seed_lo, p.seed_hi);
                nz = box_muller(r.x, r.y);
                spare = box_muller(r.z, r.w);
            } else {
                if (sym == s0) {               // (cannot happen: chunks start on even symbols) kept for safety
                    const uint4 r = philox4x32_10(make_uint4(f_lo, f_hi, (uint32_t)(sym >> 1), 1u), p.seed_lo, p.seed_hi);
                    spare = box_muller(r.z, r.w);
                }
                nz = spare;
            }
            const float2 c = s_cst[idx];
            y[sym] = make_float2(fmaf(p.sigma, nz.x, c.x), fmaf(p.sigma, nz.y, c.y));
            ++sym;
        }
    }
    if (pack4 && (i & 3)) {                                  // short last chunk: flush the partial word
        const int r = (int)(i & 3);
        for (int b = 0; b < r; ++b) msg[i - r + b] = (uint8_t)((mword >> (8 * b)) & 1u);
    }
}

// ------------------------------------------------------------------------------------------------
// Word-parallel form of the kernel above for the common link: n = 2 outputs per input bit, no puncturing, 2 / 4 / 8 bits per
// symbol (QPSK, 16-QAM, 256-QAM) and frames of whole 128-bit message blocks.  Same random streams, same outputs (the test
// suite compares the two kernels bit for bit), far fewer instructions per symbol:
//   * a thread owns ONE Philox message block (128 information bits = 256 / nb symbols) and encodes 32 bits at a time: the
//     coded stream of output j is the XOR of the message word delayed by each set tap (funnel shifts across the word
//     boundary) -- ~25 instructions per 32 bits instead of a popcount per bit and output;
//   * a symbol's nb coded bits are nb/2 consecutive bits of each of the two coded words: the constellation is re-indexed once
//     per CTA by (bits of output 0 | bits of output 1 << nb/2), so mapping is two bit-field extracts and one 8-byte load;
//   * message bytes leave as 16-byte stores (4 bits -> 4 bytes by one multiply), symbols as 16-byte stores (the two symbols
//     that share a Philox noise block).
// ------------------------------------------------------------------------------------------------
template <int NB>
__global__ void __launch_bounds__(128) conv_link_tx_fast_kernel(const Params p)
{
    constexpr int H = NB / 2;                    // information bits per symbol
    constexpr int SPW = 32 / H;                  // symbols per 32-bit message word
    __shared__ float2 s_map[1 << NB];
    for (int k = threadIdx.x; k < (1 << NB); k += blockDim.x) {
        // k = a | b << H, a / b = H consecutive bits of output 0 / 1 (bit i = step t+i); the modem's index takes the coded
        // bits in transmission order c0[t], c1[t], c0[t+1], ... MSB first (modulation.py:93-96)
        int idx = 0;
#pragma unroll
        for (int i = 0; i < H; ++i) idx |= (((k >> i) & 1) << (NB - 1 - 2 * i)) | (((k >> (H + i)) & 1) << (NB - 2 - 2 * i));
        s_map[k] = p.cst[idx];
    }
    __syncthreads();
    const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gid >= p.frames * p.chunks) return;
    const int64_t fl = gid / p.chunks;                       // frame within this call
    const uint32_t b = (uint32_t)(gid - fl * p.chunks);      // message block of the frame
    const uint64_t fg = (uint64_t)(p.first_frame + fl);
    const uint32_t f_lo = (uint32_t)fg, f_hi = (uint32_t)(fg >> 32);

    const uint4 blk = philox4x32_10(make_uint4(f_lo, f_hi, b, 0u), p.seed_lo, p.seed_hi);
    uint32_t prev = 0u;                                      // the 32 message bits before this block (state 0 before bit 0)
    if (b > 0) prev = philox4x32_10(make_uint4(f_lo, f_hi, b - 1u, 0u), p.seed_lo, p.seed_hi).w;
    const uint32_t word[4] = {blk.x, blk.y, blk.z, blk.w};

    uint8_t *msg = p.msg + fl * p.frame_bits + (int64_t)b * 128;
    float2 *y = p.y + fl * p.nsym + (int64_t)b * (4 * SPW);
    const uint32_t g0 = p.g[0], g1 = p.g[1];
#pragma unroll
    for (int w = 0; w < 4; ++w) {
        const uint32_t cur = word[w];
        // message bytes: bit i of a nibble -> byte i (x * 0x00204081 puts bit i at 8 i, stray products land on other bits)
        uint32_t mb[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) mb[q] = (((cur >> (4 * q)) & 15u) * 0x00204081u) & 0x01010101u;
        *reinterpret_cast<uint4 *>(msg + 32 * w) = make_uint4(mb[0], mb[1], mb[2], mb[3]);
        *reinterpret_cast<uint4 *>(msg + 32 * w + 16) = make_uint4(mb[4], mb[5], mb[6], mb[7]);
        // coded words: c_j bit i = XOR over taps d of u_{t+i-d}
        uint32_t c0 = 0u, c1 = 0u;
        for (int d = 0; d <= p.mem; ++d) {
            const uint32_t dl = d ? __funnelshift_l(prev, cur, d) : cur;
            if ((g0 >> d) & 1u) c0 ^= dl;
            if ((g1 >> d) & 1u) c1 ^= dl;
        }
        prev = cur;
#pragma unroll
        for (int s2 = 0; s2 < SPW; s2 += 2) {
            const uint32_t sym = (uint32_t)(w * SPW + s2);               // even: symbols sym, sym+1 share a noise block
            const uint32_t gs = b * (4u * SPW) + sym;                    // symbol index within the frame
            const uint4 r = philox4x32_10(make_uint4(f_lo, f_hi, gs >> 1, 1u), p.seed_lo, p.seed_hi);
            const float2 n0 = box_muller(r.x, r.y), n1 = box_muller(r.z, r.w);
            const uint32_t k0 = ((c0 >> (H * s2)) & ((1u << H) - 1u)) | (((c1 >> (H * s2)) & ((1u << H) - 1u)) << H);
            const uint32_t k1 = ((c0 >> (H * (s2 + 1))) & ((1u << H) - 1u)) | (((c1 >> (H * (s2 + 1))) & ((1u << H) - 1u)) << H);
            const float2 a0 = s_map[k0], a1 = s_map[k1];
            *reinterpret_cast<float4 *>(y + sym) = make_float4(fmaf(p.sigma, n0.x, a0.x), fmaf(p.sigma, n0.y, a0.y),
                                                               fmaf(p.sigma, n1.x, a1.x), fmaf(p.sigma, n1.y, a1.y));
        }
    }
}

static int gcd_int(int a, int b) { return b ? gcd_int(b, a % b) : a; }

}  // namespace txlink

static int conv_link_tx_impl(const cpbTrellis *t, const cpbModem *m, int64_t frames, int64_t frame_bits, uint64_t seed,
                             int64_t first_frame, float noise_sigma, const int32_t *punct_vec, int punct_len,
                             uint8_t *msg_dev, float *y_dev, void *stream)
{
    if (!t || !m || frames < 0 || frame_bits < 1 || first_frame < 0) return CPB_EINVAL;
    if (frames == 0) return CPB_OK;
    if (!msg_dev || !y_dev) return CPB_EINVAL;
    int k, n, S;
    cpb_trellis_dims(t, &k, &n, &S);
    if (k != 1 || n < 1 || n > 8) return CPB_EUNSUPPORTED;
    int mem = 0;
    while ((1 << mem) < S) ++mem;
    if ((1 << mem) != S || mem > 24) return CPB_EUNSUPPORTED;
    const int32_t *nst, *otab;
    cpb_trellis_host_tables(t, &nst, &otab);
    txlink::Params p;
    memset(&p, 0, sizeof(p));
    // tap masks from the tables (bit 0: input with an empty register; bit b: the state with only delay b set), then
    // verified on every entry -- a recursive or non-linear trellis is refused (CPB_EUNSUPPORTED)
    for (int j = 0; j < n; ++j) {
        uint32_t g = (uint32_t)((otab[0 * 2 + 1] >> (n - 1 - j)) & 1);
        for (int b = 1; b <= mem; ++b) g |= (uint32_t)((otab[(1 << (mem - b)) * 2 + 0] >> (n - 1 - j)) & 1) << b;
        p.g[j] = g;
    }
    for (int s = 0; s < S; ++s)
        for (int u = 0; u < 2; ++u) {
            if (nst[s * 2 + u] != ((u << (mem - 1)) | (s >> 1))) return CPB_EUNSUPPORTED;
            uint32_t reg = (uint32_t)u;
            for (int b = 1; b <= mem; ++b) reg |= (uint32_t)((s >> (mem - b)) & 1) << b;
            int sym = 0;
            for (int j = 0; j < n; ++j) sym = (sym << 1) | (__builtin_popcount(reg & p.g[j]) & 1);
            if (sym != otab[s * 2 + u]) return CPB_EUNSUPPORTED;
        }
    int Mc, nb;
    const float *cst;
    cpb_modem_info(m, &Mc, &nb, &cst);
    if (nb < 1 || nb > 16) return CPB_EUNSUPPORTED;
    // puncturing pattern over the coded stream; none = every bit of a period of n kept
    if (punct_vec) {
        if (punct_len < 1 || punct_len > 32 || (punct_len % n) != 0) return CPB_EUNSUPPORTED;
        for (int i = 0; i < punct_len; ++i)
            if (punct_vec[i] == 1) { p.punct_mask |= 1u << i; ++p.punct_ones; }
        p.punct_len = punct_len;
        if (p.punct_ones == 0) return CPB_EINVAL;
    } else {
        p.punct_len = n; p.punct_ones = n; p.punct_mask = (1u << n) - 1u;
    }
    const int64_t coded = frame_bits * n;
    const int64_t kept = (coded / p.punct_len) * p.punct_ones +
                         __builtin_popcount(p.punct_mask & ((1u << (coded % p.punct_len)) - 1u));
    if (kept % nb) return CPB_EINVAL;                        // the frame must fill whole symbols
    p.n = n; p.mem = mem; p.nb = nb; p.Mc = Mc;
    p.frames = frames; p.frame_bits = frame_bits; p.nsym = kept / nb;
    p.first_frame = first_frame;
    p.seed_lo = (uint32_t)seed; p.seed_hi = (uint32_t)(seed >> 32);
    p.sigma = noise_sigma;
    // symbols per thread: even (noise comes in pairs) and a whole number of puncturing periods, about 32
    int unit = p.punct_ones / txlink::gcd_int(p.punct_ones, nb);
    if (unit & 1) unit *= 2;
    p.spt = unit * ((32 + unit - 1) / unit);
    p.chunks = ceil_div(p.nsym, (int64_t)p.spt);
    p.cst = reinterpret_cast<const float2 *>(cst);
    p.msg = msg_dev;
    p.y = reinterpret_cast<float2 *>(y_dev);
    // word-parallel kernel: n = 2, no puncturing, 2 / 4 / 8 bits per symbol, whole 128-bit message blocks, 16-byte aligned rows
    const bool fast = !punct_vec && n == 2 && (nb == 2 || nb == 4 || nb == 8) && Mc == (1 << nb) && (frame_bits % 128) == 0 &&
                      mem >= 1 && mem < 32 && (reinterpret_cast<uintptr_t>(msg_dev) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(y_dev) & 15) == 0 && !option(CPB_OPT_TX_FORCE_GENERIC);
    if (fast) {
        p.chunks = frame_bits / 128;
        const int64_t threads = frames * p.chunks;
        const unsigned grid = (unsigned)ceil_div(threads, 128);
        if (nb == 2) txlink::conv_link_tx_fast_kernel<2><<<grid, 128, 0, (cudaStream_t)stream>>>(p);
        else if (nb == 4) txlink::conv_link_tx_fast_kernel<4><<<grid, 128, 0, (cudaStream_t)stream>>>(p);
        else txlink::conv_link_tx_fast_kernel<8><<<grid, 128, 0, (cudaStream_t)stream>>>(p);
        CPB_LAUNCH_CHECK();
        return CPB_OK;
    }
    const int64_t threads = frames * p.chunks;
    const unsigned grid = (unsigned)ceil_div(threads, 128);
    txlink::conv_link_tx_kernel<<<grid, 128, (size_t)Mc * sizeof(float2), (cudaStream_t)stream>>>(p);
    CPB_LAUNCH_CHECK();
    return CPB_OK;
}

extern "C" int cpb_conv_link_tx(const cpbTrellis *t, const cpbModem *m, int64_t frames, int64_t frame_bits,
                                uint64_t seed, int64_t first_frame, float noise_sigma, uint8_t *msg_dev, float *y_dev,
                                void *stream)
{
    return conv_link_tx_impl(t, m, frames, frame_bits, seed, first_frame, noise_sigma, nullptr, 0, msg_dev, y_dev, stream);
}

extern "C" int cpb_conv_link_tx_punctured(const cpbTrellis *t, const cpbModem *m, int64_t frames, int64_t frame_bits,
                                          uint64_t seed, int64_t first_frame, float noise_sigma,
                                          const int32_t *punct_vec_host, int punct_len, uint8_t *msg_dev, float *y_dev,
                                          void *stream)
{
    if (!punct_vec_host) return CPB_EINVAL;
    return conv_link_tx_impl(t, m, frames, frame_bits, seed, first_frame, noise_sigma, punct_vec_host, punct_len, msg_dev,
                             y_dev, stream);
}

/*
 * commpy_b200.h -- C-ABI of libcommpy_b200.so: CommPy's decoding hot path on H100 (sm_90a).
 *
 * The reference (veeresht/CommPy @ 9aecd7c) has no FFI layer: the hot path sits behind plain
 * Python functions.  Each entry point below names the reference function whose loop nest it
 * replaces (file:line, relative to the reference checkout); the Python wrappers under
 * commpy_b200/ keep the reference signatures and call these through ctypes (INTEGRATION.md).
 *
 * Conventions
 *  - every function returns a cpb status (0 = CPB_OK); no C++ exception crosses the boundary;
 *    cpb_strerror() maps a status to text, cpb_last_cuda_error() returns the failing CUDA call's text.
 *  - "_dev" pointers are device memory on the CURRENT CUDA device, caller-owned (torch tensors or cudaMalloc);
 *    "_host" pointers are host memory (pageable or pinned).  The library allocates only the opaque
 *    handles created here (a handle also owns the streams / staging buffers of the *_host calls made with it)
 *    and, when workspace == NULL, stream-ordered scratch (cudaMallocAsync).  No global mutable state.
 *  - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).  Device-buffer entry
 *    points are stream-ordered and never synchronise; *_host entry points return after their output
 *    host buffer is complete.
 *  - frames / codewords / blocks are independent: batch is the leading dimension, frame-major, dense.
 *  - bit order everywhere is CommPy's: MSB first (commpy/utilities.py:58-86).
 */
#ifndef COMMPY_B200_H
#define COMMPY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes --------------------------------------------------------------------------- */
#define CPB_OK 0
#define CPB_EINVAL 1        /* bad argument                      -> ValueError in the Python mirror */
#define CPB_EUNSUPPORTED 2  /* legal in the reference, not built -> NotImplementedError          */
#define CPB_ECUDA 3         /* CUDA runtime failure              -> RuntimeError                 */
#define CPB_ENOMEM 4
#define CPB_ETRELLIS 5      /* a trellis state does not have exactly 2^k predecessors            */

const char *cpb_strerror(int status);
const char *cpb_last_cuda_error(void);
int cpb_version(void);                     /* 10000*major + 100*minor + patch */
int cpb_device_info(int *sm_count, int *cc_major, int *cc_minor, size_t *global_mem_bytes);
/* Decoder calls made without a caller workspace take their scratch from a library-owned stream-ordered memory pool of the
 * current device, which keeps the memory for the next call (a call must not pay for gigabytes of fresh device memory).
 * cpb_release_scratch() returns whatever is not in use to the driver; no reference counterpart (housekeeping). */
int cpb_release_scratch(void);
/* Explicit switches for tests and kernel cross-checks (process wide, default 0).  The library never reads the
 * environment.  They select between kernels that implement the SAME reference semantics. */
#define CPB_OPT_VITERBI_FORCE_GENERIC 0   /* 1: every trellis goes through the table-driven Viterbi kernel */
#define CPB_OPT_LDPC_NO_BULK 1            /* 1: min-sum check pass without the bulk-copy staged kernel    */
#define CPB_OPT_BCJR_WINDOW 2             /* w > 0: MAP windows of w trellis steps (multiple of 8, 128..1024; default 1024): more
                                             parallelism per frame for small batches, 96-step warm-up either side as always */
#define CPB_OPT_BCJR_PER_STEP_SCALING 3   /* 1: MAP kernel that rescales its metrics every step (the cross-check of the default,
                                             which rescales every 4th step and falls back per block on decay)          */
#define CPB_OPT_TURBO_FRAME_MAJOR 4       /* 1: turbo loop on frame-major arrays with separate interleaver kernels (the cross-check
                                             of the default, which transposes once and indexes rows through the interleaver) */
#define CPB_OPT_TX_FORCE_GENERIC 5        /* 1: cpb_conv_link_tx always runs the bit-serial kernel (cross-check of the word-parallel one) */
#define CPB_OPT_LDPC_ENC_FORCE_DENSE 6    /* 1: the LDPC encoder uses its dense form for a peelable code that fits the dense bound
                                             (cross-check of the peeled form) */
#define CPB_OPT_COUNT 8
int cpb_set_option(int option_id, int value);
int cpb_get_option(int option_id, int *value);

/* element types of decoder inputs */
#define CPB_U8 0
#define CPB_F32 1

/* ---- Trellis descriptor: commpy/channelcoding/convcode.py:23-255 (attributes :119-128) -------- */
typedef struct cpbTrellis cpbTrellis;
/* next_state / output: S x 2^k row-major int32 host tables (Trellis.next_state_table / .output_table). */
int cpb_trellis_create(const int32_t *next_state_host, const int32_t *output_host,
                       int k, int n, int total_memory, int number_states, cpbTrellis **out);
int cpb_trellis_destroy(cpbTrellis *t);
/* 0 = generic table-driven kernels; >0 = id of the register-resident fast path that matched. */
int cpb_trellis_fast_path(const cpbTrellis *t);

/* ---- Viterbi: convcode.py:661-749 viterbi_decode (+ :590-657 _acs_traceback, :575-587 metrics) - */
#define CPB_VITERBI_HARD 0         /* in: CPB_U8 bits {0,1}                                        */
#define CPB_VITERBI_SOFT 1         /* in: CPB_F32 LLRs, positive favours bit 1, clipped to +-500   */
#define CPB_VITERBI_UNQUANTIZED 2  /* in: CPB_F32 symbols, +1 <-> bit 1                            */
/* number of decoded bits per frame, L = int(n_in*k/n) (convcode.py:699), and trellis steps T (:721) */
int cpb_viterbi_sizes(const cpbTrellis *t, int64_t n_in, int64_t *L, int64_t *T);
int cpb_viterbi_workspace_bytes(const cpbTrellis *t, int64_t batch, int64_t n_in, int tb_depth, int mode,
                                size_t *bytes);
/*
 * coded_dev: batch x n_in elements of in_dtype.  out_bits_dev: batch x L uint8 in {0,1}.
 * tb_depth <= 0 selects the reference default min(5*total_memory, L) (:701-702).
 * Output bit p is decided exactly as the reference does: by the (tb_depth-1)-step traceback that starts
 * from the lowest-index best state at step min(p + tb_depth - 1, T).
 * workspace_dev may be NULL (stream-ordered allocation) or >= cpb_viterbi_workspace_bytes().
 */
int cpb_viterbi_decode(const cpbTrellis *t, const void *coded_dev, int in_dtype, int64_t batch, int64_t n_in,
                       int tb_depth, int mode, uint8_t *out_bits_dev,
                       void *workspace_dev, size_t workspace_bytes, void *stream);
/* Host-buffer form (what a CommPy caller has): chunked H2D -> decode -> D2H pipeline on internal streams. */
int cpb_viterbi_decode_host(const cpbTrellis *t, const void *coded_host, int in_dtype, int64_t batch,
                            int64_t n_in, int tb_depth, int mode, uint8_t *out_bits_host);
/*
 * Bit-packed hard decision: 1 bit per coded bit in, 1 bit per decoded bit out, both in numpy.packbits order (element e
 * of a row is bit 7 - (e & 7) of byte e >> 3).  coded_packed: batch x n_in/8 bytes, out_packed: batch x L/8 bytes.
 * Same decision rule as cpb_viterbi_decode(CPB_VITERBI_HARD): 8x less HBM and PCIe traffic for the same answer.
 * CPB_EUNSUPPORTED unless the trellis has a register-resident fast path, n_in % 16 == 0 and (tb_depth - 2) % 4 == 0
 * (the default depth 30 of a K = 7 code qualifies).
 */
int cpb_viterbi_decode_packed(const cpbTrellis *t, const uint8_t *coded_packed_dev, int64_t batch, int64_t n_in,
                              int tb_depth, uint8_t *out_packed_dev, void *stream);
/*
 * Soft / unquantized decision on PUNCTURED rows: depuncturing (convcode.py:777-804) fused into the kernel's load.
 * llr_punct_dev: batch x n_kept float32 (what the demapper produced for the punctured stream); coded position c of the
 * n_depunct-long mother-code stream is the next unread value when punct_vec[c % punct_len] == 1 and 0.0 otherwise;
 * CPB_EINVAL when the row is shorter than the pattern needs (the reference raises IndexError).  punct_len <= 32.
 * Then exactly cpb_viterbi_decode(mode) on the n_depunct values.  K = 7 fast-path trellises; CPB_EUNSUPPORTED otherwise
 * (depuncture with commpy_b200.channelcoding.depuncturing and call cpb_viterbi_decode).
 */
int cpb_viterbi_punctured_workspace_bytes(int64_t batch, size_t *bytes);
int cpb_viterbi_decode_punctured(const cpbTrellis *t, const float *llr_punct_dev, int64_t batch, int64_t n_kept,
                                 const int32_t *punct_vec_host, int punct_len, int64_t n_depunct, int tb_depth, int mode,
                                 uint8_t *out_bits_dev, void *workspace_dev, size_t workspace_bytes, void *stream);
int cpb_viterbi_decode_host_packed(const cpbTrellis *t, const uint8_t *coded_packed_host, int64_t batch,
                                   int64_t n_in, int tb_depth, uint8_t *out_packed_host);

/* ---- BCJR / turbo: commpy/channelcoding/turbo.py:163-251 map_decode, :254-333 turbo_decode ------ */
/*
 * Rate-1/2 (n = 2, k = 1) trellis.  sys/par/L_int: batch x N float32.  mode 1 = 'decode', 0 = 'compute'.
 * L_out (batch x N) receives what the reference returns as L_ext (L_int + log(app1/app0), :145-146);
 * bits_out (nullable) receives L_out > 0 in 'decode' mode, zeros otherwise (:148-152).
 */
int cpb_map_workspace_bytes(const cpbTrellis *t, int64_t batch, int64_t N, size_t *bytes);
int cpb_map_decode(const cpbTrellis *t, const float *sys_dev, const float *par_dev, const float *L_int_dev,
                   int64_t batch, int64_t N, float noise_variance, int mode,
                   float *L_out_dev, uint8_t *bits_out_dev, void *workspace_dev, size_t workspace_bytes, void *stream);
/*
 * perm_dev: interleaver p_array (int32, length N; interleavers.py:13-47).  L_int0_dev nullable (zeros).
 * bits_out: batch x N uint8 = deinterlv(decoder-2 hard decisions of the last iteration) (:331).
 * workspace_dev (both functions) may be NULL (stream-ordered allocation) or >= cpb_*_workspace_bytes().
 */
int cpb_turbo_workspace_bytes(const cpbTrellis *t, int64_t batch, int64_t N, size_t *bytes);
int cpb_turbo_decode(const cpbTrellis *t, const float *sys_dev, const float *par1_dev, const float *par2_dev,
                     const int32_t *perm_dev, int64_t batch, int64_t N, float noise_variance, int n_iter,
                     const float *L_int0_dev, uint8_t *bits_out_dev, void *workspace_dev, size_t workspace_bytes,
                     void *stream);
/* Host-buffer forms: chunked H2D -> kernels -> D2H pipeline on the trellis handle's internal streams; every pointer is
 * host memory (perm_host included); L_out_host / bits_out_host nullable for cpb_map_decode_host. */
int cpb_map_decode_host(const cpbTrellis *t, const float *sys_host, const float *par_host, const float *L_int_host,
                        int64_t batch, int64_t N, float noise_variance, int mode, float *L_out_host, uint8_t *bits_out_host);
int cpb_turbo_decode_host(const cpbTrellis *t, const float *sys_host, const float *par1_host, const float *par2_host,
                          const int32_t *perm_host, int64_t batch, int64_t N, float noise_variance, int n_iter,
                          const float *L_int0_host, uint8_t *bits_out_host);

/* ---- LDPC min-sum BP: commpy/channelcoding/ldpc.py:144-254 (MSA branch :229-238, VN :243-248) ---- */
typedef struct cpbLdpc cpbLdpc;
/* H in CSR (row = check node): row_ptr[m+1], col_idx[nnz], host int32.  n = n_vnodes, m = n_cnodes. */
int cpb_ldpc_create(const int32_t *row_ptr_host, const int32_t *col_idx_host, int m, int n, cpbLdpc **out);
int cpb_ldpc_destroy(cpbLdpc *h);
int cpb_ldpc_workspace_bytes(const cpbLdpc *h, int64_t batch, int precision, size_t *bytes);
#define CPB_LDPC_FP32 0   /* float32 messages (throughput mode)                                      */
#define CPB_LDPC_FP64 1   /* float64 messages, reference summation order: bit-exact with the reference */
/*
 * llr_dev: batch x n, float32 (FP32) or float64 (FP64) -- clipped IN PLACE to +-500 like ldpc.py:186.
 * LLR sign convention of the reference: bit = signbit(llr) (:193).  Flooding schedule, syndrome check
 * before every iteration (:205), at most n_iters iterations per block.
 * dec_dev: batch x n uint8.  out_llr_dev (nullable): batch x n, same type as llr.  iters_dev (nullable):
 * batch int32, iterations executed per block.
 */
int cpb_ldpc_minsum(const cpbLdpc *h, void *llr_dev, int precision, int64_t batch, int n_iters,
                    uint8_t *dec_dev, void *out_llr_dev, int32_t *iters_dev,
                    void *workspace_dev, size_t workspace_bytes, void *stream);

/* Host-buffer form of cpb_ldpc_minsum / cpb_ldpc_sumproduct (algorithm 0 = MSA, 1 = SPA): llr_host is clipped in
 * place like the device form; dec_host batch x n uint8; out_llr_host / iters_host nullable. */
int cpb_ldpc_decode_host(const cpbLdpc *h, int algorithm, void *llr_host, int precision, int64_t batch, int n_iters,
                         uint8_t *dec_host, void *out_llr_host, int32_t *iters_host);

/* Sum-product variant ('SPA', ldpc.py:209-227): same arguments and schedule; check-node rule
 * R_ij = 2 atanh(clip(prod_row tanh(Q/2) / tanh(Q_ij/2), -1, 1)), clipped to +-500, evaluated in double for both
 * precisions (fp32 messages saturate at ~37.4, as the reference's do).  Agrees with the reference within the
 * conditioning of atanh near +-1 (the reference forms the product through complex log2/exp2), not bit for bit. */
int cpb_ldpc_sumproduct(const cpbLdpc *h, void *llr_dev, int precision, int64_t batch, int n_iters,
                        uint8_t *dec_dev, void *out_llr_dev, int32_t *iters_dev,
                        void *workspace_dev, size_t workspace_bytes, void *stream);

/* ---- Soft / hard demapper: commpy/modulation.py:100-141 Modem.demodulate ------------------------ */
typedef struct cpbModem cpbModem;
/* constellation: M complex points as interleaved (re, im) float64 host values, index k <-> bits MSB first. */
int cpb_modem_create(const double *constellation_host, int M, cpbModem **out);
int cpb_modem_destroy(cpbModem *m);
/* 1 when the constellation factors as pam_I[k_hi] + j*pam_Q[k_lo] (square Gray QAM): 2*sqrt(M) exps/symbol. */
int cpb_modem_is_separable(const cpbModem *m);
/*
 * y_dev: n_sym complex64 (interleaved re, im).  llr_dev: n_sym x log2(M) float32, MSB first,
 * LLR = log sum_{k: bit=1} exp(-|y-c_k|^2/noise_var) - log sum_{k: bit=0} ... (exact log-sum-exp, :127-137).
 */
int cpb_demod_soft(const cpbModem *m, const float *y_dev, int64_t n_sym, float noise_var,
                   float *llr_dev, void *stream);
/* Host-buffer form: y_host n_sym complex64, llr_host n_sym x log2(M) float32. */
int cpb_demod_soft_host(const cpbModem *m, const float *y_host, int64_t n_sym, float noise_var, float *llr_host);
/* bits_dev: n_sym x log2(M) uint8, nearest point (first minimum), MSB first (:121-123). */
int cpb_demod_hard(const cpbModem *m, const float *y_dev, int64_t n_sym, uint8_t *bits_dev, void *stream);
/*
 * Channel-aware forms for flat fading: h_dev holds n_sym complex64 gains, one per symbol, and the distances are
 * |y - h c_k|^2.  The LLRs equal the reference's demodulate(y/h, 'soft', noise_var/|h|^2) symbol by symbol, without
 * dividing by h: finite in deep fades, exactly 0 where |h|^2 is 0 (hard decision: index 0 there).  With h = 1 the output
 * equals cpb_demod_soft / cpb_demod_hard bit for bit.
 */
int cpb_demod_soft_csi(const cpbModem *m, const float *y_dev, const float *h_dev, int64_t n_sym, float noise_var,
                       float *llr_dev, void *stream);
int cpb_demod_hard_csi(const cpbModem *m, const float *y_dev, const float *h_dev, int64_t n_sym, uint8_t *bits_dev,
                       void *stream);

/* ---- error counting: commpy/links.py:335-337 (and :253-256) ------------------------------------- */
/* counters_dev[0] += # differing bits, counters_dev[1] += # frames with >= 1 differing bit (int64, device). */
int cpb_count_errors(const uint8_t *a_dev, const uint8_t *b_dev, int64_t batch, int64_t L,
                     int64_t lda, int64_t ldb, int64_t *counters_dev, void *stream);

/* ---- transmit side of a coded AWGN link, generated on the device: commpy/links.py:318-329 (per-frame loop of
 * link_performance: random message, conv_encode 'cont' convcode.py:475-558, Modem.modulate modulation.py:79-98,
 * AWGN channels.py:181-221) -- the caller of the hot path, so that 1e8-symbol BER points never touch the host. ---- */
/*
 * k = 1 feed-forward trellis (else CPB_EUNSUPPORTED), frame_bits information bits per frame ('cont' termination),
 * frame_bits * n must be a multiple of the modem's bits per symbol.  Counter-based randomness (Philox4x32-10, key =
 * seed, counter = global frame id = first_frame + local index): the output does not depend on how frames are split
 * over calls or GPUs.  msg_dev: frames x frame_bits uint8.  y_dev: frames x (frame_bits*n/bits_per_symbol) complex64
 * = constellation point + noise_sigma * (N(0,1) + j N(0,1)).
 */
int cpb_conv_link_tx(const cpbTrellis *t, const cpbModem *m, int64_t frames, int64_t frame_bits, uint64_t seed,
                     int64_t first_frame, float noise_sigma, uint8_t *msg_dev, float *y_dev, void *stream);
/* The same with puncturing (convcode.py:752-774) between the encoder and the mapper: coded bit c is kept when
 * punct_vec[c % punct_len] == 1 (punct_len a multiple of n, <= 32); the kept bits of a frame must fill whole symbols.
 * y_dev: frames x (kept bits / bits per symbol) complex64. */
int cpb_conv_link_tx_punctured(const cpbTrellis *t, const cpbModem *m, int64_t frames, int64_t frame_bits,
                               uint64_t seed, int64_t first_frame, float noise_sigma,
                               const int32_t *punct_vec_host, int punct_len, uint8_t *msg_dev, float *y_dev,
                               void *stream);
/* The same over a flat-fading SISO channel (SISOFlatChannel, channels.py:176-221): symbol s gets its own gain
 * h = (los_re + j los_im) + sqrt(nlos_var / 2) (N(0,1) + j N(0,1)) (Philox counter word 5) and y = h * point + noise, the
 * noise stream being that of cpb_conv_link_tx.  h_dev: frames x nsym complex64, laid out like y_dev.  punct_vec_host may be
 * NULL (no puncturing).  With los = 1, nlos_var = 0 the message and y equal cpb_conv_link_tx[_punctured] bit for bit. */
int cpb_conv_link_tx_fading(const cpbTrellis *t, const cpbModem *m, int64_t frames, int64_t frame_bits, uint64_t seed,
                            int64_t first_frame, float noise_sigma, float los_re, float los_im, float nlos_var,
                            const int32_t *punct_vec_host, int punct_len,
                            uint8_t *msg_dev, float *y_dev, float *h_dev, void *stream);

/* ---- transmit side of a turbo-coded BPSK-AWGN link: commpy/channelcoding/turbo.py:14-59 (turbo_encode) + mapper + AWGN ---- */
/*
 * Rate-1/2 systematic trellis (k = 1, n = 2, MSB of the output symbol = input; <= 32 states), the same for both component
 * encoders like turbo_decode assumes.  Per frame: msg (Philox bits), sys = msg, par1 = parity over msg, par2 = parity over
 * msg[perm] -- the streams turbo_encode returns (its zero-bit 'rsc' tails are cut off again, :55-57: unterminated
 * encoders started in state 0) -- each mapped to 2x-1 and disturbed by noise_sigma * N(0,1).
 * msg_dev: frames x N uint8; sys / par1 / par2: frames x N float32.  Counter-based randomness keyed by (seed, global frame).
 */
int cpb_turbo_link_tx(const cpbTrellis *t, const int32_t *perm_dev, int64_t frames, int64_t N, uint64_t seed,
                      int64_t first_frame, float noise_sigma, uint8_t *msg_dev, float *sys_dev, float *par1_dev,
                      float *par2_dev, void *stream);
/* The same over SISO flat fading (SISOFlatChannel, channels.py:176-221), receiver CSI included: value t of stream j
 * (0 = sys, 1 = par1, 2 = par2) is received as y = h x + noise_sigma (N(0,1) + j N(0,1)), x = 2 bit - 1, with its own gain
 * h = (mean_re + j mean_im) + sqrt(nlos / 2) (N(0,1) + j N(0,1)).  Re of the noise is cpb_turbo_link_tx's noise; the
 * imaginary noise and the gains come from Philox counter words 5 + j and 8 + j.  y_dev, h_dev: [3][frames][N] complex64
 * (stream-major: stream j is a contiguous frames x N block).  With mean = 1, nlos = 0 the message and Re(y) equal
 * cpb_turbo_link_tx's outputs bit for bit and h = 1.  CPB_EINVAL also for nlos < 0 or non-finite parameters. */
int cpb_turbo_link_tx_fading(const cpbTrellis *t, const int32_t *perm_dev, int64_t frames, int64_t N, uint64_t seed,
                             int64_t first_frame, float noise_sigma, float mean_re, float mean_im, float nlos,
                             uint8_t *msg_dev, float *y_dev, float *h_dev, void *stream);
/* Coherent BPSK combining: s[i] = Re(conj(h[i]) y[i]) = h_re y_re + h_im y_im (one fused multiply-add after one product),
 * y_dev, h_dev: n complex64, s_dev: n float32.  s is |h|^2 x + N(0, sigma^2 |h|^2) for y = h x + sigma (n_re + j n_im), so
 * cpb_map_decode / cpb_turbo_decode take s with noise_variance = sigma^2 and decode exactly.  s = Re(y) where h = 1 + 0j,
 * 0 where h = 0. */
int cpb_bpsk_combine(const float *y_dev, const float *h_dev, int64_t n, float *s_dev, void *stream);
/* The same turbo code over a modem (bit-interleaved coded modulation without a channel interleaver): per frame the code word
 * c = [sys | par1 | par2] (3N bits, the streams of cpb_turbo_link_tx, sys = msg) is mapped bits_per_symbol at a time MSB
 * first (Modem.modulate) and disturbed by noise_sigma (N(0,1) + j N(0,1)) per symbol.  The message is cpb_turbo_link_tx's
 * (counter word 0) bit for bit; the noise is Philox counter word 1, as in cpb_conv_link_tx.  msg_dev: frames x N uint8;
 * y_dev: frames x (3N / bits_per_symbol) complex64.  CPB_EINVAL for null pointers, N < 1, first_frame < 0 and
 * 3N % bits_per_symbol != 0; CPB_EUNSUPPORTED for a trellis cpb_turbo_link_tx refuses. */
int cpb_turbo_link_tx_modem(const cpbTrellis *t, const cpbModem *modem, const int32_t *perm_dev, int64_t frames, int64_t N,
                            uint64_t seed, int64_t first_frame, float noise_sigma, uint8_t *msg_dev, float *y_dev, void *stream);
/* The same over SISO flat fading: symbol s gets its own gain h = (mean_re + j mean_im) + sqrt(nlos / 2) (N(0,1) + j N(0,1))
 * (counter word 5, as cpb_conv_link_tx_fading) and y = h * point + noise.  h_dev: laid out like y_dev.  With mean = 1,
 * nlos = 0 the message and y equal cpb_turbo_link_tx_modem's bit for bit.  CPB_EINVAL also for nlos < 0 or non-finite
 * parameters. */
int cpb_turbo_link_tx_modem_fading(const cpbTrellis *t, const cpbModem *modem, const int32_t *perm_dev, int64_t frames,
                                   int64_t N, uint64_t seed, int64_t first_frame, float noise_sigma, float mean_re, float mean_im,
                                   float nlos, uint8_t *msg_dev, float *y_dev, float *h_dev, void *stream);

/* ---- LDPC systematic encoding and the transmit side of an LDPC-coded link: commpy/channelcoding/ldpc.py:302-354
 * (triang_ldpc_systematic_encode) + Modem.modulate + AWGN / SISO flat fading (channels.py:176-221) ---- */
/*
 * Code words are laid out as the reference lays them out: [message (k = n - m bits) | parity (m bits)], H c = 0 over GF(2).
 * The encoder plan is built from the handle's H on first use and freed with the handle:
 *   peeled form when the parity part H_p = H[:, k:] peels completely (each parity bit solved in turn from one row);
 *   dense form P = H_p^-1 H_s (GF(2)) when H_p is invertible and k * m <= 2^26.
 * CPB_EINVAL: H_p singular over GF(2).  CPB_EUNSUPPORTED: H_p does not peel and k * m > 2^26.
 * CPB_OPT_LDPC_ENC_FORCE_DENSE selects the dense form for a peelable code that fits the bound.
 * msg_dev: batch x k uint8 in {0, 1} (any nonzero byte is taken as 1); cw_dev: batch x n uint8.
 */
int cpb_ldpc_encode(const cpbLdpc *h, const uint8_t *msg_dev, int64_t batch, uint8_t *cw_dev, void *stream);
/* Host-only description of the plan cpb_ldpc_encode builds for H (CSR as in cpb_ldpc_create; no device is used), same
 * status codes.  form: 0 = peeled, 1 = dense.  order_host / pivot_host (nullable, m entries each): step t solves parity
 * bit pivot[t] from row order[t] (dense: the identity).  P_host (nullable, dense only): m rows of ceil(k / 32) uint32
 * words, bit j of row i = word j / 32, bit j % 32. */
int cpb_ldpc_encoder_plan(const int32_t *row_ptr_host, const int32_t *col_idx_host, int m, int n, int force_dense, int *form,
                          int32_t *order_host, int32_t *pivot_host, uint32_t *P_host);
/*
 * Per frame: k message bits from Philox (counter word 0, as cpb_conv_link_tx), encoded as cpb_ldpc_encode does, mapped
 * bits_per_symbol at a time MSB first (Modem.modulate), + noise_sigma (N(0,1) + j N(0,1)) per symbol (counter word 1, as
 * cpb_conv_link_tx).  Randomness keyed by (seed, global frame = first_frame + local index).  msg_dev: frames x k uint8;
 * y_dev: frames x (n / bits_per_symbol) complex64.  CPB_EINVAL when n is not a multiple of bits_per_symbol.
 */
int cpb_ldpc_link_tx(const cpbLdpc *h, const cpbModem *modem, int64_t frames, uint64_t seed, int64_t first_frame,
                     float noise_sigma, uint8_t *msg_dev, float *y_dev, void *stream);
/* The same over SISO flat fading: symbol s gets its own gain h = (mean_re + j mean_im) + sqrt(nlos / 2) (N(0,1) + j N(0,1))
 * (counter word 5, as cpb_conv_link_tx_fading) and y = h * point + noise.  h_dev: laid out like y_dev.  With mean = 1,
 * nlos = 0 the message and y equal cpb_ldpc_link_tx's bit for bit.  CPB_EINVAL also for nlos < 0 or non-finite parameters. */
int cpb_ldpc_link_tx_fading(const cpbLdpc *h, const cpbModem *modem, int64_t frames, uint64_t seed, int64_t first_frame,
                            float noise_sigma, float mean_re, float mean_im, float nlos, uint8_t *msg_dev, float *y_dev,
                            float *h_dev, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* COMMPY_B200_H */

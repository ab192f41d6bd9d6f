"""Monte-Carlo link simulation around the GPU decoding path (next row of SURVEY.md section 8f).

* `LinkModel` / `link_performance` keep the reference's sequential, callable-driven loop and signature
  (commpy/links.py:29-64, :269-342) -- host logic only, the callables it is given do the work (e.g. this
  package's `Modem.demodulate` and `viterbi_decode`).
* `AwgnSisoChannel` is the one channel convention the decoding path needs to synthesise its inputs
  (commpy/channels.py:53,74: `noise_std = sqrt((isComplex+1)*nb_tx*Es / (rate*10^(SNR/10)))`, complex noise
  `(N(0,1) + jN(0,1)) * noise_std * 0.5`).  Host-side fading channels are in `channels`.
* `ConvLinkGPU` is the batched form for config C5: random bits -> convolutional encoder -> Modem.modulate ->
  AWGN generated on the device by one CUDA kernel (`conv_link_tx` -> cpb_conv_link_tx, counter-based Philox
  randomness keyed by the GLOBAL frame index), then this package's demapper, Viterbi decoder and error
  counter; frames shard over ranks and the error counters are all-reduced so every rank takes the same
  stop decision (`links.py:313`).  With `fading_param` the batched link runs over SISO flat fading instead
  (`conv_link_tx_fading` -> cpb_conv_link_tx_fading, one gain per symbol as `channels.SISOFlatChannel` draws them), and
  the demapper uses the gains (cpb_demod_soft_csi / cpb_demod_hard_csi).
* `TurboLinkGPU` is the batched rate-1/3 turbo link over BPSK (`turbo_link_tx` -> cpb_turbo_link_tx, the turbo decoder,
  the error counter).  With `fading_param` it runs over SISO flat fading (`turbo_link_tx_fading` ->
  cpb_turbo_link_tx_fading, one gain per coded bit), and the receiver combines coherently (`bpsk_combine` ->
  cpb_bpsk_combine, s = Re(conj(h) y)) before the unchanged turbo decoder.  With `modem` the code word [sys | par1 | par2]
  is mapped onto that modem (`turbo_link_tx_modem[_fading]` -> cpb_turbo_link_tx_modem[_fading]), and the receiver hands
  the demapper's exact LLRs to the same turbo decoder.
* `LdpcLinkGPU` is the batched LDPC-coded link (`ldpc_link_tx[_fading]` -> cpb_ldpc_link_tx[_fading]: Philox message,
  systematic encoder planned from H, Modem.modulate, AWGN or flat fading), then the demapper, the LDPC decoder and the
  error counter over the message bits.
"""
import math
from fractions import Fraction
from inspect import getfullargspec

import numpy as np

from . import _lib, parallel

__all__ = ["link_performance", "LinkModel", "AwgnSisoChannel", "ConvLinkGPU", "conv_link_tx", "conv_link_tx_fading",
           "turbo_link_tx_fading", "turbo_link_tx_modem", "turbo_link_tx_modem_fading", "bpsk_combine", "idd_decoder", "LdpcLinkGPU", "ldpc_link_tx", "ldpc_link_tx_fading"]


class AwgnSisoChannel:
    """SISO AWGN channel with the reference's SNR convention (channels.py:37-93, :181-221 with fading (1+0j, 0))."""

    nb_tx = 1
    nb_rx = 1

    def __init__(self, is_complex=True, rng=None):
        self.isComplex = bool(is_complex)
        self.noise_std = None
        self.channel_gains = 1.0
        self.rng = rng if rng is not None else np.random

    def set_SNR_dB(self, SNR_dB, code_rate=1, Es=1):
        self.noise_std = math.sqrt((self.isComplex + 1) * self.nb_tx * Es / (code_rate * 10 ** (SNR_dB / 10)))

    def generate_noises(self, dims):
        if self.isComplex:
            return (self.rng.standard_normal(dims) + 1j * self.rng.standard_normal(dims)) * self.noise_std * 0.5
        return self.rng.standard_normal(dims) * self.noise_std

    def propagate(self, msg):
        msg = np.asarray(msg)
        self.noises = self.generate_noises(len(msg))
        # SISOFlatChannel draws its fading variates after the noise even when their variance is zero
        # (channels.py:213-217); the same draws are made and discarded here so that a seeded run consumes the random
        # stream exactly like the reference with fading_param = (1 + 0j, 0j) and reproduces its BERs to the last digit.
        self.rng.standard_normal(len(msg))
        if self.isComplex:
            self.rng.standard_normal(len(msg))
        self.channel_gains = np.ones(len(msg), dtype=complex if self.isComplex else float)
        self.unnoisy_output = msg
        return msg + self.noises


def link_performance(link_model, SNRs, send_max, err_min, send_chunk=None, code_rate=1):
    """Same as `link_model.link_performance(...)` (links.py:29-64)."""
    if not send_chunk:
        send_chunk = err_min
    return link_model.link_performance(SNRs, send_max, err_min, send_chunk, code_rate)


class LinkModel:
    """Link model built from callables, as in the reference (links.py:67-153):
    `modulate(bits) -> symbols`, `channel` (set_SNR_dB / propagate / channel_gains / noise_std / nb_tx),
    `receive(y, H, constellation, noise_var) -> bits or LLRs`, `decoder(array)` or the 6-argument form
    `decoder(y, H, constellation, noise_var, array, bits_per_send)` chosen by arity (links.py:306)."""

    def __init__(self, modulate, channel, receive, num_bits_symbol, constellation, Es=1, decoder=None, rate=Fraction(1, 1),
                 number_chunks_per_send=1, stop_on_surpass_error=True):
        self.modulate = modulate
        self.channel = channel
        self.receive = receive
        self.num_bits_symbol = num_bits_symbol
        self.constellation = constellation
        self.Es = Es
        self.rate = rate
        self.number_chunks_per_send = number_chunks_per_send
        self.stop_on_surpass_error = stop_on_surpass_error
        self.decoder = (lambda msg: msg) if decoder is None else decoder
        self.full_simulation_results = None

    def link_performance(self, SNRs, send_max, err_min, send_chunk=None, code_rate=1):
        """Sequential Monte-Carlo BER estimate, one chunk per iteration (links.py:269-342)."""
        BERs = np.zeros_like(SNRs, dtype=float)
        if send_chunk is None:
            send_chunk = err_min
        if type(code_rate) is float:
            code_rate = Fraction(code_rate).limit_denominator(100)
        self.rate = code_rate
        divider = (Fraction(1, self.num_bits_symbol * self.channel.nb_tx) * 1 / code_rate).denominator
        send_chunk = max(divider, send_chunk // divider * divider)
        receive_size = self.channel.nb_tx * self.num_bits_symbol
        full_args_decoder = len(getfullargspec(self.decoder).args) > 1
        for i, snr in enumerate(SNRs):
            self.channel.set_SNR_dB(snr, float(code_rate), self.Es)
            bit_send = 0
            bit_err = 0
            while bit_send < send_max and bit_err < err_min:
                msg = np.random.choice((0, 1), send_chunk)
                y = self.channel.propagate(self.modulate(msg))
                nv = self.channel.noise_std ** 2
                if np.ndim(y) > 1:           # one received vector per channel use (MIMO-shaped channels)
                    received = np.empty(int(math.ceil(len(msg) / float(self.rate))))
                    for j in range(len(y)):
                        received[receive_size * j:receive_size * (j + 1)] = \
                            self.receive(y[j], self.channel.channel_gains[j], self.constellation, nv)
                else:
                    received = self.receive(y, self.channel.channel_gains, self.constellation, nv)
                if full_args_decoder:
                    decoded = self.decoder(y, self.channel.channel_gains, self.constellation, nv, received,
                                           self.channel.nb_tx * self.num_bits_symbol)
                else:
                    decoded = self.decoder(received)
                bit_err += np.bitwise_xor(msg, np.asarray(decoded)[:len(msg)].astype(int)).sum()
                bit_send += send_chunk
            BERs[i] = bit_err / bit_send
            if bit_err < err_min:
                break
        return BERs


    def _one_transmission(self, msg, receive_size, full_args_decoder):
        y = self.channel.propagate(self.modulate(msg))
        nv = self.channel.noise_std ** 2
        if np.ndim(y) > 1:
            received = np.empty(int(math.ceil(len(msg) / float(self.rate))))
            for j in range(len(y)):
                received[receive_size * j:receive_size * (j + 1)] = \
                    self.receive(y[j], self.channel.channel_gains[j], self.constellation, nv)
        else:
            received = self.receive(y, self.channel.channel_gains, self.constellation, nv)
        if full_args_decoder:
            return self.decoder(y, self.channel.channel_gains, self.constellation, nv, received,
                                self.channel.nb_tx * self.num_bits_symbol)
        return self.decoder(received)

    def link_performance_full_metrics(self, SNRs, tx_max, err_min, send_chunk=None, code_rate=1,
                                      number_chunks_per_send=1, stop_on_surpass_error=True):
        """Per-transmission metrics (links.py:155-267): returns (BERs, BEs, CEs, NCs) and caches them on
        `full_simulation_results`.  A transmission carries `number_chunks_per_send` chunks encoded and decoded as ONE
        stream (:229-230, :250); errors are then counted per chunk (:252-256)."""
        BERs = np.zeros_like(SNRs, dtype=float)
        BEs = np.zeros((len(SNRs), tx_max), dtype=int)
        CEs = np.zeros((len(SNRs), tx_max), dtype=int)
        NCs = np.zeros((len(SNRs), tx_max), dtype=int)
        if send_chunk is None:
            send_chunk = err_min
        if type(code_rate) is float:
            code_rate = Fraction(code_rate).limit_denominator(100)
        self.rate = code_rate
        divider = (Fraction(1, self.num_bits_symbol * self.channel.nb_tx) * 1 / code_rate).denominator
        send_chunk = max(divider, send_chunk // divider * divider)
        receive_size = self.channel.nb_tx * self.num_bits_symbol
        full_args_decoder = len(getfullargspec(self.decoder).args) > 1
        for i, snr in enumerate(SNRs):
            self.channel.set_SNR_dB(snr, float(code_rate), self.Es)
            sent = 0
            bit_err = np.zeros(tx_max, dtype=int)
            chunk_count = np.zeros(tx_max, dtype=int)
            for tx in range(tx_max):
                if stop_on_surpass_error and bit_err.sum() > err_min:
                    break
                msg = np.random.choice((0, 1), send_chunk * number_chunks_per_send)
                decoded = np.asarray(self._one_transmission(msg, receive_size, full_args_decoder))
                for c in range(number_chunks_per_send):
                    sl = slice(send_chunk * c, send_chunk * (c + 1))
                    bit_err[tx] += np.bitwise_xor(msg[sl], decoded[sl].astype(int)).sum()
                chunk_count[tx] += number_chunks_per_send
                sent += 1
            BERs[i] = bit_err.sum() / (sent * send_chunk)
            BEs[i] = bit_err
            CEs[i] = np.where(bit_err > 0, 1, 0)
            NCs[i] = chunk_count
            if BEs[i].sum() < err_min:
                break
        self.full_simulation_results = BERs, BEs, CEs, NCs
        return BERs, BEs, CEs, NCs


def _ff_taps(trellis):
    """Generator taps (delay 0 = current input) of a k=1 feed-forward shift-register trellis, or None."""
    if trellis.k != 1:
        return None
    M, n = trellis.total_memory, trellis.n
    nst, otab = np.asarray(trellis.next_state_table), np.asarray(trellis.output_table)
    S = trellis.number_states
    for s in range(S):
        for u in range(2):
            if nst[s, u] != ((u << (M - 1)) | (s >> 1)):
                return None
    taps = np.zeros((n, M + 1), dtype=np.int64)
    for j in range(n):
        taps[j, 0] = (otab[0, 1] >> (n - 1 - j)) & 1
        for b in range(1, M + 1):
            taps[j, b] = (otab[1 << (M - b), 0] >> (n - 1 - j)) & 1
    for s in range(S):          # the code must be linear in (state, input) for the tap form to hold
        for u in range(2):
            regs = [u] + [(s >> (M - b)) & 1 for b in range(1, M + 1)]
            sym = 0
            for j in range(n):
                sym = (sym << 1) | (int(np.dot(taps[j], regs)) & 1)
            if sym != otab[s, u]:
                return None
    return taps


def conv_link_tx(trellis, modem, frames, frame_bits, seed, first_frame, noise_sigma, puncture=None):
    """Device-side TX chain of `frames` frames starting at GLOBAL frame index `first_frame`: random message ->
    conv_encode(..., 'cont') -> [puncturing(coded, puncture)] -> modem.modulate -> + noise_sigma * (N(0,1) + jN(0,1)).

    Returns (msg uint8 (frames, frame_bits), y complex64 (frames, frame_bits*n/bits_per_symbol)) as CUDA tensors.
    The streams depend only on (seed, global frame index): any split of the frames over calls or ranks gives the
    same frames."""
    return _conv_link_tx(trellis, modem, frames, frame_bits, seed, first_frame, noise_sigma, None, puncture)


def _fading(fading_param):
    """(mean gain, scattered power) of a SISOFlatChannel fading_param, checked like the reference checks it (ValueError when
    the channel would add or remove energy); a real-valued channel raises NotImplementedError (the device link is complex
    baseband)."""
    from .channels import SISOFlatChannel
    ch = SISOFlatChannel(fading_param=fading_param)
    if not ch.isComplex:
        raise NotImplementedError("the GPU link is complex baseband: fading_param[0] must be complex, e.g. (0j, 1)")
    return complex(fading_param[0]), float(np.real(fading_param[1]))


def conv_link_tx_fading(trellis, modem, frames, frame_bits, seed, first_frame, noise_sigma, fading_param, puncture=None):
    """`conv_link_tx` over SISO flat fading (SISOFlatChannel, channels.py:176-221): each symbol c is received as
    y = h c + noise_sigma * (N(0,1) + jN(0,1)) with its own gain h = fading_param[0] + sqrt(fading_param[1] / 2) *
    (N(0,1) + jN(0,1)), e.g. (0j, 1) for Rayleigh and (m, 1 - |m|^2) for Rician fading.  The message and the noise are
    the streams of `conv_link_tx` (at fading_param = (1 + 0j, 0) the outputs are identical to it).

    Returns (msg uint8 (frames, frame_bits), y complex64 (frames, nsym), h complex64 (frames, nsym)) as CUDA tensors."""
    return _conv_link_tx(trellis, modem, frames, frame_bits, seed, first_frame, noise_sigma, fading_param, puncture)


def _conv_link_tx(trellis, modem, frames, frame_bits, seed, first_frame, noise_sigma, fading_param, puncture):
    """conv_link_tx (fading_param None: AWGN, (msg, y)) and conv_link_tx_fading ((msg, y, h)).  AWGN calls the AWGN entry
    points, which launch the kernels without the fading code."""
    import ctypes as C
    from .channelcoding.convcode import _trellis_handle
    if fading_param is not None:
        mean, nlos = _fading(fading_param)
    torch = _lib.require_cuda()
    nb = int(modem.num_bits_symbol)
    kept = kept_bits(int(trellis.n) * int(frame_bits), puncture)
    if kept % nb:
        raise ValueError("the (punctured) coded bits of a frame must fill whole symbols")
    frames, frame_bits = int(frames), int(frame_bits)
    msg = torch.empty((frames, frame_bits), dtype=torch.uint8, device="cuda")
    y = torch.empty((frames, kept // nb), dtype=torch.complex64, device="cuda")
    pv = None if puncture is None else np.ascontiguousarray(puncture, dtype=np.int32)
    lib = _lib.load()
    head = (_trellis_handle(trellis), modem._handle(), C.c_int64(frames), C.c_int64(frame_bits),
            C.c_uint64(int(seed) & ((1 << 64) - 1)), C.c_int64(int(first_frame)), C.c_float(float(noise_sigma)))
    if fading_param is not None:
        h = torch.empty_like(y)
        rc = lib.cpb_conv_link_tx_fading(*head, C.c_float(mean.real), C.c_float(mean.imag), C.c_float(nlos), _lib.ptr(pv),
                                         0 if pv is None else len(pv), _lib.ptr(msg), _lib.ptr(y), _lib.ptr(h),
                                         _lib.stream_ptr(torch))
        _lib.check(rc, "conv_link_tx_fading")
        return msg, y, h
    if pv is None:
        rc = lib.cpb_conv_link_tx(*head, _lib.ptr(msg), _lib.ptr(y), _lib.stream_ptr(torch))
    else:
        rc = lib.cpb_conv_link_tx_punctured(*head, _lib.ptr(pv), len(pv), _lib.ptr(msg), _lib.ptr(y), _lib.stream_ptr(torch))
    _lib.check(rc, "conv_link_tx")
    return msg, y


def _count_errors(dec, msg, counters, torch):
    """cpb_count_errors: adds the bit errors and the frames with an error of the decoded rows `dec` against the first
    msg.shape[1] bits of each row to `counters` (device side, no sync)"""
    import ctypes as C
    L = msg.shape[1]
    rc = _lib.load().cpb_count_errors(_lib.ptr(dec), _lib.ptr(msg), C.c_int64(msg.shape[0]), C.c_int64(L),
                                      C.c_int64(dec.shape[1]), C.c_int64(L), _lib.ptr(counters), _lib.stream_ptr(torch))
    _lib.check(rc, "count_errors")


def kept_bits(n_coded, puncture):
    """how many of n_coded bits puncturing(message, puncture) keeps (convcode.py:752-774)"""
    if puncture is None:
        return int(n_coded)
    pv = np.asarray(puncture)
    return int(np.sum(pv[np.arange(int(n_coded)) % len(pv)] == 1))


class ConvLinkGPU:
    """Batched convolutional-code link over AWGN on the GPU(s): TX chain and RX chain in this package's CUDA.

    Parameters: `trellis` (k=1 feed-forward, e.g. the K=7 (0o133,0o171) code), `modem` (commpy_b200 Modem),
    `frame_bits` information bits per frame ('cont' termination), `frames_per_batch` frames decoded per step and rank.
    `fading_param` (a SISOFlatChannel fading_param with a complex mean, e.g. (0j, 1) for Rayleigh): the link runs over
    i.i.d. flat fading, one gain per symbol, known to the receiver's demapper; None: AWGN.
    """

    def __init__(self, trellis, modem, frame_bits=4096, frames_per_batch=4096, decoding_type="soft", tb_depth=None, seed=0,
                 puncture=None, fading_param=None):
        self.fading_param = fading_param
        if fading_param is not None:
            _fading(fading_param)
        taps = _ff_taps(trellis)
        if taps is None:
            raise NotImplementedError("ConvLinkGPU generates frames on the device for k=1 feed-forward codes only")
        if decoding_type not in ("soft", "hard"):
            raise ValueError("decoding_type must be 'soft' or 'hard'")
        self.trellis, self.modem, self.taps = trellis, modem, taps
        self.frame_bits, self.frames = int(frame_bits), int(frames_per_batch)
        self.decoding_type, self.tb_depth, self.seed = decoding_type, tb_depth, int(seed)
        nb = modem.num_bits_symbol
        # puncturing pattern over the coded stream (802.11: [1,1,1,0] = 2/3, [1,1,1,0,0,1] = 3/4, ...): punctured on the
        # device in the TX kernel, depunctured inside the Viterbi kernel's load
        self.puncture = None if puncture is None else [int(v) for v in puncture]
        if self.puncture is not None and decoding_type != "soft":
            raise ValueError("a punctured link decodes soft values")
        n_coded = trellis.n * self.frame_bits
        kept = kept_bits(n_coded, self.puncture)
        if kept % nb:
            raise ValueError("the (punctured) coded bits of a frame must fill whole symbols")
        self.rate = Fraction(trellis.k, trellis.n) * Fraction(n_coded, kept)

    # -- TX chain on the device ---------------------------------------------------------------------
    def noise_std(self, snr_db):
        """channels.py:74: noise_std = sqrt(2 Es / (rate 10^(SNR/10))); each real component gets noise_std / 2."""
        return math.sqrt(2 * self.modem.Es / (float(self.rate) * 10 ** (snr_db / 10)))

    def make_batch(self, snr_db, batch_index, torch=None):
        """(msg bits, received symbols, noise_var) for one batch of this rank -- everything stays on the device -- and,
        over fading, the channel gains as a fourth element.
        Batch `batch_index` of rank r covers the global frames [(batch_index*world + r) * frames, ... + frames)."""
        rank, world, _ = parallel.world()
        first = parallel.batch_first_frame(batch_index, self.frames, rank, max(world, 1))
        ns = self.noise_std(snr_db)
        if self.fading_param is not None:
            msg, y, h = conv_link_tx_fading(self.trellis, self.modem, self.frames, self.frame_bits, self.seed, first, 0.5 * ns,
                                            self.fading_param, self.puncture)
            return msg, y, ns ** 2, h
        msg, y = conv_link_tx(self.trellis, self.modem, self.frames, self.frame_bits, self.seed, first, 0.5 * ns,
                              self.puncture)
        return msg, y, ns ** 2                                                                     # links.py:329

    # -- RX chain: this package's kernels -------------------------------------------------------------
    def receive_decode_count(self, msg, y, noise_var, counters, torch, channel_gains=None):
        from .channelcoding import viterbi_decode_batch
        if self.decoding_type == "soft":
            rx = self.modem.demodulate_batch(y, "soft", noise_var, channel_gains)
        else:
            rx = self.modem.demodulate_batch(y, "hard", channel_gains=channel_gains)
        if self.puncture is None:
            dec = viterbi_decode_batch(rx, self.trellis, self.tb_depth, self.decoding_type)
        else:
            from .channelcoding import viterbi_decode_punctured_batch
            dec = viterbi_decode_punctured_batch(rx, self.trellis, self.puncture, self.trellis.n * self.frame_bits,
                                                 self.tb_depth, "soft")
        _count_errors(dec, msg, counters, torch)
        return dec

    def link_performance(self, SNRs, send_max, err_min, return_counters=False, stop_early=True, overlap_points=True):
        """BER per SNR (dB, `SNR = Eb/N0 + 10 log10(bits/symbol)` as in the reference's examples,
        conv_encode_decode.py:102; the code rate enters through `set_SNR_dB`, channels.py:74).  A point ends
        when the GLOBAL counters reach `err_min` errors or `send_max` bits; like the reference the sweep stops after
        the first point that ends below `err_min` errors (links.py:339-341).  The stop rule is evaluated once per
        batch (frames_per_batch * world_size frames), not once per frame.

        Nothing on the critical path waits for the host: the bit count of a point is known in advance, and the error
        count of batch b is read (from a pinned snapshot) while batch b+1 is already running -- a batch issued after the
        error threshold was crossed is discarded, so the counters are exactly those of the in-order rule.
        With return_counters=True also returns the summed [bit errors, frame errors, bits] tensor of all points.
        stop_early=False measures every point of the sweep (the reference abandons the sweep after the first point that
        ends below err_min errors).
        The counters of a point's LAST batch are read after the next point's first batch has been issued (that batch is
        discarded if the sweep ends there), so the GPU does not idle between points either; overlap_points=False reads them
        at once -- same BERs and counters, the cross-check of the test suite."""
        torch = _lib.require_cuda()
        BERs = np.zeros(len(SNRs))
        batch_index = 0
        _, world, _ = parallel.world()
        bits_per_batch = self.frames * max(world, 1) * self.frame_bits
        grand = torch.zeros(3, dtype=torch.int64, device="cuda")
        pinned = torch.empty((8, 3), dtype=torch.int64).pin_memory()       # snapshot slots: at most 3 are in flight
        nslot = 0
        deferred = None                # (point, snapshot) of a point whose LAST batch is still running
        stopped = False

        def close(point, entry):
            """take a finished point's counters; True if the sweep ends here (links.py:339-341)"""
            entry[2].synchronize()
            c = entry[1].numpy()
            grand.add_(entry[0])
            BERs[point] = c[0] / c[2]
            return bool(stop_early and c[0] < err_min)

        for i, snr in enumerate(SNRs):
            tot = torch.zeros(3, dtype=torch.int64, device="cuda")          # bit errors, frame errors, bits sent
            hist = []                                                        # (device snapshot, pinned copy, event)
            bits_known = 0
            while True:
                msg, y, nv, *gains = self.make_batch(float(snr), batch_index, torch)
                batch_index += 1
                local = torch.zeros(3, dtype=torch.int64, device="cuda")
                self.receive_decode_count(msg, y, nv, local, torch, *gains)
                local[2] = msg.numel()
                parallel.allreduce_counters(local)
                tot = tot + local
                host = pinned[nslot]
                nslot = (nslot + 1) % pinned.shape[0]
                host.copy_(tot, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                hist.append((tot, host, ev))
                bits_known += bits_per_batch
                if deferred is not None:
                    # the previous point's last batch ran while this point's first batch was being issued: the GPU never
                    # waits for the host between points (this batch is discarded if the sweep ends at that point)
                    point, entry = deferred
                    deferred = None
                    if close(point, entry):
                        stopped = True
                        break
                if len(hist) >= 2:                                           # batch b-1, while batch b runs
                    hist[-2][2].synchronize()
                    if int(hist[-2][1][0]) >= err_min:
                        if close(i, hist[-2]):
                            stopped = True
                        break
                if bits_known >= send_max:
                    if overlap_points:
                        deferred = (i, hist[-1])
                    elif close(i, hist[-1]):
                        stopped = True
                    break
            if stopped:
                break
        if deferred is not None and not stopped:
            close(*deferred)
        if return_counters:
            return BERs, grand
        return BERs


def ldpc_link_tx(ldpc_code_params, modem, frames, seed, first_frame, noise_sigma):
    """Device-side TX chain of an LDPC-coded link (cpb_ldpc_link_tx) for `frames` frames starting at GLOBAL frame
    `first_frame`: k random message bits -> ldpc_encode_batch ([message | parity]) -> modem.modulate -> + noise_sigma *
    (N(0,1) + jN(0,1)).  The message and noise streams are those of `conv_link_tx`.

    Returns (msg uint8 (frames, k), y complex64 (frames, n / bits_per_symbol)) as CUDA tensors."""
    return _ldpc_link_tx(ldpc_code_params, modem, frames, seed, first_frame, noise_sigma, None)


def ldpc_link_tx_fading(ldpc_code_params, modem, frames, seed, first_frame, noise_sigma, fading_param):
    """`ldpc_link_tx` over SISO flat fading (cpb_ldpc_link_tx_fading): each symbol c is received as y = h c + noise with its
    own gain h = fading_param[0] + sqrt(fading_param[1] / 2) * (N(0,1) + jN(0,1)), drawn as `conv_link_tx_fading` draws
    them.  At fading_param = (1 + 0j, 0) the outputs equal `ldpc_link_tx`'s bit for bit.

    Returns (msg uint8 (frames, k), y complex64 (frames, nsym), h complex64 (frames, nsym)) as CUDA tensors."""
    return _ldpc_link_tx(ldpc_code_params, modem, frames, seed, first_frame, noise_sigma, fading_param)


def _ldpc_link_tx(ldpc_code_params, modem, frames, seed, first_frame, noise_sigma, fading_param):
    import ctypes as C
    from .channelcoding.ldpc import _code_dims, _ldpc_handle
    if fading_param is not None:
        mean, nlos = _fading(fading_param)
    n, m = _code_dims(ldpc_code_params)
    nb = int(modem.num_bits_symbol)
    if n % nb:
        raise ValueError("the code words must fill whole symbols: n = %d is not a multiple of %d bits per symbol" % (n, nb))
    torch = _lib.require_cuda()
    handle, _ = _ldpc_handle(ldpc_code_params)
    frames = int(frames)
    msg = torch.empty((frames, n - m), dtype=torch.uint8, device="cuda")
    y = torch.empty((frames, n // nb), dtype=torch.complex64, device="cuda")
    lib = _lib.load()
    head = (handle, modem._handle(), C.c_int64(frames), C.c_uint64(int(seed) & ((1 << 64) - 1)), C.c_int64(int(first_frame)),
            C.c_float(float(noise_sigma)))
    if fading_param is not None:
        h = torch.empty_like(y)
        rc = lib.cpb_ldpc_link_tx_fading(*head, C.c_float(mean.real), C.c_float(mean.imag), C.c_float(nlos), _lib.ptr(msg),
                                         _lib.ptr(y), _lib.ptr(h), _lib.stream_ptr(torch))
        _lib.check(rc, "ldpc_link_tx_fading")
        return msg, y, h
    rc = lib.cpb_ldpc_link_tx(*head, _lib.ptr(msg), _lib.ptr(y), _lib.stream_ptr(torch))
    _lib.check(rc, "ldpc_link_tx")
    return msg, y


class LdpcLinkGPU(ConvLinkGPU):
    """Batched LDPC-coded link on the GPU(s): frames generated and encoded on the device (cpb_ldpc_link_tx[_fading]),
    demapped (Modem.demodulate_batch, with the channel gains over fading), decoded (ldpc_bp_decode_batch) and counted over
    the k message bits (cpb_count_errors).  `link_performance`, `noise_std`, the counters, the stop rule and the rank
    sharding are ConvLinkGPU's.

    Parameters: `ldpc_code_params` (a design-file dict or a dict with a 'parity_check_matrix'; H_p = H[:, k:] must be
    invertible over GF(2)), `modem` (n must be a multiple of its bits per symbol), `frames_per_batch` frames per step and
    rank, `n_iters` / `decoder_algorithm` ('MSA' or 'SPA') / `precision` ('fp32' or 'fp64') of the decoder, `seed`, and
    `fading_param` as for ConvLinkGPU (None: AWGN).  rate = k / n."""

    def __init__(self, ldpc_code_params, modem, frames_per_batch, n_iters=15, decoder_algorithm="MSA", precision="fp32", seed=0,
                 fading_param=None):
        from .channelcoding.ldpc import _code_dims
        self.fading_param = fading_param
        if fading_param is not None:
            _fading(fading_param)
        if decoder_algorithm not in ("MSA", "SPA"):
            raise ValueError("decoder_algorithm must be 'MSA' or 'SPA'")
        if precision not in ("fp32", "fp64"):
            raise ValueError("precision must be 'fp32' or 'fp64'")
        n, m = _code_dims(ldpc_code_params)
        if n % modem.num_bits_symbol:
            raise ValueError("the code words must fill whole symbols: n = %d is not a multiple of %d bits per symbol"
                             % (n, modem.num_bits_symbol))
        self.params, self.modem = ldpc_code_params, modem
        self.n, self.frame_bits, self.frames = n, n - m, int(frames_per_batch)
        self.n_iters, self.decoder_algorithm, self.precision, self.seed = int(n_iters), decoder_algorithm, precision, int(seed)
        self.rate = Fraction(n - m, n)

    def make_batch(self, snr_db, batch_index, torch=None):
        """(msg bits, received symbols, noise_var) for one batch of this rank -- and, over fading, the channel gains."""
        rank, world, _ = parallel.world()
        first = parallel.batch_first_frame(batch_index, self.frames, rank, max(world, 1))
        ns = self.noise_std(snr_db)
        if self.fading_param is not None:
            msg, y, h = ldpc_link_tx_fading(self.params, self.modem, self.frames, self.seed, first, 0.5 * ns, self.fading_param)
            return msg, y, ns ** 2, h
        msg, y = ldpc_link_tx(self.params, self.modem, self.frames, self.seed, first, 0.5 * ns)
        return msg, y, ns ** 2

    def llrs(self, y, noise_var, channel_gains=None):
        """decoder-convention LLRs (positive favours 0, bit = signbit(llr)) of the received symbols: the demapper's
        log P(1) / P(0), negated.  (frames, n), float32 or float64 as the precision."""
        llr = self.modem.demodulate_batch(y, "soft", noise_var, channel_gains).neg_()
        return llr.double() if self.precision == "fp64" else llr

    def receive_decode_count(self, msg, y, noise_var, counters, torch, channel_gains=None):
        from .channelcoding import ldpc_bp_decode_batch
        dec = ldpc_bp_decode_batch(self.llrs(y, noise_var, channel_gains), self.params, self.n_iters, self.precision,
                                   return_llrs=False, decoder_algorithm=self.decoder_algorithm)
        _count_errors(dec, msg, counters, torch)
        return dec


def turbo_link_tx(trellis, interleaver, frames, frame_bits, seed, first_frame, noise_sigma):
    """Device-side TX chain of a turbo-coded BPSK link (cpb_turbo_link_tx): random message -> turbo_encode(msg, trellis,
    trellis, interleaver) -> 2x-1 -> + noise_sigma * N(0,1), for `frames` frames starting at GLOBAL frame `first_frame`.

    Returns (msg uint8, sys, par1, par2 float32), each (frames, frame_bits), CUDA tensors: what map_decode / turbo_decode
    take.  The streams depend only on (seed, global frame index)."""
    return _turbo_link_tx(trellis, interleaver, frames, frame_bits, seed, first_frame, noise_sigma, None)


def turbo_link_tx_fading(trellis, interleaver, frames, frame_bits, seed, first_frame, noise_sigma, fading_param):
    """`turbo_link_tx` over SISO flat fading (SISOFlatChannel, channels.py:176-221): each coded bit x = 2b - 1 of each stream
    is received as y = h x + noise_sigma * (N(0,1) + jN(0,1)) with its own gain h = fading_param[0] + sqrt(fading_param[1] /
    2) * (N(0,1) + jN(0,1)), e.g. (0j, 1) for Rayleigh and (m, 1 - |m|^2) for Rician fading.  The message and Re of the
    noise are the streams of `turbo_link_tx` (at fading_param = (1 + 0j, 0), Re(y) equals its output bit for bit).

    Returns (msg uint8 (frames, frame_bits), y complex64 (3, frames, frame_bits), h complex64 (3, frames, frame_bits)) as
    CUDA tensors; stream 0 is systematic, 1 and 2 the parity streams.  `bpsk_combine(y, h)` gives what turbo_decode
    takes at noise_variance = noise_sigma ** 2."""
    return _turbo_link_tx(trellis, interleaver, frames, frame_bits, seed, first_frame, noise_sigma, fading_param)


def _turbo_link_tx(trellis, interleaver, frames, frame_bits, seed, first_frame, noise_sigma, fading_param):
    """turbo_link_tx (fading_param None: AWGN, (msg, sys, par1, par2)) and turbo_link_tx_fading ((msg, y, h))."""
    import ctypes as C
    from .channelcoding.convcode import _trellis_handle
    from .channelcoding.turbo import _checked_perm
    if fading_param is not None:
        mean, nlos = _fading(fading_param)
    torch = _lib.require_cuda()
    N = int(frame_bits)
    perm = torch.from_numpy(_checked_perm(interleaver, N)).cuda()
    frames = int(frames)
    msg = torch.empty((frames, N), dtype=torch.uint8, device="cuda")
    lib = _lib.load()
    head = (_trellis_handle(trellis), _lib.ptr(perm), C.c_int64(frames), C.c_int64(N),
            C.c_uint64(int(seed) & ((1 << 64) - 1)), C.c_int64(int(first_frame)), C.c_float(float(noise_sigma)))
    if fading_param is not None:
        y, h = (torch.empty((3, frames, N), dtype=torch.complex64, device="cuda") for _ in range(2))
        rc = lib.cpb_turbo_link_tx_fading(*head, C.c_float(mean.real), C.c_float(mean.imag), C.c_float(nlos), _lib.ptr(msg),
                                          _lib.ptr(y), _lib.ptr(h), _lib.stream_ptr(torch))
        _lib.check(rc, "turbo_link_tx_fading")
        return msg, y, h
    ys, y1, y2 = (torch.empty((frames, N), dtype=torch.float32, device="cuda") for _ in range(3))
    rc = lib.cpb_turbo_link_tx(*head, _lib.ptr(msg), _lib.ptr(ys), _lib.ptr(y1), _lib.ptr(y2), _lib.stream_ptr(torch))
    _lib.check(rc, "turbo_link_tx")
    return msg, ys, y1, y2

def turbo_link_tx_modem(trellis, interleaver, modem, frames, frame_bits, seed, first_frame, noise_sigma):
    """Device-side TX chain of a turbo-coded link over `modem` (cpb_turbo_link_tx_modem): the message of `turbo_link_tx`,
    the code word c = np.concatenate(turbo_encode(msg, trellis, trellis, interleaver) streams, each cut to frame_bits) =
    [sys | par1 | par2] -> modem.modulate (MSB first, no channel interleaver) -> + noise_sigma * (N(0,1) + jN(0,1)), the
    noise stream of `conv_link_tx`.  3 * frame_bits must be a multiple of the modem's bits per symbol.

    Returns (msg uint8 (frames, frame_bits), y complex64 (frames, 3 frame_bits / bits_per_symbol)) as CUDA tensors."""
    return _turbo_link_tx_modem(trellis, interleaver, modem, frames, frame_bits, seed, first_frame, noise_sigma, None)


def turbo_link_tx_modem_fading(trellis, interleaver, modem, frames, frame_bits, seed, first_frame, noise_sigma, fading_param):
    """`turbo_link_tx_modem` over SISO flat fading (cpb_turbo_link_tx_modem_fading): each symbol c is received as
    y = h c + noise with its own gain h = fading_param[0] + sqrt(fading_param[1] / 2) * (N(0,1) + jN(0,1)), drawn as
    `conv_link_tx_fading` draws them.  At fading_param = (1 + 0j, 0) the outputs equal `turbo_link_tx_modem`'s bit for bit.

    Returns (msg uint8 (frames, frame_bits), y complex64 (frames, nsym), h complex64 (frames, nsym)) as CUDA tensors."""
    return _turbo_link_tx_modem(trellis, interleaver, modem, frames, frame_bits, seed, first_frame, noise_sigma, fading_param)


def _turbo_link_tx_modem(trellis, interleaver, modem, frames, frame_bits, seed, first_frame, noise_sigma, fading_param):
    import ctypes as C
    from .channelcoding.convcode import _trellis_handle
    from .channelcoding.turbo import _checked_perm
    if fading_param is not None:
        mean, nlos = _fading(fading_param)
    N, nb = int(frame_bits), int(modem.num_bits_symbol)
    if (3 * N) % nb:
        raise ValueError("the code words must fill whole symbols: 3 * %d bits is not a multiple of %d bits per symbol" % (N, nb))
    torch = _lib.require_cuda()
    perm = torch.from_numpy(_checked_perm(interleaver, N)).cuda()
    frames = int(frames)
    msg = torch.empty((frames, N), dtype=torch.uint8, device="cuda")
    y = torch.empty((frames, 3 * N // nb), dtype=torch.complex64, device="cuda")
    lib = _lib.load()
    head = (_trellis_handle(trellis), modem._handle(), _lib.ptr(perm), C.c_int64(frames), C.c_int64(N),
            C.c_uint64(int(seed) & ((1 << 64) - 1)), C.c_int64(int(first_frame)), C.c_float(float(noise_sigma)))
    if fading_param is not None:
        h = torch.empty_like(y)
        rc = lib.cpb_turbo_link_tx_modem_fading(*head, C.c_float(mean.real), C.c_float(mean.imag), C.c_float(nlos),
                                                _lib.ptr(msg), _lib.ptr(y), _lib.ptr(h), _lib.stream_ptr(torch))
        _lib.check(rc, "turbo_link_tx_modem_fading")
        return msg, y, h
    rc = lib.cpb_turbo_link_tx_modem(*head, _lib.ptr(msg), _lib.ptr(y), _lib.stream_ptr(torch))
    _lib.check(rc, "turbo_link_tx_modem")
    return msg, y


def bpsk_combine(y, h):
    """Coherent BPSK combining (cpb_bpsk_combine): s = Re(conj(h) y) for complex64 CUDA tensors y and h of one shape;
    returns float32 s of that shape.  For y = h x + sigma (n_re + j n_im), s = |h|^2 x + N(0, sigma^2 |h|^2), whose exact
    LLR 2 s / sigma^2 is what map_decode / turbo_decode compute from s at noise_variance = sigma^2."""
    import ctypes as C
    torch = _lib.require_cuda()
    for name, t in (("y", y), ("h", h)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.complex64:
            raise ValueError("bpsk_combine: %s must be a complex64 CUDA tensor" % name)
    if y.shape != h.shape:
        raise ValueError("bpsk_combine: y and h must have the same shape, got %s and %s" % (tuple(y.shape), tuple(h.shape)))
    y, h = y.contiguous(), h.contiguous()
    s = torch.empty(y.shape, dtype=torch.float32, device=y.device)
    rc = _lib.load().cpb_bpsk_combine(_lib.ptr(y), _lib.ptr(h), C.c_int64(y.numel()), _lib.ptr(s), _lib.stream_ptr(torch))
    _lib.check(rc, "bpsk_combine")
    return s


class TurboLinkGPU:
    """Batched rate-1/3 turbo link over BPSK-AWGN on the GPU(s): frames generated (cpb_turbo_link_tx), decoded
    (cpb_turbo_decode) and counted (cpb_count_errors) on the device; the error counters are the only thing all-reduced.

    `fading_param` (a SISOFlatChannel fading_param with a complex mean, e.g. (0j, 1) for Rayleigh): the link runs over i.i.d.
    flat fading, one gain per coded bit (cpb_turbo_link_tx_fading), and the receiver, which knows the gains, combines each
    value coherently (cpb_bpsk_combine) before the same turbo decoder at the same noise variance; None: AWGN.

    `modem` (a commpy_b200 Modem; 3 * frame_bits must be a multiple of its bits per symbol): the code word [sys | par1 |
    par2] is mapped onto it (cpb_turbo_link_tx_modem[_fading], one gain per symbol over fading), the receiver demaps with
    the true complex noise variance N0 (and the gains over fading) into exact LLRs log P(1) / P(0), and the turbo decoder
    takes the three LLR streams as symbols at noise_variance = 2, where its channel term 2 r / nv is the LLR itself.
    None: BPSK, one real value per coded bit, every path as without the argument."""

    def __init__(self, trellis, interleaver, frame_bits, frames_per_batch=1024, iterations=6, seed=0, fading_param=None,
                 modem=None):
        self.fading_param = fading_param
        if fading_param is not None:
            _fading(fading_param)
        if modem is not None and (3 * int(frame_bits)) % int(modem.num_bits_symbol):
            raise ValueError("the code words must fill whole symbols: 3 * %d bits is not a multiple of %d bits per symbol"
                             % (int(frame_bits), int(modem.num_bits_symbol)))
        self.trellis, self.interleaver, self.modem = trellis, interleaver, modem
        self.frame_bits, self.frames, self.iterations, self.seed = int(frame_bits), int(frames_per_batch), int(iterations), int(seed)

    def noise_variance(self, ebn0_db):
        """sigma^2 per real component at Eb/N0 (dB) for rate 1/3 and Es = 1; over fading E|h|^2 = 1 for every valid
        fading_param, so Eb/N0 is the mean Eb/N0.  With a modem: sigma^2 = Es / (2 R nb Eb/N0), nb bits per symbol of
        energy Es (the reference's SISOFlatChannel.set_SNR_dB(EbN0 + 10 log10 nb, 1/3, Es), channels.py:74)."""
        if self.modem is not None:
            nb = int(self.modem.num_bits_symbol)
            return float(self.modem.Es) / (2.0 * (1.0 / 3.0) * nb * 10 ** (ebn0_db / 10.0))
        return 1.0 / (2.0 * (1.0 / 3.0) * 10 ** (ebn0_db / 10.0))

    def make_batch(self, ebn0_db, batch_index):
        """(msg, sys, par1, par2, sigma^2) over AWGN; (msg, y, h, sigma^2) over fading (y, h: (3, frames, frame_bits)).
        With a modem: (msg, y, N0) over AWGN and (msg, y, h, N0) over fading, y and h (frames, 3 frame_bits / nb) and
        N0 = 2 sigma^2 the complex noise variance."""
        rank, world, _ = parallel.world()
        first = parallel.batch_first_frame(batch_index, self.frames, rank, max(world, 1))
        s2 = self.noise_variance(ebn0_db)
        if self.modem is not None:
            args = (self.trellis, self.interleaver, self.modem, self.frames, self.frame_bits, self.seed, first, math.sqrt(s2))
            if self.fading_param is not None:
                return turbo_link_tx_modem_fading(*args, self.fading_param) + (2.0 * s2,)
            return turbo_link_tx_modem(*args) + (2.0 * s2,)
        if self.fading_param is not None:
            return turbo_link_tx_fading(self.trellis, self.interleaver, self.frames, self.frame_bits, self.seed, first,
                                        math.sqrt(s2), self.fading_param) + (s2,)
        return turbo_link_tx(self.trellis, self.interleaver, self.frames, self.frame_bits, self.seed, first, math.sqrt(s2)) + (s2,)

    def decode_count(self, msg, *args):
        """decode_count(*make_batch(...), counters, torch): decode(msg, sys, par1, par2, s2, counters, torch) over AWGN,
        (msg, y, h, s2, counters, torch) over fading -- y and h are combined first.  Adds the errors to `counters`.
        With a modem: (msg, y, N0, counters, torch) or (msg, y, h, N0, counters, torch)."""
        from .channelcoding import turbo_decode_batch
        *rx, s2, counters, torch = args
        if self.modem is not None:
            ys, y1, y2 = self.llr_streams(*rx, s2)
            dec = turbo_decode_batch(ys, y1, y2, self.trellis, 2.0, self.iterations, self.interleaver)
            _count_errors(dec, msg, counters, torch)
            return dec
        if self.fading_param is not None:
            y, h = rx
            ys, y1, y2 = bpsk_combine(y, h)
        else:
            ys, y1, y2 = rx
        dec = turbo_decode_batch(ys, y1, y2, self.trellis, s2, self.iterations, self.interleaver)
        _count_errors(dec, msg, counters, torch)
        return dec

    def llr_streams(self, y, *rest):
        """llr_streams(y, N0) or (y, h, N0) of a modem link: the demapper's exact LLRs log P(1) / P(0) of the (frames, 3N)
        code bits (no clamp), split into three contiguous (frames, N) float32 streams sys, par1, par2."""
        *h, N0 = rest
        llr = self.modem.demodulate_batch(y, "soft", N0, h[0] if h else None).view(y.shape[0], 3 * self.frame_bits)
        N = self.frame_bits
        return tuple(llr[:, j * N:(j + 1) * N].contiguous() for j in range(3))

    def link_performance(self, EbN0s, send_max, err_min):
        """BER per Eb/N0 (dB): a point ends when the global counters reach `err_min` bit errors or `send_max` bits."""
        torch = _lib.require_cuda()
        BERs = np.zeros(len(EbN0s))
        batch_index = 0
        for i, e in enumerate(EbN0s):
            tot = torch.zeros(3, dtype=torch.int64, device="cuda")
            while True:
                batch = self.make_batch(float(e), batch_index)
                batch_index += 1
                local = torch.zeros(3, dtype=torch.int64, device="cuda")
                self.decode_count(*batch, local, torch)
                local[2] = batch[0].numel()
                parallel.allreduce_counters(local)
                tot += local
                c = tot.cpu().numpy()
                if not parallel.stop_rule(c, send_max, err_min):
                    break
            BERs[i] = c[0] / c[2]
        return BERs


def idd_decoder(detector, decoder, decision, n_it):
    """Iterative detection and decoding for a coded MIMO link (links.py:345-407): returns the 6-argument decoder LinkModel
    calls.  Each iteration decodes the current a-priori LLRs, hands the extrinsic part to `detector(y_i, H_i, constellation,
    noise_var, a_priori_i)` vector by vector, and keeps the detector's extrinsic for the next round; `decision` maps the
    final LLRs to bits."""
    def decode(y, h, constellation, noise_var, a_priori, bits_per_send):
        to_decoder = np.array(a_priori, dtype=float)
        nb_vect = h.shape[0]
        to_detector = np.zeros_like(to_decoder)
        for _ in range(n_it):
            to_detector = decoder(to_decoder) - to_decoder
            for i in range(nb_vect):
                sl = slice(i * bits_per_send, (i + 1) * bits_per_send)
                to_decoder[sl] = detector(y[i], h[i], constellation, noise_var, to_detector[sl])
            to_decoder -= to_detector
        return decision(to_decoder + to_detector)
    return decode

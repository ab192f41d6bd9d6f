"""802.11 (up to VHT) physical-layer parameters around the GPU decoding path.

Mirror of commpy/wifi80211.py:23-216: MCS -> modem / code-rate tables, the rate-1/2 mother code with
puncturing, and `link_performance` assembling modulate / receiver / decoder closures for `LinkModel`.  The
receiver (soft demapper) and the decoder (soft Viterbi) run in this package's CUDA kernels.

The reference builds its trellis from the DECIMAL pair (133, 171) (wifi80211.py:49) which `Trellis` reads as the
taps (5, 43) -- a different, weaker code than the standard's octal (133, 171).  The quirk is kept (same tables,
same BER curves as the reference); that trellis has its own register-resident kernel instance
(`Code5_43` in csrc/viterbi.cu).
"""
import math

import numpy as np

from . import links as lk
from . import modulation as mod
from .channelcoding import convcode as cc

__all__ = ["Wifi80211"]


class Wifi80211:
    memory = np.array(6, ndmin=1)
    generator_matrix = np.array((133, 171), ndmin=2)      # decimal, as in the reference

    _constellation_size = (2, 4, 4, 16, 16, 64, 64, 64, 256, 256)                       # wifi80211.py:56-67
    _coding = ((1, 2), (1, 2), (3, 4), (1, 2), (3, 4), (2, 3), (3, 4), (5, 6), (3, 4), (5, 6))   # :90-101

    def __init__(self, mcs):
        """mcs 0..9: BPSK 1/2, QPSK 1/2, QPSK 3/4, 16-QAM 1/2, 16-QAM 3/4, 64-QAM 2/3, 3/4, 5/6, 256-QAM 3/4, 5/6."""
        self.mcs = mcs
        self.modem = None

    def get_modem(self):
        size = self._constellation_size[self.mcs]
        return mod.PSKModem(size) if self.mcs <= 2 else mod.QAMModem(size)

    @staticmethod
    def _get_puncture_matrix(numerator, denominator):
        return {(2, 3): [1, 1, 1, 0], (3, 4): [1, 1, 1, 0, 0, 1],
                (5, 6): [1, 1, 1, 0, 0, 1, 1, 0, 0, 1]}.get((numerator, denominator))

    def _get_coding(self):
        return self._coding[self.mcs]

    @staticmethod
    def _get_trellis():
        return cc.Trellis(Wifi80211.memory, Wifi80211.generator_matrix)

    def link_performance_gpu(self, SNRs, send_max, err_min, send_chunk=4096, frames_per_batch=4096, seed=0, stop_early=True,
                             fading_param=None):
        """The same MCS over an AWGN SISO channel, batched on the GPU(s): frames are generated, punctured, mapped and
        disturbed on the device (cpb_conv_link_tx[_punctured]), demapped (cpb_demod_soft) and decoded with the depuncturing
        fused into the Viterbi kernel's load (cpb_viterbi_decode_punctured).  `send_chunk` information bits per frame
        (rounded down so that the punctured frame fills whole symbols and whole puncturing periods).  Returns the BER per
        SNR like `ConvLinkGPU.link_performance`.  `fading_param` (e.g. (0j, 1), Rayleigh): SISO flat fading instead of AWGN,
        with a demapper that knows the gains (see `ConvLinkGPU`)."""
        num, den = self._get_coding()
        modem = self.get_modem()
        pattern = Wifi80211._get_puncture_matrix(num, den)
        nb = modem.num_bits_symbol
        unit = 1
        while (lk.kept_bits(2 * unit, pattern) % nb) or (pattern and (2 * unit) % len(pattern)):
            unit += 1
        frame_bits = max(unit, (int(send_chunk) // unit) * unit)
        self.gpu_link = lk.ConvLinkGPU(Wifi80211._get_trellis(), modem, frame_bits=frame_bits, frames_per_batch=frames_per_batch,
                                       decoding_type="soft", seed=seed, puncture=pattern, fading_param=fading_param)
        return self.gpu_link.link_performance(SNRs, send_max, err_min, stop_early=stop_early)

    def link_performance(self, channel, SNRs, tx_max, err_min, send_chunk=None, frame_aggregation=1, receiver=None,
                         stop_on_surpass_error=True):
        """Monte-Carlo BER of the selected MCS over `channel` (wifi80211.py:132-216): returns
        `LinkModel.link_performance_full_metrics(...)` = (BERs, BEs, CEs, NCs)."""
        trellis = Wifi80211._get_trellis()
        num, den = self._get_coding()
        modem = self.get_modem()
        pattern = Wifi80211._get_puncture_matrix(num, den)

        def modulate(bits):
            coded = cc.conv_encode(bits, trellis, "cont")
            return modem.modulate(cc.puncturing(coded, pattern) if pattern else coded)

        def _receiver(y, h, constellation, noise_var):
            return modem.demodulate(y, "soft", noise_var)

        def decoder_soft(msg):
            llr = msg
            if pattern:
                try:
                    llr = cc.depuncturing(msg, pattern, math.ceil(len(msg) * num / den * 2))
                except IndexError as e:                    # the reference prints and decodes the punctured stream
                    print(e)
                    print("Decoded message size %d" % (math.ceil(len(msg) * num / den * 2)))
                    print("Encoded message size %d" % len(msg))
                    print("Coding %d/%d" % (num, den))
            return cc.viterbi_decode(llr, trellis, decoding_type="soft")

        self.model = lk.LinkModel(modulate, channel, receiver or _receiver, modem.num_bits_symbol, modem.constellation,
                                  modem.Es, decoder_soft, num / den)
        return self.model.link_performance_full_metrics(SNRs, tx_max, err_min=err_min, send_chunk=send_chunk,
                                                        code_rate=num / den, number_chunks_per_send=frame_aggregation,
                                                        stop_on_surpass_error=stop_on_surpass_error)

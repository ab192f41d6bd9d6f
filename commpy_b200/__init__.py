"""commpy_b200 -- H100-native (sm_90a CUDA) implementation of CommPy's decoding hot path.

Module layout mirrors the reference so that `import commpy_b200 as commpy` resolves the same names:

    commpy_b200.channelcoding   Trellis, conv_encode, viterbi_decode, map_decode, turbo_decode,
                                turbo_encode, RandInterlv, get_ldpc_code_params, ldpc_bp_decode, ...
    commpy_b200.modulation      Modem, PSKModem, QAMModem (.demodulate on the GPU)
    commpy_b200.utilities       dec2bitarray, bitarray2dec, hamming_dist, euclid_dist, signal_power
    commpy_b200.links           LinkModel, link_performance (batched multi-GPU Monte-Carlo driver)

All decoding runs in hand-written CUDA behind the C-ABI of include/commpy_b200.h
(commpy_b200/libcommpy_b200.so); there is no CPU fallback.
"""
from . import utilities  # noqa: F401
from . import channelcoding  # noqa: F401
from . import modulation  # noqa: F401

__version__ = "0.1.0"

"""Channel coding: same public names as commpy.channelcoding (commpy/channelcoding/__init__.py:65-71)."""
from .convcode import (Trellis, conv_encode, viterbi_decode, viterbi_decode_batch, viterbi_decode_punctured_batch,  # noqa: F401
                       puncturing, depuncturing)
from .interleavers import RandInterlv  # noqa: F401
from .ldpc import (get_ldpc_code_params, ldpc_bp_decode, ldpc_bp_decode_batch, ldpc_bp_decode_batch_host,  # noqa: F401
                   triang_ldpc_systematic_encode, write_ldpc_params, build_matrix, ldpc_encode_batch)
from .turbo import (turbo_encode, map_decode, turbo_decode, map_decode_batch, turbo_decode_batch,  # noqa: F401
                    map_decode_batch_host, turbo_decode_batch_host, suggest_map_window, set_map_window)

"""Convolutional codes: Trellis descriptor, encoder, puncturing and the GPU Viterbi decoder.

Mirror of commpy/channelcoding/convcode.py (reference file:line cited per function).  The
descriptor / encoder side is small host code; `viterbi_decode` runs in CUDA
(commpy_b200/csrc/viterbi.cu) through `cpb_viterbi_decode` -- there is no CPU decode path.
"""
import ctypes as C
from warnings import warn

import numpy as np

from .. import _lib
from ..utilities import bitarray2dec, dec2bitarray, decimal2bitarray

__all__ = ["Trellis", "conv_encode", "viterbi_decode", "viterbi_decode_batch", "viterbi_decode_punctured_batch", "puncturing",
           "depuncturing"]


def _tap_bits(number, width, polynomial_format):
    """Bits of a generator / feedback polynomial indexed by delay (0 = current input).

    convcode.py:212-222 reads `dec2bitarray(number, width)[::bit_order]`; the helper keeps the
    index wrap of utilities.py:78-85 for numbers wider than `width`."""
    msb_first = decimal2bitarray(number, width)
    return msb_first[::-1] if polynomial_format == "MSB" else msb_first


class Trellis:
    """Finite-state-machine tables of a convolutional code (convcode.py:23-255).

    Parameters and attributes are the reference's: `k, n, total_memory, number_states, number_inputs,
    next_state_table, output_table, code_type`.  State bits are MSB first per shift register, the newest
    bit first; output symbols are MSB first (first generator column = MSB).
    """

    def __init__(self, memory, g_matrix, feedback=None, code_type="default", polynomial_format="MSB"):
        memory = np.asarray(memory)
        self.k, self.n = g_matrix.shape
        self.code_type = code_type
        self.total_memory = int(memory.sum())
        self.number_states = 2 ** self.total_memory
        self.number_inputs = 2 ** self.k
        self.next_state_table = np.zeros((self.number_states, self.number_inputs), "int")
        self.output_table = np.zeros((self.number_states, self.number_inputs), "int")
        if isinstance(feedback, int):
            warn("Trellis  will only accept feedback as a matrix in the future. "
                 "Using the backwards compatibility version that may contain bugs for k > 1 or with LSB format.",
                 DeprecationWarning)
            self._fill_legacy(memory, g_matrix, feedback)
        else:
            self._fill(memory, g_matrix, feedback, polynomial_format)

    # -- matrix-feedback / feed-forward construction: convcode.py:195-255 ----------------------------
    def _fill(self, memory, g_matrix, feedback, polynomial_format):
        if polynomial_format not in ("MSB", "LSB", "Matlab"):
            raise ValueError('polynomial_format must be "LSB", "MSB" or "Matlab"')
        k, n, M = self.k, self.n, self.total_memory
        width = int(memory.max()) + 1
        if feedback is None:
            feedback = np.identity(k, int)
            if polynomial_format != "MSB":
                feedback = feedback * 2 ** int(memory.max())
        g_taps = np.zeros((width, k, n), np.int64)     # [delay, input register, output]
        f_taps = np.zeros((width, k, k), np.int64)     # [delay, fed register, source register]
        for i in range(k):
            for j in range(n):
                g_taps[:, i, j] = _tap_bits(g_matrix[i, j], width, polynomial_format)
            for j in range(k):
                f_taps[:, i, j] = _tap_bits(feedback[i, j], width, polynomial_format)
        offsets = np.concatenate(([0], np.cumsum(memory)[:-1])).astype(int)
        for state in range(self.number_states):
            sbits = decimal2bitarray(state, M).astype(np.int64)
            for word in range(self.number_inputs):
                lines = np.zeros((width, k), np.int64)         # row b = delay b of every register
                lines[0] = decimal2bitarray(word, k)
                for i, (off, mem) in enumerate(zip(offsets, memory)):
                    lines[1:mem + 1, i] = sbits[off:off + mem]
                outputs = np.einsum("bi,bij->j", lines, g_taps) % 2
                self.output_table[state, word] = bitarray2dec(outputs)
                fed = np.einsum("bs,bfs->f", lines, f_taps) % 2   # what enters each register
                nxt = sbits.copy()
                for i, (off, mem) in enumerate(zip(offsets, memory)):
                    if mem > 0:
                        nxt[off] = fed[i]
                        nxt[off + 1:off + mem] = lines[1:mem, i]
                self.next_state_table[state, word] = bitarray2dec(nxt)

    # -- integer-feedback backwards-compatibility construction: convcode.py:130-193 -------------------
    def _fill_legacy(self, memory, g_matrix, feedback):
        k, n, M = self.k, self.n, self.total_memory
        if self.code_type == "rsc":
            for i in range(k):
                g_matrix[i][i] = feedback                      # the reference overwrites the caller's matrix
        for state in range(self.number_states):
            for word in range(self.number_inputs):
                in_bits = decimal2bitarray(word, k)
                outbits = np.zeros(n, "int")
                reg = None
                for r in range(n):
                    reg = decimal2bitarray(state, M).astype(int)
                    direct = np.zeros(k, "int")
                    fb = 0
                    for l in range(k):
                        gen = decimal2bitarray(g_matrix[l][r], memory[l] + 1)
                        for i in range(memory[l]):
                            outbits[r] = (outbits[r] + reg[i + l] * gen[i + 1]) % 2
                        direct[l] = gen[0]
                        if l == 0:
                            fb = int((decimal2bitarray(feedback, memory[l] + 1)[1:] * reg[0:memory[l]]).sum())
                            reg[1:memory[l]] = reg[0:memory[l] - 1].copy()
                            reg[0] = (in_bits[0] + fb) % 2
                        else:
                            lo = l + memory[l - 1] - 1
                            fb = int((decimal2bitarray(feedback, memory[l] + 1) * reg[lo:lo + memory[l]]).sum())
                            reg[lo + 1:lo + memory[l]] = reg[lo:lo + memory[l] - 1].copy()
                            reg[lo] = (in_bits[l] + fb) % 2
                    outbits[r] = (outbits[r] + (np.sum(in_bits * direct + fb) % 2)) % 2
                self.output_table[state, word] = bitarray2dec(outbits)
                self.next_state_table[state, word] = bitarray2dec(reg)

    # -- device handle (created on first decode, one per CUDA device) --------------------------------
    def _handle(self):
        return _trellis_handle(self)


class _HandleBox:
    """Owns a cpbTrellis* and frees it with the Python object."""

    def __init__(self, ptr):
        self.ptr = ptr

    def __del__(self):
        try:
            if self.ptr:
                _lib.load().cpb_trellis_destroy(self.ptr)
        except Exception:
            pass


def _trellis_handle(trellis):
    """cpbTrellis handle for any object with the reference's Trellis attributes (duck-typed)."""
    torch = _lib.require_cuda()
    dev = torch.cuda.current_device()
    cache = trellis.__dict__.setdefault("_cpb_handles", {})
    nst = np.ascontiguousarray(trellis.next_state_table, dtype=np.int32)
    out = np.ascontiguousarray(trellis.output_table, dtype=np.int32)
    key = (dev, nst.tobytes(), out.tobytes())
    box = cache.get(dev)
    if box is None or box[0] != key:
        h = C.c_void_p()
        rc = _lib.load().cpb_trellis_create(_lib.ptr(nst), _lib.ptr(out), int(trellis.k), int(trellis.n),
                                            int(trellis.total_memory), int(trellis.number_states), C.byref(h))
        _lib.check(rc, "Trellis")
        box = (key, _HandleBox(h))
        cache[dev] = box
    return box[1].ptr


def conv_encode(message_bits, trellis, termination="term", puncture_matrix=None):
    """Convolutional encoder (convcode.py:475-558): table walk from state 0.

    'term' appends `total_memory` zero inputs (feed-forward codes) or drives an 'rsc' code back with the
    reversed state bits; puncturing keeps position i when `puncture_matrix[0][i % ncols] == 1` and, like the
    reference, leaves the output at its unpunctured length with trailing zeros."""
    k, n = trellis.k, trellis.n
    M = trellis.total_memory
    rate = float(k) / n
    if puncture_matrix is None:
        puncture_matrix = np.ones((k, n))
    message_bits = np.asarray(message_bits)
    n_msg = np.size(message_bits)
    if termination == "cont":
        inbits = message_bits
        n_in = n_msg
        n_out = int(n_in / rate)
    elif trellis.code_type == "rsc":
        inbits = message_bits
        n_in = n_msg
        n_out = int((n_in + k * M) / rate)
    else:
        n_in = n_msg + M + M % k
        inbits = np.zeros(n_in, "int")
        inbits[:n_msg] = message_bits
        n_out = int(n_in / rate)
    outbits = np.zeros(n_out, "int")
    nst, otab = trellis.next_state_table, trellis.output_table
    weights = 1 << np.arange(k - 1, -1, -1)
    state = 0
    pos = 0
    for i in range(int(n_in / k)):
        word = int(np.dot(np.asarray(inbits[i * k:(i + 1) * k], dtype=np.int64), weights))
        outbits[pos:pos + n] = dec2bitarray(int(otab[state][word]), n)
        state = nst[state][word]
        pos += n
    if trellis.code_type == "rsc" and termination == "term":
        tail = dec2bitarray(int(state), M)[::-1]
        for i in range(M):
            word = bitarray2dec(tail[i * k:(i + 1) * k])
            outbits[pos:pos + n] = dec2bitarray(int(otab[state][word]), n)
            state = nst[state][word]
            pos += n
    ncols = np.size(puncture_matrix, 1)
    keep = np.asarray(puncture_matrix)[0][np.arange(n_out) % ncols] == 1
    p_outbits = np.zeros(n_out, "int")
    kept = outbits[keep]
    p_outbits[:kept.size] = kept
    return p_outbits


def puncturing(message, punct_vec):
    """Keep message[i] where punct_vec[i % len(punct_vec)] == 1 (convcode.py:752-774)."""
    message = np.asarray(message)
    punct_vec = np.asarray(punct_vec)
    mask = punct_vec[np.arange(len(message)) % len(punct_vec)] == 1
    return np.array(message[mask])


def depuncturing(punctured, punct_vec, shouldbe):
    """Re-insert 0.0 at punctured positions (convcode.py:777-804); IndexError if `punctured` runs short."""
    punctured = np.asarray(punctured)
    punct_vec = np.asarray(punct_vec)
    mask = punct_vec[np.arange(shouldbe) % len(punct_vec)] == 1
    need = int(mask.sum())
    if need > len(punctured):
        raise IndexError("index %d is out of bounds for axis 0 with size %d" % (len(punctured), len(punctured)))
    out = np.zeros((shouldbe,))
    out[mask] = punctured[:need].astype(float)
    return out


# ----------------------------------------------------------------------------------------------------
# Viterbi on the GPU
# ----------------------------------------------------------------------------------------------------
_MODE_ERR = 'The available decoding types are "hard", "soft" and "unquantized'


def _decoded_bits(trellis, n_in, tb_depth):
    """Decoded bits L of a frame of n_in coded values; ValueError when tb_depth leaves no complete traceback window."""
    L = int(n_in * (trellis.k / trellis.n))                        # convcode.py:699
    T = int((L + trellis.total_memory) / trellis.k) - 1            # :721
    D = min(5 * trellis.total_memory, L) if tb_depth is None else int(tb_depth)      # :701-702
    if D < 2 or T < D - 1:
        raise ValueError("tb_depth=%d leaves no complete traceback window for %d trellis steps "
                         "(the reference returns uninitialised memory here)" % (D, T))
    return L


def _numpy_rows(coded, hard):
    """numpy rows in the kernel's dtype: uint8 bits (hard decision, values checked) or float32."""
    a = np.asarray(coded)
    if not hard:
        return np.ascontiguousarray(a, dtype=np.float32)
    ai = a if a.dtype == np.uint8 else a.astype(np.int64)          # astype(int): convcode.py:579
    if ai.size and (ai.min() < 0 or ai.max() > 1):
        raise ValueError("hard-decision input must contain only 0 and 1")
    return np.ascontiguousarray(ai, dtype=np.uint8)


def _check_out(out, shape, like, torch):
    """A caller-supplied result buffer must be a dense uint8 array of the right shape, of the same kind as the input."""
    if hasattr(like, "data_ptr") != hasattr(out, "data_ptr"):
        raise ValueError("`out` must be the same kind of array as the input (torch tensor / numpy array)")
    if hasattr(out, "data_ptr"):
        ok = out.dtype == torch.uint8 and tuple(out.shape) == tuple(shape) and out.is_contiguous() and out.device == like.device
    else:
        ok = out.dtype == np.uint8 and out.shape == tuple(shape) and out.flags["C_CONTIGUOUS"]
    if not ok:
        raise ValueError("`out` must be a contiguous uint8 array of shape %s on the input's device" % (tuple(shape),))


def viterbi_decode_batch(coded, trellis, tb_depth=None, decoding_type="hard", out=None, packed=False):
    """Decode a batch of independent frames on the GPU.

    coded : (batch, n_in) array.  'hard': values in {0, 1} (uint8 is the zero-copy layout);
            'soft' / 'unquantized': float32 is zero-copy.
        * torch CUDA tensor -> decoded in place on the current stream, returns a (batch, L) uint8 CUDA tensor;
        * numpy array or CPU torch tensor (pinned memory overlaps best) -> `cpb_viterbi_decode_host`: chunked
          H2D / decode / D2H pipeline, returns a numpy array (or CPU tensor) of uint8 bits.
    `out` may supply the result buffer (same kind as the input, contiguous uint8 of the result's shape).
    packed=True ('hard' only): `coded` holds 1 bit per coded bit, rows packed like numpy.packbits(bits, axis=1), and the
    result is packed the same way, (batch, L/8) -- the same decisions with 8x less PCIe / HBM traffic
    (cpb_viterbi_decode_packed; K=7 fast-path codes, (tb_depth - 2) % 4 == 0, n_in % 16 == 0).
    """
    if decoding_type not in _lib.VITERBI_MODES:
        raise ValueError(_MODE_ERR)
    hard = decoding_type == "hard"
    two_d = getattr(coded, "ndim", None) == 2 or (hasattr(coded, "dim") and coded.dim() == 2)
    if packed and not hard:
        raise ValueError("packed=True is a hard-decision format")
    if packed and not two_d:
        raise ValueError("coded must be (batch, n_in / 8)")
    torch = _lib.require_cuda()
    lib = _lib.load()
    if not two_d:
        raise ValueError("coded must be (batch, n_in)")
    is_torch = hasattr(coded, "data_ptr")
    on_device = is_torch and coded.is_cuda
    handle = _trellis_handle(trellis)
    if packed:
        x = coded.contiguous() if is_torch else np.ascontiguousarray(coded)
        if x.dtype != (torch.uint8 if is_torch else np.uint8):
            raise ValueError("packed input must be uint8")
    elif is_torch:
        want = torch.uint8 if hard else torch.float32
        x = (coded if coded.dtype == want else coded.to(want)).contiguous()
    else:
        x = _numpy_rows(coded, hard)
    batch, n_in = x.shape[0], x.shape[1] * (8 if packed else 1)
    L = _decoded_bits(trellis, n_in, tb_depth)
    if packed and L % 8:
        raise NotImplementedError("packed decode needs a whole number of output bytes per frame")
    shape = (batch, L // 8 if packed else L)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=x.device) if is_torch else np.empty(shape, np.uint8)
    else:
        _check_out(out, shape, x, torch)
    depth = int(tb_depth or 0)
    in_dtype, mode = _lib.CPB_U8 if hard else _lib.CPB_F32, _lib.VITERBI_MODES[decoding_type]
    if packed and on_device:
        rc = lib.cpb_viterbi_decode_packed(handle, _lib.ptr(x), C.c_int64(batch), C.c_int64(n_in), depth, _lib.ptr(out),
                                           _lib.stream_ptr(torch))
    elif packed:
        rc = lib.cpb_viterbi_decode_host_packed(handle, _lib.ptr(x), C.c_int64(batch), C.c_int64(n_in), depth, _lib.ptr(out))
    elif on_device:
        rc = lib.cpb_viterbi_decode(handle, _lib.ptr(x), in_dtype, C.c_int64(batch), C.c_int64(n_in), depth, mode,
                                    _lib.ptr(out), C.c_void_p(0), C.c_size_t(0), _lib.stream_ptr(torch))
    else:
        rc = lib.cpb_viterbi_decode_host(handle, _lib.ptr(x), in_dtype, C.c_int64(batch), C.c_int64(n_in), depth, mode,
                                         _lib.ptr(out))
    _lib.check(rc, "viterbi_decode (packed)" if packed else "viterbi_decode")
    return out


def viterbi_decode_punctured_batch(llr, trellis, punct_vec, shouldbe, tb_depth=None, decoding_type="soft"):
    """depuncturing(row, punct_vec, shouldbe) + viterbi_decode(..., decoding_type) for a batch of PUNCTURED rows in one kernel
    (cpb_viterbi_decode_punctured: the zeros of convcode.py:777-804 are inserted in the kernel's load, nothing is
    materialised).  llr: (batch, n_kept) float32 CUDA tensor or array.  Returns a (batch, L) uint8 CUDA tensor.
    Trellises without a register-resident kernel take the two-step route (host depuncturing mirror + viterbi_decode_batch)."""
    if decoding_type not in ("soft", "unquantized"):
        raise ValueError("punctured decoding takes soft values ('soft' or 'unquantized')")
    torch = _lib.require_cuda()
    lib = _lib.load()
    if hasattr(llr, "data_ptr"):
        x = (llr if llr.is_cuda else llr.cuda()).to(torch.float32).contiguous()
    else:
        x = torch.from_numpy(np.ascontiguousarray(llr, dtype=np.float32)).cuda()
    if x.dim() != 2:
        raise ValueError("llr must be (batch, n_kept)")
    pv = np.ascontiguousarray(punct_vec, dtype=np.int32)
    batch, n_kept = x.shape
    L = _decoded_bits(trellis, int(shouldbe), tb_depth)
    handle = _trellis_handle(trellis)
    out = torch.empty((batch, L), dtype=torch.uint8, device=x.device)
    rc = lib.cpb_viterbi_decode_punctured(handle, _lib.ptr(x), C.c_int64(batch), C.c_int64(n_kept), _lib.ptr(pv), int(len(pv)),
                                          C.c_int64(int(shouldbe)), int(tb_depth or 0), _lib.VITERBI_MODES[decoding_type],
                                          _lib.ptr(out), C.c_void_p(0), C.c_size_t(0), _lib.stream_ptr(torch))
    if rc == _lib.CPB_EUNSUPPORTED:
        rows = x.cpu().numpy()
        dep = np.stack([depuncturing(r, pv, int(shouldbe)) for r in rows]).astype(np.float32)
        return viterbi_decode_batch(torch.from_numpy(dep).cuda(), trellis, tb_depth, decoding_type)
    if rc == _lib.CPB_EINVAL and n_kept < int(np.sum(pv[np.arange(int(shouldbe)) % len(pv)] == 1)):
        raise IndexError("index %d is out of bounds for axis 0 with size %d" % (n_kept, n_kept))
    _lib.check(rc, "viterbi_decode (punctured)")
    return out


def viterbi_decode(coded_bits, trellis, tb_depth=None, decoding_type="hard"):
    """Drop-in for commpy.channelcoding.viterbi_decode (convcode.py:661-749): one frame, 1-D in, 1-D int out.

    Differences from the reference, all deliberate (SURVEY.md section 8b):
      * an unknown `decoding_type` raises ValueError up front (the documented behaviour, :682-685);
      * the caller's `coded_bits` is never written (the reference pads through a view of it, :724-732);
      * a `tb_depth` for which the reference would return uninitialised memory raises ValueError.
    Soft / unquantized inputs are decoded with fixed-point metrics (2^-17 of the frame's OWN largest magnitude, so a
    frame decodes identically whatever it is batched with) instead of float64: identical BER, bit agreement reported
    by the parity tests.
    """
    if decoding_type not in _lib.VITERBI_MODES:
        raise ValueError(_MODE_ERR)
    a = np.asarray(coded_bits)
    if a.ndim != 1:
        raise ValueError("coded_bits must be 1-D (use viterbi_decode_batch for a batch of frames)")
    return viterbi_decode_batch(a[None, :], trellis, tb_depth, decoding_type)[0].astype("int")

"""Turbo codes: encoder (host) and BCJR / turbo decoding on the GPU.

Mirror of commpy/channelcoding/turbo.py.  `map_decode` / `turbo_decode` run in CUDA
(commpy_b200/csrc/bcjr.cu) through `cpb_map_decode[_host]` / `cpb_turbo_decode[_host]`; there is no CPU decode path.
The hot kernel works, like the reference, with renormalised probabilities (float32 instead of float64, branch weights
taken relative to the step's most likely (input, parity) pair so nothing overflows; rescaled every 4th step, a block
whose metric sum decays is redone with the reference's per-step rescaling); one thread owns a window of 1024 trellis
steps of a frame and warms its recursions up over 96 steps of the neighbouring windows (<= 3.4e-7 on the LLRs against
the reference's full-frame recursion).  `turbo_decode` transposes the symbol streams to step-major once, so the
interleaver is a row index of the MAP kernel instead of a data movement.  Unaligned frame lengths and other trellises
take the log-domain exact max* kernels.  LLRs agree to ~1e-5 where the reference is finite (it returns +-inf once its exponentials underflow; the
GPU path stays finite there).
"""
import ctypes as C

import numpy as np

from .. import _lib
from .convcode import _trellis_handle, conv_encode

__all__ = ["turbo_encode", "map_decode", "turbo_decode", "map_decode_batch", "turbo_decode_batch", "map_decode_batch_host",
           "turbo_decode_batch_host", "suggest_map_window", "set_map_window"]


def turbo_encode(msg_bits, trellis1, trellis2, interleaver):
    """Rate-1/3 parallel concatenation (turbo.py:14-59): returns [sys, parity1, parity2].

    Exactly like the reference the two RSC encoders run 'rsc'-terminated and the last `total_memory`
    entries of each stream are dropped; the second parity stream comes from a punctured conv_encode whose
    output keeps its unpunctured length, so it is longer than the other two (SURVEY.md section 8c)."""
    stream = conv_encode(msg_bits, trellis1, "rsc")
    sys_stream = stream[::2]
    non_sys_stream_1 = stream[1::2]
    interlv_msg_bits = interleaver.interlv(sys_stream)
    non_sys_stream_2 = conv_encode(interlv_msg_bits, trellis2, "rsc", np.array([[0, 1]]))
    m1, m2 = trellis1.total_memory, trellis2.total_memory
    return [sys_stream[0:-m1], non_sys_stream_1[0:-m1], non_sys_stream_2[0:-m2]]


def _dev_f32(x, torch):
    if hasattr(x, "data_ptr"):
        t = x if x.is_cuda else x.cuda()
        return t.to(torch.float32).contiguous()
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()


def map_decode_batch(sys_symbols, non_sys_symbols, trellis, noise_variance, L_int, mode="decode"):
    """Batched MAP decoder: (batch, N) inputs -> (L (batch, N) float32, bits (batch, N) uint8) torch CUDA tensors."""
    torch = _lib.require_cuda()
    s = _dev_f32(sys_symbols, torch)
    p = _dev_f32(non_sys_symbols, torch)
    la = _dev_f32(L_int, torch)
    if s.dim() != 2 or s.shape != p.shape or s.shape != la.shape:
        raise ValueError("sys_symbols, non_sys_symbols and L_int must share the shape (batch, N)")
    batch, N = s.shape
    L = torch.empty_like(s)
    bits = torch.empty((batch, N), dtype=torch.uint8, device=s.device)
    rc = _lib.load().cpb_map_decode(_trellis_handle(trellis), _lib.ptr(s), _lib.ptr(p), _lib.ptr(la),
                                    C.c_int64(batch), C.c_int64(N), C.c_float(noise_variance),
                                    1 if mode == "decode" else 0, _lib.ptr(L), _lib.ptr(bits), C.c_void_p(0), C.c_size_t(0),
                                    _lib.stream_ptr(torch))
    _lib.check(rc, "map_decode")
    return L, bits


def map_decode_batch_host(sys_symbols, non_sys_symbols, trellis, noise_variance, L_int, mode="decode"):
    """Batched MAP decoder for HOST arrays through the pipelined host entry point (cpb_map_decode_host):
    (batch, N) float arrays -> (L (batch, N) float32, bits (batch, N) uint8) numpy arrays."""
    _lib.require_cuda()
    s = np.ascontiguousarray(sys_symbols, dtype=np.float32)
    p = np.ascontiguousarray(non_sys_symbols, dtype=np.float32)
    la = np.ascontiguousarray(L_int, dtype=np.float32)
    if s.ndim != 2 or s.shape != p.shape or s.shape != la.shape:
        raise ValueError("sys_symbols, non_sys_symbols and L_int must share the shape (batch, N)")
    batch, N = s.shape
    L = np.empty((batch, N), dtype=np.float32)
    bits = np.empty((batch, N), dtype=np.uint8)
    rc = _lib.load().cpb_map_decode_host(_trellis_handle(trellis), _lib.ptr(s), _lib.ptr(p), _lib.ptr(la), C.c_int64(batch),
                                         C.c_int64(N), C.c_float(noise_variance), 1 if mode == "decode" else 0,
                                         _lib.ptr(L), _lib.ptr(bits))
    _lib.check(rc, "map_decode")
    return L, bits


def _host_out(out, shape, dtype, what):
    """caller-supplied host output (numpy array or CPU torch tensor; pinned memory keeps the D2H copies asynchronous, a
    pageable destination makes every chunk's copy-back block the host and serialises the pipeline) or a fresh array"""
    if out is None:
        return np.empty(shape, dtype=dtype)
    arr = out.numpy() if hasattr(out, "numpy") and not isinstance(out, np.ndarray) else out
    if not isinstance(arr, np.ndarray) or arr.shape != tuple(shape) or arr.dtype != np.dtype(dtype) or not arr.flags["C_CONTIGUOUS"]:
        raise ValueError("%s must be a C-contiguous %s host array of shape %s" % (what, np.dtype(dtype).name, tuple(shape)))
    return arr


def turbo_decode_batch_host(sys_symbols, non_sys_symbols_1, non_sys_symbols_2, trellis, noise_variance,
                            number_iterations, interleaver, L_int=None, out=None):
    """Batched turbo decoder for HOST arrays through the pipelined host entry point (cpb_turbo_decode_host):
    (batch, N) float arrays -> (batch, N) uint8 numpy array (`out`, if given: e.g. a pinned buffer)."""
    _lib.require_cuda()
    s = np.ascontiguousarray(sys_symbols, dtype=np.float32)
    p1 = np.ascontiguousarray(non_sys_symbols_1, dtype=np.float32)
    p2 = np.ascontiguousarray(non_sys_symbols_2, dtype=np.float32)
    if s.ndim != 2 or s.shape != p1.shape or s.shape != p2.shape:
        raise ValueError("the three symbol streams must share the shape (batch, N)")
    batch, N = s.shape
    perm = _checked_perm(interleaver, N)
    la = None if L_int is None else np.ascontiguousarray(L_int, dtype=np.float32)
    bits = _host_out(out, (batch, N), np.uint8, "out")
    rc = _lib.load().cpb_turbo_decode_host(_trellis_handle(trellis), _lib.ptr(s), _lib.ptr(p1), _lib.ptr(p2), _lib.ptr(perm),
                                           C.c_int64(batch), C.c_int64(N), C.c_float(noise_variance), int(number_iterations),
                                           _lib.ptr(la), _lib.ptr(bits))
    _lib.check(rc, "turbo_decode")
    return bits


def suggest_map_window(batch, N, target_threads=49152):
    """MAP window length (trellis steps per thread) that fills one GPU for `batch` frames of N steps: the kernels give every
    (frame, window) its own thread, so a small batch wants shorter windows (each pays 96 warm-up steps either side).
    Pass the result to `set_map_window`; the library default (1024) does not look at the batch, so that a frame decodes
    identically whatever it is batched with -- pinning ANY fixed window keeps that property."""
    nwin = max(1, -(-int(target_threads) // max(1, int(batch))))
    w = (int(N) // nwin) // 8 * 8
    return int(min(1024, max(128, w)))


def set_map_window(steps):
    """cpb_set_option(CPB_OPT_BCJR_WINDOW): 0 restores the default (1024-step windows)."""
    _lib.set_option(_lib.OPT_BCJR_WINDOW, int(steps))


def _checked_perm(interleaver, N):
    """p_array as int32, validated: the kernels gather / scatter through it, so it must be a permutation of 0..N-1 (the
    reference raises IndexError on an out-of-range entry; a repeated entry would leave part of the output unwritten)"""
    perm_np = np.ascontiguousarray(interleaver.p_array, dtype=np.int64)
    if len(perm_np) != N:
        raise ValueError("interleaver length does not match the frame length")
    if N and (perm_np.min() < 0 or perm_np.max() >= N):
        raise IndexError("interleaver.p_array holds an index outside [0, %d)" % N)
    if np.unique(perm_np).size != N:
        raise ValueError("interleaver.p_array is not a permutation")
    return perm_np.astype(np.int32)


def map_decode(sys_symbols, non_sys_symbols, trellis, noise_variance, L_int, mode="decode"):
    """Drop-in for commpy.channelcoding.map_decode (turbo.py:163-251): returns [L_ext, decoded_bits].

    `L_ext` is, as in the reference, the full a-posteriori LLR  L_int + log(app1/app0)  (:145-146);
    `decoded_bits` is (L_ext > 0) in mode 'decode' and zeros in mode 'compute' (:148-152)."""
    L, bits = map_decode_batch_host(np.asarray(sys_symbols)[None, :], np.asarray(non_sys_symbols)[None, :], trellis,
                                    noise_variance, np.asarray(L_int)[None, :], mode)
    return [L[0].astype(np.float64), bits[0].astype("int")]


def turbo_decode_batch(sys_symbols, non_sys_symbols_1, non_sys_symbols_2, trellis, noise_variance,
                       number_iterations, interleaver, L_int=None):
    """Batched turbo decoder: (batch, N) inputs -> (batch, N) uint8 torch CUDA tensor."""
    torch = _lib.require_cuda()
    s = _dev_f32(sys_symbols, torch)
    p1 = _dev_f32(non_sys_symbols_1, torch)
    p2 = _dev_f32(non_sys_symbols_2, torch)
    if s.dim() != 2 or s.shape != p1.shape or s.shape != p2.shape:
        raise ValueError("the three symbol streams must share the shape (batch, N)")
    batch, N = s.shape
    perm_np = _checked_perm(interleaver, N)
    perm = torch.from_numpy(perm_np).cuda()
    la = None if L_int is None else _dev_f32(L_int, torch)
    bits = torch.empty((batch, N), dtype=torch.uint8, device=s.device)
    rc = _lib.load().cpb_turbo_decode(_trellis_handle(trellis), _lib.ptr(s), _lib.ptr(p1), _lib.ptr(p2), _lib.ptr(perm),
                                      C.c_int64(batch), C.c_int64(N), C.c_float(noise_variance),
                                      int(number_iterations), _lib.ptr(la), _lib.ptr(bits), C.c_void_p(0), C.c_size_t(0),
                                      _lib.stream_ptr(torch))
    _lib.check(rc, "turbo_decode")
    return bits


def turbo_decode(sys_symbols, non_sys_symbols_1, non_sys_symbols_2, trellis, noise_variance,
                 number_iterations, interleaver, L_int=None):
    """Drop-in for commpy.channelcoding.turbo_decode (turbo.py:254-333): 1-D in, 1-D int out.

    Keeps the reference's loop exactly, including the systematic double counting (only the prior is removed
    from each decoder's output, :318 and :328) and the final de-interleave of decoder 2's hard decisions (:331)."""
    la = None if L_int is None else np.asarray(L_int)[None, :]
    bits = turbo_decode_batch_host(np.asarray(sys_symbols)[None, :], np.asarray(non_sys_symbols_1)[None, :],
                                   np.asarray(non_sys_symbols_2)[None, :], trellis, noise_variance, number_iterations,
                                   interleaver, la)
    return bits[0].astype("int")

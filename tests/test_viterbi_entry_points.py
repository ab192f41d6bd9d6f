"""The status every Viterbi C entry point returns for bad arguments, the workspace sizes it reports and the fast-path id of
each trellis.

Several arguments are wrong at once in some rows: the order of the checks decides which status comes back, and a caller
(the Python wrappers included) maps that status to an exception type.  Every rejected call must be rejected on the host
before anything is launched, so its output buffer still holds the sentinel afterwards; the calls that succeed decode an
all-zero code word and must return all-zero bits.  Pointers are null or real buffers of the stated size, never made up.
"""
import ctypes as C

import numpy as np
import pytest

import helpers
from commpy_b200 import _lib
from commpy_b200.channelcoding.convcode import _trellis_handle

pytestmark = pytest.mark.gpu

OK, EINVAL, EUNSUP = _lib.CPB_OK, _lib.CPB_EINVAL, _lib.CPB_EUNSUPPORTED
U8, F32 = _lib.CPB_U8, _lib.CPB_F32
HARD, SOFT, UNQ = 0, 1, 2
SENTINEL = 0xAB
NULL = C.c_void_p(0)
B = 5                                    # frames per call: not a multiple of the 32 or 64 frames of a CTA
PV = np.array([1, 1, 1, 0, 0, 1], np.int32)     # keeps 4 of every 6 coded values


def _need(n_depunct):
    """values the depuncturing of n_depunct positions consumes with PV"""
    return int((PV[np.arange(n_depunct) % len(PV)] == 1).sum())


@pytest.fixture(scope="module")
def env():
    torch = _lib.require_cuda()
    lib = _lib.load()
    keep = {"k7": helpers.k7(), "k3": helpers.reference_test_trellises()[0]}     # a handle lives as long as its Trellis
    h = {name: _trellis_handle(tr) for name, tr in keep.items()}
    yield torch, lib, h


def _coded(torch, n_in, dtype, batch=B):
    """an all-zero code word in the input format of dtype (float: -1, which favours bit 0 in every soft mode)"""
    if dtype == U8:
        return torch.zeros((max(batch, 1), max(n_in, 1)), dtype=torch.uint8, device="cuda")
    return torch.full((max(batch, 1), max(n_in, 1)), -1.0, dtype=torch.float32, device="cuda")


def _out(torch, nbytes, batch=B):
    return torch.full((max(batch, 1), max(nbytes, 1)), SENTINEL, dtype=torch.uint8, device="cuda")


def _settle(torch, rc, want, out):
    torch.cuda.synchronize()
    assert rc == want
    if out is None:
        return
    o = out.cpu().numpy() if hasattr(out, "cpu") else out
    if want == OK:
        assert (o == 0).all()
    else:
        assert (o == SENTINEL).all(), "a rejected call wrote its output"


# ------------------------------------------------------------------------------------------------ cpb_viterbi_decode
# (trellis, dtype, batch, n_in, tb_depth, mode, null_in, null_out, status)
DECODE = [
    ("k7", U8, B, 2048, 0, 3, False, False, EINVAL),          # mode
    ("k7", U8, B, 2048, 0, -1, False, False, EINVAL),
    (None, U8, 0, 2048, 0, 3, True, True, EINVAL),            # mode before everything
    ("k7", U8, 0, 2048, 0, 3, False, False, EINVAL),          # mode before the empty batch
    ("k7", 7, 0, -4, 1, HARD, True, True, OK),                # empty batch before nulls, dtype, sizes
    ("k7", U8, 0, 2048, 0, HARD, True, True, OK),
    (None, U8, 0, 2048, 0, HARD, False, False, EINVAL),
    (None, U8, B, 2048, 0, HARD, False, False, EINVAL),
    ("k7", U8, B, 2048, 0, HARD, True, False, EINVAL),
    ("k7", U8, B, 2048, 0, HARD, False, True, EINVAL),
    ("k7", U8, -1, 2048, 0, HARD, False, False, EINVAL),
    ("k7", U8, B, -2, 0, HARD, False, False, EINVAL),
    ("k7", 2, B, 2048, 0, HARD, False, False, EINVAL),        # dtype
    ("k7", -1, B, 2048, 0, SOFT, False, False, EINVAL),
    ("k7", U8, B, 2048, 0, SOFT, False, False, EINVAL),       # soft / unquantized need float
    ("k7", U8, B, 2048, 0, UNQ, False, False, EINVAL),
    ("k7", F32, B, 2048, 0, HARD, False, False, OK),          # hard takes float too
    ("k7", U8, B, 0, 0, HARD, False, False, EINVAL),          # L = 0
    ("k7", F32, B, 1, 0, SOFT, False, False, EINVAL),
    ("k7", U8, B, 2048, 1, HARD, False, False, EINVAL),       # D < 2
    ("k7", U8, B, 40, 27, HARD, False, False, EINVAL),        # T = 25 < D - 1
    ("k7", U8, B, 40, 26, HARD, False, False, OK),            # T = D - 1
    ("k3", U8, B, 40, 24, HARD, False, False, EINVAL),        # T = 21 < D - 1 (generic)
    ("k3", U8, B, 40, 22, HARD, False, False, OK),
    ("k3", F32, B, 2048, 1, UNQ, False, False, EINVAL),
    ("k7", U8, B, 4, 0, HARD, False, False, OK),              # D = L = 2
    ("k7", F32, B, 2048, 47, SOFT, False, False, OK),         # deeper than the fast path: generic kernel
    ("k7", U8, 1, 2 * (2 ** 24 - 4), 0, HARD, False, False, EINVAL),   # T = 2^24 + 1
]


@pytest.mark.parametrize("tr,dtype,batch,n_in,tb,mode,null_in,null_out,want", DECODE)
def test_decode_status(env, tr, dtype, batch, n_in, tb, mode, null_in, null_out, want):
    torch, lib, h = env
    x = _coded(torch, n_in, dtype if dtype in (U8, F32) else U8, batch)
    out = None if null_out else _out(torch, n_in // 2, batch)
    rc = lib.cpb_viterbi_decode(h[tr] if tr else NULL, NULL if null_in else _lib.ptr(x), dtype, C.c_int64(batch),
                                C.c_int64(n_in), tb, mode, _lib.ptr(out), NULL, C.c_size_t(0), _lib.stream_ptr(torch))
    _settle(torch, rc, want, out if batch > 0 else None)


# ------------------------------------------------------------------------------------------------ cpb_viterbi_decode_packed
# (trellis, batch, n_in, tb_depth, null_in, null_out, status)
PACKED = [
    ("k7", 0, 0, 1, True, True, OK),                          # empty batch before everything
    (None, 0, 2048, 0, False, False, EINVAL),
    ("k7", B, 2048, 0, True, False, EINVAL),
    ("k7", B, 2048, 0, False, True, EINVAL),
    ("k7", -1, 2048, 0, False, False, EINVAL),
    ("k7", B, 0, 0, False, False, EINVAL),
    ("k7", B, -8, 0, False, False, EINVAL),
    ("k7", B, 2048, 1, False, False, EINVAL),                 # D < 2
    ("k3", B, 2048, 1, False, False, EINVAL),                 # ... before "not fast"
    ("k7", B, 2044, 1, False, False, EINVAL),                 # ... before n_in % 8
    ("k7", B, 48, 32, False, False, EINVAL),                  # T = 29 < D - 1 before (D - 2) % 4
    ("k7", B, 2048, 0, False, False, OK),
    ("k7", B, 2048, 10, False, False, OK),
    ("k7", B, 2048, 46, False, False, OK),
    ("k3", B, 2048, 0, False, False, EUNSUP),                 # not fast
    ("k7", B, 2048, 50, False, False, EUNSUP),                # D > 46
    ("k7", B, 2052, 0, False, False, EUNSUP),                 # n_in % 8
    ("k7", B, 2056, 0, False, False, EUNSUP),                 # L % 8
    ("k7", B, 2048, 31, False, False, EUNSUP),                # (D - 2) % 4
]


@pytest.mark.parametrize("tr,batch,n_in,tb,null_in,null_out,want", PACKED)
def test_decode_packed_status(env, tr, batch, n_in, tb, null_in, null_out, want):
    torch, lib, h = env
    x = torch.zeros((max(batch, 1), max(n_in // 8, 1)), dtype=torch.uint8, device="cuda")
    out = None if null_out else _out(torch, n_in // 16, batch)
    rc = lib.cpb_viterbi_decode_packed(h[tr] if tr else NULL, NULL if null_in else _lib.ptr(x), C.c_int64(batch),
                                       C.c_int64(n_in), tb, _lib.ptr(out), _lib.stream_ptr(torch))
    _settle(torch, rc, want, out if batch > 0 else None)


# ------------------------------------------------------------------------------------------------ cpb_viterbi_decode_punctured
# (trellis, batch, n_kept, punct_len, n_depunct, tb_depth, mode, nulls, workspace, status); nulls names the null pointers
# among in / out / pv; workspace: None = library scratch, d = caller workspace of (reported size + d) bytes
N_DEP = 2048
KEPT = _need(N_DEP)
PUNCT = [
    ("k7", B, KEPT, 6, N_DEP, 0, HARD, "", None, EINVAL),                # mode
    ("k7", B, KEPT, 6, N_DEP, 0, 3, "", None, EINVAL),
    (None, 0, KEPT, 6, N_DEP, 0, HARD, "in,out,pv", None, EINVAL),      # mode before everything
    ("k7", 0, -1, 0, 0, 1, SOFT, "in,out,pv", None, OK),                # empty batch before nulls and sizes
    (None, B, KEPT, 6, N_DEP, 0, SOFT, "", None, EINVAL),
    ("k7", B, KEPT, 6, N_DEP, 0, SOFT, "in", None, EINVAL),
    ("k7", B, KEPT, 6, N_DEP, 0, SOFT, "out", None, EINVAL),
    ("k7", B, KEPT, 6, N_DEP, 0, SOFT, "pv", None, EINVAL),
    ("k7", -1, KEPT, 6, N_DEP, 0, SOFT, "", None, EINVAL),
    ("k7", B, -1, 6, N_DEP, 0, SOFT, "", None, EINVAL),
    ("k7", B, KEPT, 6, 0, 0, SOFT, "", None, EINVAL),
    ("k7", B, KEPT, 0, N_DEP, 0, SOFT, "in", None, EINVAL),             # nulls before the pattern length
    ("k7", B, KEPT, 0, N_DEP, 0, SOFT, "", None, EUNSUP),               # pattern length
    ("k7", B, KEPT, 33, N_DEP, 0, SOFT, "", None, EUNSUP),
    ("k7", B, 0, 33, N_DEP, 0, SOFT, "", None, EUNSUP),                 # ... before the kept count
    ("k7", B, KEPT - 1, 6, N_DEP, 0, SOFT, "", None, EINVAL),           # too few kept values
    ("k3", B, KEPT - 1, 6, N_DEP, 0, UNQ, "", None, EINVAL),            # ... before "not fast"
    ("k7", B, KEPT - 1, 6, N_DEP, 1, SOFT, "", None, EINVAL),
    ("k7", B, KEPT, 6, N_DEP, 1, SOFT, "", None, EINVAL),               # D < 2
    ("k3", B, KEPT, 6, N_DEP, 1, SOFT, "", None, EINVAL),               # ... before "not fast"
    ("k7", B, _need(40), 6, 40, 27, SOFT, "", None, EINVAL),            # T = 25 < D - 1
    ("k7", B, _need(40), 6, 40, 26, SOFT, "", None, OK),
    ("k3", B, KEPT, 6, N_DEP, 0, SOFT, "", None, EUNSUP),               # not fast
    ("k7", B, KEPT, 6, N_DEP, 47, UNQ, "", None, EUNSUP),               # D > 46
    ("k3", B, KEPT, 6, N_DEP, 0, SOFT, "", -1, EUNSUP),                 # "not fast" before the workspace
    ("k7", B, KEPT, 6, N_DEP, 0, SOFT, "", -1, EINVAL),                 # workspace one byte short
    ("k7", B, KEPT, 6, N_DEP, 0, SOFT, "", 0, OK),
    ("k7", B, KEPT + 7, 6, N_DEP, 0, UNQ, "", None, OK),
    ("k7", B, N_DEP, 32, N_DEP, 0, SOFT, "", None, OK),      # every position kept
]


@pytest.mark.parametrize("tr,batch,n_kept,plen,n_dep,tb,mode,nulls,ws,want", PUNCT)
def test_decode_punctured_status(env, tr, batch, n_kept, plen, n_dep, tb, mode, nulls, ws, want):
    torch, lib, h = env
    pv = np.ones(32, np.int32) if plen == 32 else np.resize(PV, max(plen, 1))
    x = _coded(torch, n_kept, F32, batch)
    out = _out(torch, n_dep // 2, batch)
    wbuf, wbytes = None, 0
    if ws is not None:
        size = C.c_size_t()
        assert lib.cpb_viterbi_punctured_workspace_bytes(C.c_int64(batch), C.byref(size)) == OK
        wbytes = size.value + ws
        wbuf = torch.empty(wbytes, dtype=torch.uint8, device="cuda")
    rc = lib.cpb_viterbi_decode_punctured(
        h[tr] if tr else NULL, NULL if "in" in nulls else _lib.ptr(x), C.c_int64(batch), C.c_int64(n_kept),
        NULL if "pv" in nulls else _lib.ptr(np.ascontiguousarray(pv, np.int32)), plen, C.c_int64(n_dep), tb, mode,
        NULL if "out" in nulls else _lib.ptr(out), _lib.ptr(wbuf), C.c_size_t(wbytes), _lib.stream_ptr(torch))
    _settle(torch, rc, want, out if batch > 0 else None)


# ------------------------------------------------------------------------------------------------ host-buffer forms
# (trellis, dtype, batch, n_in, tb_depth, mode, null_in, null_out, status)
HOST = [
    (None, 7, 0, 2048, 0, HARD, True, True, EINVAL),          # dtype before everything
    ("k7", 2, B, 2048, 0, HARD, False, False, EINVAL),
    ("k7", U8, 0, -4, 1, 3, True, True, OK),                  # empty batch before nulls, sizes and mode
    (None, U8, B, 2048, 0, HARD, False, False, EINVAL),
    ("k7", U8, B, 2048, 0, HARD, True, False, EINVAL),
    ("k7", U8, B, 2048, 0, HARD, False, True, EINVAL),
    ("k7", U8, -1, 2048, 0, HARD, False, False, EINVAL),
    ("k7", U8, B, 0, 0, HARD, False, False, EINVAL),
    ("k7", U8, B, 2048, 0, 3, False, False, EINVAL),          # then exactly cpb_viterbi_decode
    ("k7", U8, B, 2048, 0, SOFT, False, False, EINVAL),
    ("k7", U8, B, 2048, 1, HARD, False, False, EINVAL),
    ("k7", U8, B, 40, 27, HARD, False, False, EINVAL),
    ("k7", U8, B, 2048, 0, HARD, False, False, OK),
    ("k7", F32, B, 2048, 0, UNQ, False, False, OK),
    ("k3", F32, B, 2048, 15, SOFT, False, False, OK),
]


@pytest.mark.parametrize("tr,dtype,batch,n_in,tb,mode,null_in,null_out,want", HOST)
def test_decode_host_status(env, tr, dtype, batch, n_in, tb, mode, null_in, null_out, want):
    torch, lib, h = env
    shape = (max(batch, 1), max(n_in, 1))
    x = np.full(shape, -1.0, np.float32) if dtype == F32 else np.zeros(shape, np.uint8)
    out = np.full((max(batch, 1), max(n_in // 2, 1)), SENTINEL, np.uint8)
    rc = lib.cpb_viterbi_decode_host(h[tr] if tr else NULL, NULL if null_in else _lib.ptr(x), dtype, C.c_int64(batch),
                                     C.c_int64(n_in), tb, mode, NULL if null_out else _lib.ptr(out))
    _settle(torch, rc, want, out if batch > 0 and not null_out else None)


# (trellis, batch, n_in, tb_depth, null_in, null_out, status)
HOST_PACKED = [
    ("k7", 0, 0, 1, True, True, OK),
    (None, B, 2048, 0, False, False, EINVAL),
    ("k7", B, 2048, 0, True, False, EINVAL),
    ("k7", B, 2048, 0, False, True, EINVAL),
    ("k7", -1, 2048, 0, False, False, EINVAL),
    ("k7", B, 0, 0, False, False, EINVAL),
    ("k7", B, 2052, 0, False, False, EINVAL),                 # n_in % 8: EINVAL here, EUNSUPPORTED on the device
    ("k7", B, 2056, 0, False, False, EUNSUP),                 # L % 8
    ("k7", B, 2056, 1, False, False, EUNSUP),                 # ... before the depth
    ("k7", B, 2048, 1, False, False, EINVAL),                 # then exactly cpb_viterbi_decode_packed
    ("k3", B, 2048, 0, False, False, EUNSUP),
    ("k7", B, 2048, 31, False, False, EUNSUP),
    ("k7", B, 2048, 0, False, False, OK),
]


@pytest.mark.parametrize("tr,batch,n_in,tb,null_in,null_out,want", HOST_PACKED)
def test_decode_host_packed_status(env, tr, batch, n_in, tb, null_in, null_out, want):
    torch, lib, h = env
    x = np.zeros((max(batch, 1), max(n_in // 8, 1)), np.uint8)
    out = np.full((max(batch, 1), max(n_in // 16, 1)), SENTINEL, np.uint8)
    rc = lib.cpb_viterbi_decode_host_packed(h[tr] if tr else NULL, NULL if null_in else _lib.ptr(x), C.c_int64(batch),
                                            C.c_int64(n_in), tb, NULL if null_out else _lib.ptr(out))
    _settle(torch, rc, want, out if batch > 0 and not null_out else None)


# ------------------------------------------------------------------------------------------------ workspace sizes
def test_workspace_queries_reject_bad_arguments(env):
    torch, lib, h = env
    size = C.c_size_t()
    assert lib.cpb_viterbi_workspace_bytes(NULL, C.c_int64(B), C.c_int64(2048), 0, HARD, C.byref(size)) == EINVAL
    assert lib.cpb_viterbi_workspace_bytes(h["k7"], C.c_int64(B), C.c_int64(2048), 0, HARD, NULL) == EINVAL
    assert lib.cpb_viterbi_workspace_bytes(h["k7"], C.c_int64(-1), C.c_int64(2048), 0, HARD, C.byref(size)) == EINVAL
    assert lib.cpb_viterbi_punctured_workspace_bytes(C.c_int64(B), NULL) == EINVAL
    assert lib.cpb_viterbi_punctured_workspace_bytes(C.c_int64(-1), C.byref(size)) == EINVAL
    assert lib.cpb_viterbi_punctured_workspace_bytes(C.c_int64(0), C.byref(size)) == OK and size.value == 256
    assert lib.cpb_viterbi_punctured_workspace_bytes(C.c_int64(1000), C.byref(size)) == OK and size.value == 4256


# (trellis, dtype, mode, tb_depth, reported size, bytes the decode acquires)
WORKSPACE = [
    ("k7", U8, HARD, 0, 256, 256),                            # fast hard: nothing but the alignment slack
    ("k7", F32, SOFT, 0, 256 + 4 * B, 256 + 4 * B),           # fast float: one scale per frame
    ("k7", F32, UNQ, 46, 256 + 4 * B, 256 + 4 * B),
    ("k7", F32, SOFT, 47, None, None),                        # generic: 256 bytes more than the decode acquires
    ("k3", U8, HARD, 0, None, None),
    ("k3", F32, UNQ, 15, None, None),
]


@pytest.mark.parametrize("tr,dtype,mode,tb,reported,acquired", WORKSPACE)
def test_decode_workspace_size(env, tr, dtype, mode, tb, reported, acquired):
    torch, lib, h = env
    n_in = 2048
    size = C.c_size_t()
    assert lib.cpb_viterbi_workspace_bytes(h[tr], C.c_int64(B), C.c_int64(n_in), tb, mode, C.byref(size)) == OK
    if reported is None:
        # survivors: (T + 1) * (S + 1) bytes per frame, for the batch rounded up to the generic kernel's 64 frames
        T = n_in // 2 + (6 if tr == "k7" else 2) - 1
        S = 64 if tr == "k7" else 4
        acquired = (T + 1) * (S + 1) * 64
        reported = acquired + 256
    assert size.value == reported
    x = _coded(torch, n_in, dtype)
    for nbytes, want in ((reported, OK), (acquired, OK), (acquired - 1, EINVAL)):
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        out = _out(torch, n_in // 2)
        rc = lib.cpb_viterbi_decode(h[tr], _lib.ptr(x), dtype, C.c_int64(B), C.c_int64(n_in), tb, mode, _lib.ptr(out),
                                    _lib.ptr(ws), C.c_size_t(nbytes), _lib.stream_ptr(torch))
        _settle(torch, rc, want, out)


def test_punctured_workspace_size(env):
    torch, lib, h = env
    size = C.c_size_t()
    assert lib.cpb_viterbi_punctured_workspace_bytes(C.c_int64(B), C.byref(size)) == OK
    assert size.value == 256 + 4 * B
    x = _coded(torch, KEPT, F32)
    for nbytes, want in ((size.value, OK), (size.value - 1, EINVAL)):
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        out = _out(torch, N_DEP // 2)
        rc = lib.cpb_viterbi_decode_punctured(h["k7"], _lib.ptr(x), C.c_int64(B), C.c_int64(KEPT), _lib.ptr(PV), len(PV),
                                              C.c_int64(N_DEP), 0, SOFT, _lib.ptr(out), _lib.ptr(ws), C.c_size_t(nbytes),
                                              _lib.stream_ptr(torch))
        _settle(torch, rc, want, out)


# ------------------------------------------------------------------------------------------------ fast-path ids
def test_trellis_fast_path_ids(env):
    torch, lib, h = env
    trellises = [helpers.k7(), helpers.k7_171_133(), helpers.k7_wifi_quirk(), helpers.mem6_5_7(), helpers.rsc_k4()]
    trellises += helpers.reference_test_trellises()
    got = [lib.cpb_trellis_fast_path(_trellis_handle(tr)) for tr in trellises]
    assert got == [1, 2, 3, 4] + [0] * 6
    assert lib.cpb_trellis_fast_path(NULL) == 0

"""Every kernel instance the C entry points dispatch to, against the fp64 oracle (oracle/oracle.py) or an fp64 NumPy /
SciPy restatement of the same operation, at the shapes that select it.  Each test asserts, through the CUDA profiler,
that the kernel it names actually ran, so a later change of a dispatch threshold fails here instead of quietly moving
the test onto another kernel.  Library-vs-library comparisons appear only where the contract is bit identity between
two paths of the same arithmetic: host pipeline vs device entry, a frame in a big batch vs alone, bulk vs
register-staged LDPC check pass, frame-major vs step-major turbo loop."""
import ctypes as C
import functools
import os
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import helpers
from oracle import oracle
from commpy_b200 import _lib
from commpy_b200.channelcoding import (RandInterlv, Trellis, depuncturing, ldpc_bp_decode_batch, map_decode_batch,
                                        map_decode_batch_host, puncturing, turbo_decode_batch, turbo_decode_batch_host,
                                        turbo_encode, viterbi_decode_batch, viterbi_decode_punctured_batch)
from commpy_b200.channelcoding.convcode import _trellis_handle
from commpy_b200.channelcoding.ldpc import ldpc_bp_decode_batch_host
from commpy_b200.modulation import Modem, PSKModem, QAMModem

gpu = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MAP_ATOL, MAP_RTOL = 1e-4, 1e-4                   # the tolerances of tests/test_decoders_gpu.py (SURVEY.md section 8c)
DEMAP_ATOL, DEMAP_RTOL = 5e-4, 5e-4


# ---------------------------------------------------------------- which kernel ran
@functools.lru_cache(maxsize=None)
def _profiler_sees_library():
    """True when the profiler records a kernel the ctypes library launched (demod_hard_kernel on a 1-symbol input)."""
    y = torch.zeros(1, dtype=torch.complex64, device="cuda")
    names = helpers.launched_kernels(lambda: QAMModem(4).demodulate_batch(y, "hard"))
    return any("demap::demod_hard_kernel" in n for n in names)


def _ran(fn, want=(), absent=()):
    """fn() under the profiler; asserts that a kernel name containing each `want` substring ran and none containing an
    `absent` one did (normalised names: helpers.normalize_kernel_name).  Returns fn's result."""
    want = [want] if isinstance(want, str) else list(want)
    absent = [absent] if isinstance(absent, str) else list(absent)
    # a profiling session now and then records the API calls but none of the kernel activity; such a session is
    # repeated (at most twice), and the absent kernels are checked on the session that recorded the wanted ones
    for _ in range(3):
        box = []
        names = helpers.launched_kernels(lambda: box.append(fn()))
        if not _profiler_sees_library():
            pytest.skip("torch.profiler does not record the kernels of libcommpy_b200.so on this system: "
                        "the dispatch of this path cannot be checked")
        if all(any(w in n for n in names) for w in want):
            break
    for w in want:
        assert any(w in n for n in names), (w, sorted(names))
    for a in absent:
        assert not any(a in n for n in names), (a, sorted(names))
    return box[0]


def test_normalize_kernel_name_matches_both_demanglings():
    a = "void fast::viterbi_fast_kernel_hard<FFCode<(int)6, (unsigned int)5, (unsigned int)7>>(fast::Params)"
    b = "void fast::viterbi_fast_kernel_hard<FFCode<6, 5u, 7u> >(fast::Params)"
    assert helpers.normalize_kernel_name(a) == helpers.normalize_kernel_name(b)
    assert "viterbi_fast_kernel_hard<FFCode<6,5,7>>" in helpers.normalize_kernel_name(b)
    c = "void bcjr::tpf::map_lin2_kernel<bcjr::tpf::CT<(int)4, (unsigned long long)2986128, (unsigned int)39372>, (bool)0>(p)"
    d = "void bcjr::tpf::map_lin2_kernel<bcjr::tpf::CT<4, 2986128ull, 39372u>, false>(p)"
    assert "tpf::CT<4,2986128,39372>" in helpers.normalize_kernel_name(c)
    assert "tpf::CT<4,2986128,39372>" in helpers.normalize_kernel_name(d)


def test_mixed_degree_H_has_the_requested_degrees():
    degs = [2] * 30 + list(range(3, 17)) * 3 + [32]
    H = helpers.mixed_degree_H(degs, 300, seed=1)
    assert np.array_equal(np.diff(H.indptr), degs)
    assert H.max() == 1 and (np.asarray(H.sum(axis=0)) > 0).all()


@gpu
def test_launched_kernels_sees_library_kernels():
    """The profiler records kernels launched through ctypes on the library's own streams (host pipeline), not only
    torch's: demod_hard_kernel on the current stream and demod_soft_separable<2> inside cpb_demod_soft_host."""
    if not _profiler_sees_library():
        pytest.skip("torch.profiler does not record the kernels of libcommpy_b200.so on this system")
    q = QAMModem(16)
    names = helpers.launched_kernels(lambda: q.demodulate(np.array([0.5 + 1.5j, -3 - 1j]), "soft", 1.0))
    assert any("demap::demod_soft_separable<2>" in n for n in names), sorted(names)
    assert not any("demod_soft_general" in n for n in names)


# ---------------------------------------------------------------- Viterbi
def _tr(mem, gens, fb=None, ct="default"):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if fb is None:
            return Trellis(np.array(mem), np.array(gens))
        return Trellis(np.array(mem), np.array(gens), np.array(fb) if isinstance(fb, list) else fb, ct)


# the four codes with register-resident kernels (viterbi.cu, Code133_171 .. Code5_7) and their template arguments
FAST_CODES = {
    "133_171": (helpers.k7, "FFCode<6,91,121>"),
    "171_133": (helpers.k7_171_133, "FFCode<6,121,91>"),
    "decimal_quirk": (helpers.k7_wifi_quirk, "FFCode<6,5,43>"),
    "5_7_mem6": (helpers.mem6_5_7, "FFCode<6,5,7>"),
}


def _dev(x, hard):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.uint8 if hard else np.float32)).cuda()


def _vit(x, tr, tb, mode, force_generic=False, **kw):
    _lib.set_option(_lib.OPT_VITERBI_FORCE_GENERIC, int(force_generic))
    try:
        return viterbi_decode_batch(_dev(x, mode == "hard"), tr, tb, mode, **kw).cpu().numpy()
    finally:
        _lib.set_option(_lib.OPT_VITERBI_FORCE_GENERIC, 0)


@gpu
@pytest.mark.parametrize("code", sorted(FAST_CODES))
def test_fast_codes_every_kernel_vs_oracle(code):
    """Byte hard, bit-packed hard, soft, unquantized and punctured (soft, unquantized) kernels of each fast code."""
    make, tag = FAST_CODES[code]
    tr = make()
    rs = np.random.RandomState(51)
    for mode in ("hard", "soft", "unquantized"):
        _, x = helpers.channel_frames(tr, rs, 70, 1024, mode, "cont", flip=0.06, ebn0_db=2.5)
        want = oracle.viterbi_decode_batch(x, tr, None, mode, threads=8)
        kern = "viterbi_fast_kernel_%s<%s>" % ("hard" if mode == "hard" else "soft", tag)
        got = _ran(lambda: _vit(x, tr, None, mode), kern)
        if mode == "hard":
            assert np.array_equal(got, want)
            xp = torch.from_numpy(np.packbits(x.astype(np.uint8), axis=1)).cuda()
            gp = _ran(lambda: viterbi_decode_batch(xp, tr, None, "hard", packed=True).cpu().numpy(),
                      "viterbi_fast_kernel_hard_packed<%s>" % tag)
            assert np.array_equal(np.unpackbits(gp, axis=1), want)
        else:
            assert (got != want).mean() <= 1e-4, (mode, int((got != want).sum()))
            pv = [1, 1, 1, 0, 0, 1]
            rows = np.stack([puncturing(r, pv) for r in x])
            gotp = _ran(lambda: viterbi_decode_punctured_batch(rows.astype(np.float32), tr, pv, x.shape[1], None,
                                                               mode).cpu().numpy(),
                        "viterbi_fast_kernel_soft_punct<%s>" % tag)
            dep = np.stack([depuncturing(r, pv, x.shape[1]) for r in rows])
            wantp = oracle.viterbi_decode_batch(dep, tr, None, mode, threads=8)
            assert (gotp != wantp).mean() <= 2e-4, (mode, int((gotp != wantp).sum()))


DYADIC = np.array([-2.0, -1.0, -0.5, 0.0, 0.5, 1.0, 2.0])


@gpu
@pytest.mark.parametrize("code", sorted(FAST_CODES))
def test_exact_ties_bit_exact_fast_and_generic(code):
    """Inputs where many paths tie exactly, decoded bit-exactly like the oracle by the fast kernels and by the generic one.
    hard: pure noise (flip = 0.5), all-ones and alternating rows.  unquantized: values on the dyadic grid {-2 .. 2}, where
    the oracle's squared Euclidean metric is exact in fp64 and the per-frame power-of-two scale maps every value (and the
    -1 padding) exactly into the kernel's fixed point; the kernel metric equals the oracle's up to a factor 4 and a
    per-step constant, so every comparison -- ties included -- goes the same way.  soft: all-zero rows, every branch ties."""
    make, tag = FAST_CODES[code]
    tr = make()
    rs = np.random.RandomState(52)
    for nbits in (200, 1024, 333):
        n_in = 2 * nbits
        alt = np.zeros((4, n_in))
        alt[0] = 1
        alt[1, ::2] = 1
        alt[2, 1::2] = 1
        alt[3, ::4] = 1
        cases = [("hard", helpers.channel_frames(tr, rs, 70, nbits, "hard", "cont", flip=0.5)[1]),
                 ("hard", alt),
                 ("unquantized", rs.choice(DYADIC, (70, n_in))),
                 ("soft", np.zeros((5, n_in)))]
        for tb in (None, 15, 7, 46, 48):
            for mode, x in cases:
                want = oracle.viterbi_decode_batch(x, tr, tb, mode, threads=8)
                fast_ok = tb != 48                              # 48 > the deepest traceback of the fast kernels
                for force in (False, True):
                    if nbits == 200 and tb in (None, 48):
                        if force or not fast_ok:
                            kern, other = "gen::viterbi_generic_kernel", "viterbi_fast_kernel"
                        else:
                            kern = "viterbi_fast_kernel_%s<%s>" % ("hard" if mode == "hard" else "soft", tag)
                            other = "viterbi_generic_kernel"
                        got = _ran(lambda: _vit(x, tr, tb, mode, force), kern, other)
                    else:
                        got = _vit(x, tr, tb, mode, force)
                    assert np.array_equal(got, want), (mode, nbits, tb, force, int((got != want).sum()))
                if mode == "hard" and n_in % 16 == 0 and tb in (None, 46):
                    xp = torch.from_numpy(np.packbits(x.astype(np.uint8), axis=1)).cuda()
                    gp = viterbi_decode_batch(xp, tr, tb, "hard", packed=True).cpu().numpy()
                    assert np.array_equal(np.unpackbits(gp, axis=1), want), (nbits, tb)


def _ff_encode(msgs, g0, g1, mem=6):
    """Rate-1/2 feed-forward encoder ('cont') as a mod-2 convolution: generator bit b taps the input b steps back
    (the Trellis convention of viterbi.cu FFCode)."""
    out = np.zeros((msgs.shape[0], 2 * msgs.shape[1]), np.uint8)
    m = msgs.astype(np.uint8)
    for j, g in enumerate((g0, g1)):
        for b in range(mem + 1):
            if (g >> b) & 1:
                out[:, j::2][:, b:] ^= m[:, :m.shape[1] - b]
    return out


@gpu
def test_long_frames_metric_renormalisation():
    """4 frames of 2^20 information bits: the 6-bit (hard) and 22-bit (float) metric fields renormalise over a million steps."""
    tr = helpers.k7()
    rs = np.random.RandomState(53)
    msgs = rs.randint(0, 2, (4, 1 << 20))
    coded = _ff_encode(msgs, 0o133, 0o171)
    assert np.array_equal(coded[:, :1000], helpers.encode_batch(msgs[:, :500], tr))
    sigma2 = 1.0 / (2 * 0.5 * 10 ** (3.0 / 10))
    y = (2.0 * coded - 1) + np.sqrt(sigma2) * rs.randn(*coded.shape)
    for mode, x in (("hard", np.abs(coded - (rs.rand(*coded.shape) < 0.03))), ("soft", 2 * y / sigma2),
                    ("unquantized", y)):
        want = oracle.viterbi_decode_batch(x, tr, None, mode, threads=4)
        got = _ran(lambda: _vit(x, tr, None, mode),
                   "viterbi_fast_kernel_%s<FFCode<6,91,121>>" % ("hard" if mode == "hard" else "soft"))
        if mode == "hard":
            assert np.array_equal(got, want)
        else:
            assert (got != want).mean() <= 1e-4, (mode, int((got != want).sum()))
        assert abs(int((got != msgs).sum()) - int((want != msgs).sum())) <= max(8, 0.02 * (want != msgs).sum())


@gpu
@pytest.mark.parametrize("mode", ["soft", "unquantized"])
def test_values_past_the_used_length_are_ignored(mode):
    """The last value of an odd-length row and punctured values past the ones the depuncturing consumes take no part in
    the decode -- in particular not in the frame's fixed-point scale (frame_scale_kernel)."""
    tr = helpers.k7()
    rs = np.random.RandomState(54)
    _, x = helpers.channel_frames(tr, rs, 33, 500, mode, "cont", ebn0_db=2.0)
    xo = np.concatenate([x, np.zeros((33, 1))], axis=1)            # 1001 values: L = 500
    base = _ran(lambda: _vit(xo, tr, None, mode), ["fast::frame_scale_kernel", "viterbi_fast_kernel_soft<"])
    want = oracle.viterbi_decode_batch(xo, tr, None, mode, threads=8)
    assert (base != want).mean() <= 1e-4
    for v in (1e30, np.inf, -np.inf):
        xv = xo.copy()
        xv[:, -1] = v
        assert np.array_equal(_vit(xv, tr, None, mode), base), v
    pv = [1, 1, 1, 0, 0, 1]
    rows = np.stack([puncturing(r, pv) for r in x])
    extra = np.zeros((33, 7))
    p0 = viterbi_decode_punctured_batch(np.concatenate([rows, extra], 1).astype(np.float32), tr, pv, 1000, None, mode)
    for v in (1e30, np.inf):
        p1 = _ran(lambda: viterbi_decode_punctured_batch(np.concatenate([rows, extra + v], 1).astype(np.float32), tr, pv,
                                                         1000, None, mode),
                  ["fast::frame_scale_kernel", "viterbi_fast_kernel_soft_punct<FFCode<6,91,121>>"])
        assert torch.equal(p0, p1), v


@gpu
@pytest.mark.parametrize("code", sorted(FAST_CODES))
def test_punctured_patterns_and_partial_periods(code):
    """Punctured decode in 'soft' and 'unquantized' mode with patterns [1], a 32-long one (the longest taken), one that
    starts with an erasure and the 802.11 rate-3/4 one, at frame lengths that end inside a period, against depuncturing()
    followed by the oracle."""
    make, tag = FAST_CODES[code]
    tr = make()
    rs = np.random.RandomState(55)
    p32 = [int(v) for v in rs.rand(32) < 0.75]
    p32[0] = 1
    patterns = ([1], p32, [0, 1, 1, 1, 0, 1], [1, 1, 1, 0, 0, 1])
    for mode in ("soft", "unquantized"):
        for pv in patterns:
            for nbits in (601, 700):
                _, x = helpers.channel_frames(tr, rs, 24, nbits, mode, "cont", ebn0_db=3.5)
                shouldbe = x.shape[1]
                rows = np.stack([puncturing(r, pv) for r in x]).astype(np.float32)
                got = _ran(lambda: viterbi_decode_punctured_batch(rows, tr, pv, shouldbe, None, mode).cpu().numpy(),
                           "viterbi_fast_kernel_soft_punct<%s>" % tag)
                dep = np.stack([depuncturing(r, pv, shouldbe) for r in rows.astype(np.float64)])
                want = oracle.viterbi_decode_batch(dep, tr, None, mode, threads=8)
                assert (got != want).mean() <= 2e-4, (mode, len(pv), nbits, int((got != want).sum()))


@gpu
def test_generic_kernel_across_survivor_chunks():
    """T = 8,192, S = 64: the generic kernel's survivor scratch holds 2,816 frames (viterbi.cu generic_chunk), so 2,900
    frames run as two chunks.  Frames on both sides of the boundary equal the oracle; the second chunk equals those frames
    decoded alone."""
    tr = helpers.k7()
    rs = np.random.RandomState(56)
    _, x = helpers.channel_frames(tr, rs, 2900, 8187, "hard", "cont", flip=0.06)
    per_frame = (8192 + 1) * (64 + 1)
    chunk = int(1.5e9 / per_frame) // 64 * 64
    assert chunk == 2816
    xd = _dev(x, True)
    _lib.set_option(_lib.OPT_VITERBI_FORCE_GENERIC, 1)
    try:
        got = _ran(lambda: viterbi_decode_batch(xd, tr, None, "hard").cpu().numpy(), "gen::viterbi_generic_kernel")
        alone = viterbi_decode_batch(xd[chunk:].contiguous(), tr, None, "hard").cpu().numpy()
    finally:
        _lib.set_option(_lib.OPT_VITERBI_FORCE_GENERIC, 0)
    idx = [0, chunk - 1, chunk, chunk + 1, 2899]
    want = oracle.viterbi_decode_batch(x[idx], tr, None, "hard", threads=5)
    assert np.array_equal(got[idx], want)
    assert np.array_equal(got[chunk:], alone)


@gpu
def test_host_pipelines_across_chunks():
    """cpb_viterbi_decode_host with 40,000 frames runs chunks of 16,384 + 16,384 + 7,232 over all three stream slots;
    the packed host path with 70,000 frames runs 32,768 + 32,768 + 4,464.  Both equal the device-tensor call bit for bit."""
    tr = helpers.k7()
    rs = np.random.RandomState(57)
    for mode in ("hard", "soft"):
        _, x = helpers.channel_frames(tr, rs, 40000, 256, mode, "cont", flip=0.05, ebn0_db=2.0)
        xin = x.astype(np.uint8) if mode == "hard" else x.astype(np.float32)
        host = _ran(lambda: viterbi_decode_batch(xin, tr, None, mode),
                    "viterbi_fast_kernel_%s<FFCode<6,91,121>>" % ("hard" if mode == "hard" else "soft"))
        dev = viterbi_decode_batch(torch.from_numpy(xin).cuda(), tr, None, mode).cpu().numpy()
        assert np.array_equal(host, dev), mode
        idx = [0, 16383, 16384, 32767, 32768, 39999]
        want = oracle.viterbi_decode_batch(x[idx], tr, None, mode, threads=6)
        if mode == "hard":
            assert np.array_equal(host[idx], want)
        else:
            assert (host[idx] != want).mean() <= 1e-3
    _, x = helpers.channel_frames(tr, rs, 70000, 256, "hard", "cont", flip=0.05)
    xp = np.packbits(x.astype(np.uint8), axis=1)
    host = _ran(lambda: viterbi_decode_batch(xp, tr, None, "hard", packed=True),
                "viterbi_fast_kernel_hard_packed<FFCode<6,91,121>>")
    dev = viterbi_decode_batch(torch.from_numpy(xp).cuda(), tr, None, "hard", packed=True).cpu().numpy()
    assert np.array_equal(host, dev)
    idx = [0, 32767, 32768, 65535, 65536, 69999]
    assert np.array_equal(np.unpackbits(host[idx], axis=1), oracle.viterbi_decode_batch(x[idx], tr, None, "hard", threads=6))


# ---------------------------------------------------------------- BCJR / turbo
MAP_CASES = {
    # name: (trellis, kernel of N % 4 == 0, kernel of N % 4 != 0)
    "rsc_k3_legacy": (lambda: _tr([2], [[1, 7]], 5, "rsc"), "tpf::CT<4,2986128,39372>",
                      "map_tpf_kernel<bcjr::tpf::CT<4,2986128,39372>,1>"),
    "table_S2": (lambda: _tr([1], [[1, 3]]), "bcjr::map_kernel<2>", "bcjr::map_kernel<2>"),
    "table_S4": (lambda: _tr([2], [[7, 5]]), "bcjr::map_kernel<4>", "bcjr::map_kernel<4>"),
    "table_S32": (lambda: _tr([5], [[0o53, 0o75]]), "bcjr::map_kernel<32>", "bcjr::map_kernel<32>"),
}


@gpu
@pytest.mark.parametrize("case", sorted(MAP_CASES))
def test_map_instances_vs_oracle(case):
    make, k_al, k_un = MAP_CASES[case]
    tr = make()
    rs = np.random.RandomState(61)
    for N, kern in ((512, k_al), (513, k_un)):
        batch = 6
        msgs = rs.randint(0, 2, (batch, N))
        coded = helpers.encode_batch(msgs, tr, "cont")
        s2 = 0.7
        ys = 2.0 * coded[:, 0::2] - 1 + np.sqrt(s2) * rs.randn(batch, N)
        yp = 2.0 * coded[:, 1::2] - 1 + np.sqrt(s2) * rs.randn(batch, N)
        La = rs.randn(batch, N)
        L, bits = _ran(lambda: map_decode_batch(ys, yp, tr, s2, La, "decode"), kern)
        L, bits = L.cpu().numpy().astype(np.float64), bits.cpu().numpy()
        for b in range(batch):
            Lo, bo = oracle.map_decode(ys[b], yp[b], tr, s2, La[b], "decode")
            err = np.abs(L[b] - Lo) - MAP_RTOL * np.abs(Lo)
            assert (err <= MAP_ATOL).all(), (case, N, b, float(err.max()))
            safe = np.abs(Lo) > 1e-3
            assert np.array_equal(bits[b][safe], bo[safe])


@gpu
def test_map_64_states_is_unsupported():
    tr = helpers.k7()
    z = np.zeros((2, 64))
    with pytest.raises(NotImplementedError):
        map_decode_batch(z, z, tr, 0.5, z)


def _turbo_frames(tr, rs, batch, N, s2):
    il = RandInterlv(N, 5)
    ys, y1, y2 = [], [], []
    for _ in range(batch):
        s_, p1, p2 = turbo_encode(rs.randint(0, 2, N), tr, tr, il)
        ys.append(2.0 * s_[:N] - 1 + np.sqrt(s2) * rs.randn(N))
        y1.append(2.0 * p1[:N] - 1 + np.sqrt(s2) * rs.randn(N))
        y2.append(2.0 * p2[:N] - 1 + np.sqrt(s2) * rs.randn(N))
    return il, np.stack(ys), np.stack(y1), np.stack(y2)


FRAME_MAJOR = ["bcjr::gather_sub_kernel", "bcjr::scatter_sub_kernel", "bcjr::scatter_bits_kernel"]


@gpu
def test_turbo_frame_major_long_frames():
    """N > 24,576 steps: the frame-major turbo loop uses the grid-stride interleaver kernels (no row staging).  N = 30,000
    forced frame-major equals the step-major loop bit for bit; N = 30,001 (N % 4 != 0) and an RSC without a compiled
    instance are frame-major by necessity.  All agree with the oracle."""
    rs = np.random.RandomState(62)
    s2 = 1.0 / (2 * (1 / 3) * 10 ** (1.0 / 10))
    k4 = helpers.rsc_k4()
    other = _tr([3], [[1, 0o17]], [[0o15]], "rsc")
    iters = 4
    il, ys, y1, y2 = _turbo_frames(k4, rs, 3, 30000, s2)
    sm = _ran(lambda: turbo_decode_batch(ys, y1, y2, k4, s2, iters, il).cpu().numpy(), "bcjr::to_step_major_kernel",
              FRAME_MAJOR)
    _lib.set_option(_lib.OPT_TURBO_FRAME_MAJOR, 1)
    try:
        fm = _ran(lambda: turbo_decode_batch(ys, y1, y2, k4, s2, iters, il).cpu().numpy(), FRAME_MAJOR,
                  ["row_gather_sub_kernel", "to_step_major_kernel"])
    finally:
        _lib.set_option(_lib.OPT_TURBO_FRAME_MAJOR, 0)
    assert np.array_equal(sm, fm)
    want = oracle.turbo_decode_batch(ys, y1, y2, k4, s2, iters, il, threads=3)
    assert (fm == want).mean() >= 0.999, float((fm == want).mean())
    for tr, N, extra in ((k4, 30001, []), (other, 30000, ["bcjr::map_kernel<8>"])):
        il, ys, y1, y2 = _turbo_frames(tr, rs, 2, N, s2)
        got = _ran(lambda: turbo_decode_batch(ys, y1, y2, tr, s2, iters, il).cpu().numpy(), FRAME_MAJOR + extra,
                   ["row_gather_sub_kernel", "to_step_major_kernel"])
        want = oracle.turbo_decode_batch(ys, y1, y2, tr, s2, iters, il, threads=2)
        assert (got == want).mean() >= 0.999, (N, float((got == want).mean()))


@gpu
def test_map_and_turbo_host_pipelines_across_chunks():
    """cpb_map_decode_host / cpb_turbo_decode_host with 5,000 frames of N = 512 run chunks of 2,048 + 2,048 + 904; every
    output equals the device call bit for bit, with and without L_int, and with L_out not requested (MAP)."""
    tr = helpers.rsc_k4()
    rs = np.random.RandomState(63)
    batch, N, s2 = 5000, 512, 0.8
    coded = helpers.encode_batch(rs.randint(0, 2, (batch, N)), tr, "cont")
    ys, yp = (2.0 * coded[:, j::2] - 1 + np.sqrt(s2) * rs.randn(batch, N) for j in (0, 1))
    y2 = rs.choice([-1.0, 1.0], (batch, N)) + np.sqrt(s2) * rs.randn(batch, N)
    ys, yp, y2 = (a.astype(np.float32) for a in (ys, yp, y2))
    La = rs.randn(batch, N).astype(np.float32)
    Lh, bh = _ran(lambda: map_decode_batch_host(ys, yp, tr, s2, La, "decode"), "map_lin2_kernel")
    Ld, bd = map_decode_batch(ys, yp, tr, s2, La, "decode")
    assert np.array_equal(Lh.view(np.int32), Ld.cpu().numpy().view(np.int32))
    assert np.array_equal(bh, bd.cpu().numpy())
    bits = np.empty((batch, N), np.uint8)
    rc = _lib.load().cpb_map_decode_host(_trellis_handle(tr), _lib.ptr(ys), _lib.ptr(yp), _lib.ptr(La), C.c_int64(batch),
                                         C.c_int64(N), C.c_float(s2), 1, C.c_void_p(0), _lib.ptr(bits))
    _lib.check(rc, "map_decode_host")
    assert np.array_equal(bits, bh)
    for b in (0, 2047, 2048, 4095, 4096, 4999):
        Lo, _ = oracle.map_decode(ys[b], yp[b], tr, s2, La[b], "decode")
        assert (np.abs(Lh[b] - Lo) <= MAP_ATOL + MAP_RTOL * np.abs(Lo)).all(), b
    il = RandInterlv(N, 9)
    for L_int in (None, La):
        th = _ran(lambda: turbo_decode_batch_host(ys, yp, y2, tr, s2, 3, il, L_int), "map_lin2_kernel")
        td = turbo_decode_batch(ys, yp, y2, tr, s2, 3, il, L_int).cpu().numpy()
        assert np.array_equal(th, td), L_int is None


# ---------------------------------------------------------------- LDPC
def _params(H):
    H = sp.csr_matrix(H)
    return {"n_vnodes": H.shape[1], "n_cnodes": H.shape[0], "parity_check_matrix": H.tocsc()}


def _wimax_960():
    g = np.load(os.path.join(GOLD, "ldpc.npz"))
    m, n = int(g["l04_meta"][3]), int(g["l04_meta"][4])
    return sp.csr_matrix((np.ones(len(g["l04_indices"]), np.int8), g["l04_indices"], g["l04_indptr"]), shape=(m, n))


def _awgn_llr(rs, batch, n, ebn0_lo, ebn0_hi, rate=0.5):
    """All-zero code word over BPSK-AWGN, one Eb/N0 per frame spread over [lo, hi] dB."""
    eb = np.linspace(ebn0_lo, ebn0_hi, batch)[rs.permutation(batch)]
    sigma = 1.0 / np.sqrt(2 * rate * 10 ** (eb / 10))[:, None]
    return 2.0 * (1.0 + sigma * rs.randn(batch, n)) / sigma ** 2


def _ldpc_oracle(llr, params, iters):
    n = llr.shape[1]
    d, o, it = oracle.ldpc_bp_decode(llr.reshape(-1).copy(), params, "MSA", iters, return_iters=True, threads=8)
    return d.reshape(n, -1).T, o.reshape(n, -1).T, it


def _ldpc(llr, params, iters, precision, no_bulk=False):
    _lib.set_option(_lib.OPT_LDPC_NO_BULK, int(no_bulk))
    try:
        return ldpc_bp_decode_batch(llr.copy(), params, iters, precision, return_iters=True)
    finally:
        _lib.set_option(_lib.OPT_LDPC_NO_BULK, 0)


def _assert_ldpc_exact(got, want):
    dec, out, it = (t.cpu().numpy() for t in got)
    assert np.array_equal(it, want[2])
    assert np.array_equal(dec, want[0])
    assert np.array_equal(out, want[1])


def _assert_bulk_equals_register_staged(llr, params, iters):
    a = _ldpc(llr, params, iters, "fp32")
    b = _ran(lambda: _ldpc(llr, params, iters, "fp32", no_bulk=True), "ldpc::cn_kernel<float,", "cn_bulk_kernel")
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2])
    assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


@gpu
@pytest.mark.parametrize("batch", [64, 128, 256, 384])
def test_ldpc_row_degree_above_8(batch):
    """WiMax 960.720.a (check degrees 14-15).  64 frames: no bulk chunk, cn_kernel<T, 0>.  128 and 384: bulk at 128 frames
    per tile.  256: bulk at 256 in fp32; in fp64 that tile needs more than 200 KB of shared memory and the register-staged
    kernel runs.  fp64 is bit-exact with the oracle on every frame (converged or not); fp32 bulk equals fp32 register-staged."""
    H = _wimax_960()
    params = _params(H)
    rs = np.random.RandomState(64 + batch)
    llr = _awgn_llr(rs, batch, H.shape[1], 2.0, 4.5, rate=0.75)
    iters = 15
    want = _ldpc_oracle(llr, params, iters)
    assert (want[2] < iters).sum() >= batch // 8 and (want[2] == iters).sum() >= 1
    k64 = ["ldpc::cn_kernel<double,0>"] if batch in (64, 256) else ["ldpc::bulk::cn_bulk_kernel<double>"]
    no64 = ["cn_bulk_kernel"] if batch in (64, 256) else ["ldpc::cn_kernel<"]
    _assert_ldpc_exact(_ran(lambda: _ldpc(llr, params, iters, "fp64"), k64, no64), want)
    if batch == 64:
        dec, out, it = (t.cpu().numpy() for t in _ran(lambda: _ldpc(llr, params, iters, "fp32"), "ldpc::cn_kernel<float,0>",
                                                        "cn_bulk_kernel"))
        conv = want[2] < iters
        assert np.array_equal(dec[conv], want[0][conv]) and np.array_equal(it[conv], want[2][conv])
    else:
        _ran(lambda: _ldpc(llr, params, iters, "fp32"), "ldpc::bulk::cn_bulk_kernel<float>")
        _assert_bulk_equals_register_staged(llr, params, iters)


@gpu
def test_ldpc_bulk_degree_edges():
    """Synthetic H with degree-2 rows and mixed degrees up to 16 (fp64 bulk: unrolled and generic row bodies), one with a
    row of degree 32 (bulk::MAXDEG: fp32 bulk; fp64 too large for shared memory) and one with a row of degree 33 (never
    bulk).  fp64 bit-exact with the oracle at a bulk-sized batch; fp32 bulk equals register-staged."""
    base = [2] * 60 + list(range(3, 17)) * 6
    rs = np.random.RandomState(65)
    for top, k64, k32 in ((16, "cn_bulk_kernel<double>", "cn_bulk_kernel<float>"),
                          (32, "ldpc::cn_kernel<double,0>", "cn_bulk_kernel<float>"),
                          (33, "ldpc::cn_kernel<double,0>", "ldpc::cn_kernel<float,0>")):
        H = helpers.mixed_degree_H(base + [top], 480, seed=top)
        assert np.diff(H.indptr).max() == top
        params = _params(H)
        llr = _awgn_llr(rs, 128, 480, 1.0, 4.0)
        want = _ldpc_oracle(llr, params, 12)
        _assert_ldpc_exact(_ran(lambda: _ldpc(llr, params, 12, "fp64"), k64), want)
        _ran(lambda: _ldpc(llr, params, 12, "fp32"), k32)
        if "bulk" in k32:
            _assert_bulk_equals_register_staged(llr, params, 12)


@gpu
def test_ldpc_across_workspace_chunks():
    """C4 surrogate (64800 x 32400) in fp64: a 6 GB workspace holds 2,080 frames, so 2,100 frames run as 2,080 + 20.
    Frames on both sides of the boundary equal the oracle; the second chunk equals those 20 frames decoded alone."""
    H = helpers.dvbs2_like_H()
    params = _params(H)
    n = 64800
    per = (H.nnz + 2.0 * n) * 8 + 12
    chunk = int(6.0e9 / per) // 32 * 32
    assert chunk == 2080
    rng = np.random.default_rng(66)
    sigma = 1.0 / np.sqrt(2 * 0.5 * 10 ** (np.linspace(0.5, 2.5, 2100) / 10))[:, None].astype(np.float32)
    llr = (2.0 * (1.0 + sigma * rng.standard_normal((2100, n), dtype=np.float32)) / sigma ** 2).astype(np.float64)
    x = torch.from_numpy(llr).cuda()
    dec, out, it = _ran(lambda: ldpc_bp_decode_batch(x, params, 5, "fp64", return_iters=True), "ldpc::vn_kernel<double>")
    dec, out, it = dec.cpu().numpy(), out.cpu().numpy(), it.cpu().numpy()
    del x
    idx = [0, chunk - 1, chunk, 2099]
    want = _ldpc_oracle(llr[idx], params, 5)
    assert np.array_equal(dec[idx], want[0]) and np.array_equal(out[idx], want[1]) and np.array_equal(it[idx], want[2])
    d2, o2, i2 = (t.cpu().numpy() for t in ldpc_bp_decode_batch(llr[chunk:].copy(), params, 5, "fp64", return_iters=True))
    assert np.array_equal(dec[chunk:], d2) and np.array_equal(out[chunk:], o2) and np.array_equal(it[chunk:], i2)


@gpu
@pytest.mark.parametrize("precision", ["fp32", "fp64"])
def test_ldpc_host_pipeline_across_chunks(precision):
    """cpb_ldpc_decode_host with 1,000 frames of 960.720.a: chunks of 128 and a ragged 104.  Decisions, out_llrs and
    iterations equal the device call; the caller's array comes back clipped to +-500 in place (ldpc.py:186)."""
    H = _wimax_960()
    params = _params(H)
    rs = np.random.RandomState(67)
    llr = _awgn_llr(rs, 1000, H.shape[1], 2.0, 4.5, rate=0.75)
    llr[::7, ::5] *= 40.0                                       # values beyond the +-500 clip
    dt = np.float64 if precision == "fp64" else np.float32
    x = np.ascontiguousarray(llr, dtype=dt)
    x0 = x.copy()
    dh, oh, ih = _ran(lambda: ldpc_bp_decode_batch_host(x, params, 15, precision, return_iters=True),
                      "ldpc::bulk::cn_bulk_kernel<%s>" % ("double" if precision == "fp64" else "float"))
    assert np.array_equal(x, np.clip(x0, -500, 500)) and np.abs(x0).max() > 500
    dd, od, idd = (t.cpu().numpy() for t in ldpc_bp_decode_batch(x0.copy(), params, 15, precision, return_iters=True))
    assert np.array_equal(dh, dd) and np.array_equal(ih, idd)
    assert np.array_equal(oh.view(np.uint8), od.view(np.uint8))


# ---------------------------------------------------------------- demapper
def _gray_qam_raw(m):
    side = int(np.sqrt(m))
    pam = np.arange(-side + 1, side, 2)
    return np.tile(np.hstack((pam, pam[::-1])), side // 2) * 1j + pam.repeat(side)


DEMAP_CASES = {
    "qam4": (lambda: QAMModem(4), "demod_soft_separable<1>"),
    "qam16": (lambda: QAMModem(16), "demod_soft_separable<2>"),
    "qam64": (lambda: QAMModem(64), "demod_soft_separable<3>"),
    "qam256": (lambda: QAMModem(256), "demod_soft_separable<4>"),
    "qam1024": (lambda: QAMModem(1024), "demod_soft_separable<5>"),
    "qam4096": (lambda: QAMModem(4096), "demod_soft_separable<6>"),
    "psk8": (lambda: PSKModem(8), "demod_soft_general<3>"),
    "psk32": (lambda: PSKModem(32), "demod_soft_general<5>"),
    "psk64": (lambda: PSKModem(64), "demod_soft_general<6>"),
    "psk256": (lambda: PSKModem(256), "demod_soft_general<8>"),
    "custom64": (lambda: Modem(np.random.RandomState(7).randn(64) + 1j * np.random.RandomState(8).randn(64)),
                 "demod_soft_general<6>"),
    "custom256": (lambda: Modem(3 * np.random.RandomState(9).randn(256) + 3j * np.random.RandomState(10).randn(256)),
                  "demod_soft_general<8>"),
    "qam16_no_gray": (lambda: Modem(_gray_qam_raw(16), reorder_as_gray=False), None),
}


def _symbols(cst, nv, rs, n_near=400, n_far=100):
    """Points near the constellation (noise of 0.3 .. 3 standard deviations) and points outside it, placed so that
    the nearest squared distance over nv stays below ~300 (where fp32 distances still carry the LLR to the tolerance)."""
    near = cst[rs.randint(0, len(cst), n_near)] + np.sqrt(nv / 2) * rs.uniform(0.3, 3, n_near) * (
        rs.randn(n_near) + 1j * rs.randn(n_near))
    outer = cst[np.abs(cst) >= 0.8 * np.abs(cst).max()]
    p = outer[rs.randint(0, len(outer), n_far)]
    far = p + p / np.abs(p) * rs.uniform(0, np.sqrt(300 * nv), n_far)       # outward from an outer point
    return np.concatenate([near, far])


def _lse_llr(y, cst, nv):
    """fp64 log-sum-exp LLRs (MSB first, positive favours 1): finite wherever the true LLR is."""
    from scipy.special import logsumexp
    M = len(cst)
    nb = int(np.log2(M))
    out = np.empty((len(y), nb))
    for lo in range(0, len(y), 256):
        e = -np.abs(y[lo:lo + 256, None] - cst[None, :]) ** 2 / nv
        for b in range(nb):
            one = ((np.arange(M) >> (nb - 1 - b)) & 1) == 1
            out[lo:lo + 256, b] = logsumexp(e[:, one], axis=1) - logsumexp(e[:, ~one], axis=1)
    return out.reshape(-1)


@gpu
@pytest.mark.parametrize("case", sorted(DEMAP_CASES))
def test_demod_soft_and_hard_vs_fp64(case):
    """Every LLR within DEMAP_ATOL + DEMAP_RTOL * |LLR| of an fp64 log-sum-exp over the bit-1 / bit-0 subsets, for noise
    variances 1e-3 .. 10 and symbols outside the constellation, including |LLR| of thousands (the kernels' per-group
    re-accumulation).  The reference takes the symbols and points at the fp32 precision the kernels read them in.  Hard
    decisions equal an fp64 first-minimum argmin wherever the two nearest points are not a near tie."""
    make, kern = DEMAP_CASES[case]
    md = make()
    if kern is None:
        sep = _lib.load().cpb_modem_is_separable(md._handle())
        kern = "demod_soft_separable<2>" if sep else "demod_soft_general<4>"
    cst = np.asarray(md.constellation).astype(np.complex64).astype(np.complex128)
    rs = np.random.RandomState(70)
    big = 0.0
    for nv in (1e-3, 0.1, 1.0, 10.0):
        y = _symbols(cst, nv, rs).astype(np.complex64)
        got = _ran(lambda: md.demodulate(y, "soft", nv), "demap::" + kern)
        ref = _lse_llr(y.astype(np.complex128), cst, nv)
        assert np.isfinite(ref).all()
        err = np.abs(got - ref) - DEMAP_RTOL * np.abs(ref)
        assert (err <= DEMAP_ATOL).all(), (case, nv, float(err.max()), float(ref[np.argmax(err)]))
        big = max(big, float(np.abs(ref).max()))
        d = np.abs(y.astype(np.complex128)[:, None] - cst[None, :]) ** 2
        arg = np.argmin(d, axis=1)
        two = np.sort(d, axis=1)[:, :2]
        ok = (two[:, 1] - two[:, 0]) > 1e-5 * np.maximum(two[:, 1], 1e-30)
        nb = md.num_bits_symbol
        want = ((arg[:, None] >> np.arange(nb - 1, -1, -1)) & 1).astype(np.int8)
        hard = _ran(lambda: md.demodulate(y, "hard"), "demap::demod_hard_kernel").reshape(-1, nb)
        assert np.array_equal(hard[ok], want[ok]), (case, nv)
    assert big > 1000.0, big                               # the underflow re-accumulation ran


@gpu
def test_demod_soft_host_pipeline_across_chunks():
    """cpb_demod_soft_host with 3 * 2^20 + 5 symbols runs three 2^20-symbol chunks and a 5-symbol tail; the LLRs equal the
    device call bit for bit."""
    md = QAMModem(64)
    rs = np.random.RandomState(71)
    n = 3 * (1 << 20) + 5
    y = (rs.randn(n) * 5 + 1j * rs.randn(n) * 5).astype(np.complex64)
    host = _ran(lambda: md.demodulate_soft_host(y, 1.3), "demap::demod_soft_separable<3>")
    dev = md.demodulate_batch(torch.from_numpy(y).cuda(), "soft", 1.3).cpu().numpy()
    assert np.array_equal(host.view(np.int32), dev.view(np.int32))

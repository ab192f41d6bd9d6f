"""Turbo-coded links over SISO flat fading: the fading turbo TX kernel (cpb_turbo_link_tx_fading), the coherent BPSK combiner
(cpb_bpsk_combine) and TurboLinkGPU with fading_param, against a float64 model of the random streams, the fp64 oracle's
turbo decoder and the reference (tests/golden/turbo_fading_ber.npz, written by oracle/make_turbo_fading_golden.py)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import helpers
from commpy_b200 import _lib
from commpy_b200.channelcoding import RandInterlv
from commpy_b200.links import TurboLinkGPU, bpsk_combine, turbo_link_tx, turbo_link_tx_fading

gpu = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RAYLEIGH = (0j, 1)
RICIAN = (0.6 + 0j, 0.64)             # passes the reference's exact energy check (0.64 + 0.6^2 == 1 in binary64)
STRONG_RICIAN = (0.95 + 0j, 0.0975)   # Rice factor ~9.3; 0.0975 + 0.95^2 == 1 in binary64 too
UNIT = (1 + 0j, 0)
FP32_EPS = 2.0 ** -23


# ---------------------------------------------------------------- float64 model of the streams
def fading_model(trellis, interleaver, frames, N, seed, first_frame, fading_param):
    """(msg, x, n_re, n_im, h), each stream-major (3, frames, N) but msg, exactly as cpb_turbo_link_tx_fading defines them:
    x = 2 bit - 1 of turbo_encode's streams (helpers.turbo_link_tx_model), n_re its noise (counter word 2 + j), n_im counter
    word 5 + j (values 4q .. 4q+3 = Re, Im of the first Box-Muller, Re, Im of the second), h = mean + sqrt(nlos / 2) g with g
    from counter word 8 + j (one complex gain per Box-Muller: values 2c, 2c+1 from counter c)."""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    msg, *xs = helpers.turbo_link_tx_model(trellis, interleaver, frames, N, seed, first_frame, 0.0)
    _, *ys = helpers.turbo_link_tx_model(trellis, interleaver, frames, N, seed, first_frame, 1.0)
    x = np.stack(xs)
    n_re = np.stack(ys) - x
    mean, nlos = complex(fading_param[0]), float(np.real(fading_param[1]))
    n_im = np.zeros((3, frames, N))
    h = np.zeros((3, frames, N), dtype=np.complex128)
    for fl in range(frames):
        f = first_frame + fl
        for j in range(3):
            z = helpers.philox_normals(f, -(-N // 4), 5 + j, key)
            n_im[j, fl] = np.stack([z.real, z.imag], axis=2).reshape(-1)[:N]
            h[j, fl] = mean + math.sqrt(nlos / 2) * helpers.philox_normals(f, -(-N // 2), 8 + j, key).reshape(-1)[:N]
    return msg, x, n_re, n_im, h


def test_fading_model_at_unit_gain_is_the_awgn_model():
    """No GPU: at (1 + 0j, 0) the model's h is exactly 1, Re of its output is helpers.turbo_link_tx_model's output, and the
    imaginary noise is a standard normal stream distinct from the real one."""
    tr, il = helpers.rsc_k4(), RandInterlv(203, 4)
    seed, first, sigma = 0xabcdef0123, (1 << 32) - 1, 0.7
    msg, x, n_re, n_im, h = fading_model(tr, il, 3, 203, seed, first, UNIT)
    want = helpers.turbo_link_tx_model(tr, il, 3, 203, seed, first, sigma)
    assert np.array_equal(msg, want[0]) and (h == 1).all()
    for j in range(3):
        assert np.allclose(h[j].real * x[j] + sigma * n_re[j], want[1 + j], rtol=0, atol=1e-12)
    assert abs(n_im.mean()) < 0.1 and abs(n_im.std() - 1) < 0.1 and np.abs(n_im - n_re).min() > 0


# ---------------------------------------------------------------- input errors (no GPU)
def test_fading_param_is_validated_like_the_reference():
    tr, il = helpers.rsc_k4(), RandInterlv(64, 1)
    with pytest.raises(ValueError):
        TurboLinkGPU(tr, il, 64, fading_param=(0.5 + 0j, 0.5))          # adds energy: 0.5 + 0.25 != 1
    with pytest.raises(ValueError):
        turbo_link_tx_fading(tr, il, 2, 64, 0, 0, 0.1, (0.5 + 0j, 0.7))
    with pytest.raises(NotImplementedError):
        TurboLinkGPU(tr, il, 64, fading_param=(0.0, 1.0))                # real channel
    for fp in (RAYLEIGH, RICIAN, STRONG_RICIAN, UNIT):
        TurboLinkGPU(tr, il, 64, fading_param=fp)


def test_c_entry_points_reject_bad_arguments_before_any_device_call():
    """Null trellis / pointers and negative lengths are refused with CPB_EINVAL before anything touches the device."""
    lib = _lib.load()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    null = C.c_void_p(0)
    assert lib.cpb_bpsk_combine(null, p, C.c_int64(4), p, null) == _lib.CPB_EINVAL
    assert lib.cpb_bpsk_combine(p, null, C.c_int64(4), p, null) == _lib.CPB_EINVAL
    assert lib.cpb_bpsk_combine(p, p, C.c_int64(4), null, null) == _lib.CPB_EINVAL
    assert lib.cpb_bpsk_combine(p, p, C.c_int64(-1), p, null) == _lib.CPB_EINVAL
    assert lib.cpb_bpsk_combine(null, null, C.c_int64(0), null, null) == _lib.CPB_OK          # nothing to do
    assert lib.cpb_turbo_link_tx_fading(null, p, C.c_int64(2), C.c_int64(64), C.c_uint64(1), C.c_int64(0), C.c_float(0.5),
                                        C.c_float(0.0), C.c_float(0.0), C.c_float(1.0), p, p, p, null) == _lib.CPB_EINVAL


# ---------------------------------------------------------------- TX kernel
@gpu
@pytest.mark.parametrize("N", [256, 1000, 6144])
def test_unit_gain_equals_awgn_link_bit_for_bit(N):
    """fading_param = (1 + 0j, 0): msg and Re(y) equal turbo_link_tx bit for bit for all three streams, h == 1 + 0j exactly,
    bpsk_combine(y, h) == Re(y) exactly, and TurboLinkGPU gives the AWGN link's counters and BERs."""
    import torch
    tr, il = helpers.rsc_k4(), RandInterlv(N, 3)
    seed, first, sigma = 0x5eed0123456789, (1 << 32) - 3, 0.8
    msg_a, *awgn = turbo_link_tx(tr, il, 7, N, seed, first, sigma)
    msg, y, h = turbo_link_tx_fading(tr, il, 7, N, seed, first, sigma, UNIT)
    assert y.shape == (3, 7, N) and h.shape == (3, 7, N)
    assert torch.equal(msg, msg_a)
    for j in range(3):
        assert torch.equal(y[j].real, awgn[j]), j
    assert (h == 1).all() and torch.equal(h.real, torch.ones_like(h.real)) and torch.equal(h.imag, torch.zeros_like(h.imag))
    assert torch.equal(bpsk_combine(y, h), y.real.contiguous())

    links = {fp: TurboLinkGPU(tr, il, N, frames_per_batch=48, iterations=6, seed=11, fading_param=fp) for fp in (None, UNIT)}
    counters = {}
    for fp, link in links.items():
        c = torch.zeros(3, dtype=torch.int64, device="cuda")
        for b in range(2):
            batch = link.make_batch(0.5, b)
            link.decode_count(*batch, c, torch)
        counters[fp] = c.cpu().numpy()
    assert counters[None][0] > 0 and np.array_equal(counters[None], counters[UNIT]), counters
    bers = {fp: link.link_performance([0.0, 1.0], send_max=3 * 48 * N, err_min=10 ** 9) for fp, link in links.items()}
    assert np.array_equal(bers[None], bers[UNIT]), bers


@gpu
@pytest.mark.parametrize("N", [1000, 203])
def test_fading_tx_matches_numpy_model(N):
    """Rayleigh and Rician, frames across first_frame = 2^32, N a multiple of 4 or not: the message is exact, h is within 2e-3
    of the float64 model, y - h x matches sigma (n_re + j n_im) within 2e-3 on both components, and two calls covering a
    batch give what one call gives."""
    import torch
    tr, il = helpers.rsc_k4(), RandInterlv(N, 2)
    frames, seed, first, sigma = 5, 0x1234567890abcdef, (1 << 32) - 2, 0.75
    for fp in (RAYLEIGH, RICIAN):
        want_msg, x, n_re, n_im, want_h = fading_model(tr, il, frames, N, seed, first, fp)
        msg, y, h = turbo_link_tx_fading(tr, il, frames, N, seed, first, sigma, fp)
        assert np.array_equal(msg.cpu().numpy(), want_msg)
        hn = h.cpu().numpy().astype(np.complex128)
        assert np.abs(hn - want_h).max() < 2e-3, fp
        noise = y.cpu().numpy().astype(np.complex128) - hn * x
        assert np.abs(noise.real - sigma * n_re).max() < 2e-3, fp
        assert np.abs(noise.imag - sigma * n_im).max() < 2e-3, fp
        msg2, y2, h2 = turbo_link_tx_fading(tr, il, 2, N, seed, first, sigma, fp)
        msg3, y3, h3 = turbo_link_tx_fading(tr, il, 3, N, seed, first + 2, sigma, fp)
        assert torch.equal(torch.cat([msg2, msg3]), msg)
        assert helpers.same(torch.cat([y2, y3], dim=1), y) and helpers.same(torch.cat([h2, h3], dim=1), h)


@gpu
def test_fading_gain_statistics():
    """>= 1e6 gains: Rayleigh (0j, 1) and Rician (0.6 + 0j, 0.64) have the right mean and mean power (5 sigma) and |h|^2 follows
    Exp(1), resp. (nlos/2) * ncx2(2, |m|^2 / (nlos/2)) (Kolmogorov-Smirnov, p > 1e-3)."""
    from scipy import stats
    tr, il = helpers.rsc_k4(), RandInterlv(6144, 1)
    for fp in (RAYLEIGH, RICIAN):
        _, _, h = turbo_link_tx_fading(tr, il, 64, 6144, 2024, 0, 0.5, fp)
        h = h.cpu().numpy().reshape(-1).astype(np.complex128)
        n = h.size
        assert n >= 1_000_000
        m, nlos = complex(fp[0]), float(fp[1])
        assert abs(h.real.mean() - m.real) < 5 * math.sqrt(nlos / 2 / n)
        assert abs(h.imag.mean() - m.imag) < 5 * math.sqrt(nlos / 2 / n)
        p = np.abs(h) ** 2
        assert abs(p.mean() - 1.0) < 5 * p.std() / math.sqrt(n), (fp, p.mean())
        dist = stats.expon() if m == 0 else stats.ncx2(2, abs(m) ** 2 / (nlos / 2), scale=nlos / 2)
        pv = stats.kstest(p, dist.cdf).pvalue
        assert pv > 1e-3, (fp, pv)


# ---------------------------------------------------------------- combiner
def _ran(fn, want):
    """fn() under the profiler; asserts that a kernel whose normalised name contains `want` ran (a profiling session that
    recorded no kernel activity is repeated, at most four times)"""
    for _ in range(5):
        box = []
        names = helpers.launched_kernels(lambda: box.append(fn()))
        if any(want in n for n in names):
            break
    assert any(want in n for n in names), (want, sorted(names))
    return box[0]


def _check_combined(s, y, h):
    """s (float32) within 2 ulp(1) * (|h_re y_re| + |h_im y_im|) of Re(conj(h) y) in float64; exactly 0 where h = 0 and exactly
    Re(y) where h = 1"""
    s = np.asarray(s, dtype=np.float64)
    y64, h64 = y.astype(np.complex128), h.astype(np.complex128)
    want = (np.conj(h64) * y64).real
    bound = 2 * FP32_EPS * (np.abs(h64.real * y64.real) + np.abs(h64.imag * y64.imag))
    assert (np.abs(s - want) <= bound).all(), float(np.max(np.abs(s - want) - bound))
    assert (s[h64 == 0] == 0).all()
    assert np.array_equal(s[h64 == 1], y64.real[h64 == 1])


@gpu
def test_combiner_vs_fp64():
    """bpsk_combine against float64 for |h| from 1e-6 to 10 with random phases, h = 0 and h = 1; lengths 1, 3, 4, 5 and a large
    odd length; 16-byte aligned tensors (vector path and scalar tail) and views 8 bytes off (scalar path); the combiner kernel
    is the one that ran."""
    import torch
    rs = np.random.RandomState(8)
    n = 1_000_003
    mags = np.concatenate([10.0 ** rs.uniform(-6, 1, n - 3000), np.full(1000, 1e-6), np.full(1000, 10.0), np.zeros(1000)])
    rs.shuffle(mags)
    h = (mags * np.exp(2j * np.pi * rs.rand(n))).astype(np.complex64)
    h[rs.randint(0, n, 500)] = 1
    y = ((rs.randn(n) + 1j * rs.randn(n)) * 10.0 ** rs.uniform(-3, 1, n)).astype(np.complex64)
    yt, ht = torch.from_numpy(y).cuda(), torch.from_numpy(h).cuda()
    s = _ran(lambda: bpsk_combine(yt, ht), "turbolink::bpsk_combine_kernel")
    _check_combined(s.cpu().numpy(), y, h)
    for off in (0, 1):
        for L in (1, 3, 4, 5, 1000, n - off):
            ys, hs = yt[off:off + L], ht[off:off + L]
            assert (ys.data_ptr() % 16 == 0) == (off == 0)
            _check_combined(bpsk_combine(ys, hs).cpu().numpy(), y[off:off + L], h[off:off + L])
    # shapes are kept; y and h at different alignments take the scalar path
    s = bpsk_combine(yt[:600].reshape(3, 200), ht[1:601].reshape(3, 200))
    assert s.shape == (3, 200) and s.dtype == torch.float32
    _check_combined(s.cpu().numpy().reshape(-1), y[:600], h[1:601])


@gpu
def test_combiner_input_errors():
    import torch
    y = torch.zeros((3, 4, 10), dtype=torch.complex64, device="cuda")
    with pytest.raises(ValueError):
        bpsk_combine(y, torch.zeros((3, 4, 9), dtype=torch.complex64, device="cuda"))
    with pytest.raises(ValueError):
        bpsk_combine(y, torch.zeros((4, 10), dtype=torch.complex64, device="cuda"))
    with pytest.raises(ValueError):
        bpsk_combine(y, torch.zeros((3, 4, 10), dtype=torch.complex128, device="cuda"))
    with pytest.raises(ValueError):
        bpsk_combine(y.cpu(), y.cpu())
    assert bpsk_combine(y[:, :0], y[:, :0]).shape == (3, 0, 10)


@gpu
def test_c_entry_points_reject_bad_fading_arguments():
    """CPB_EINVAL for null pointers, nlos < 0 and non-finite parameters; CPB_EUNSUPPORTED for a non-systematic trellis."""
    import torch
    from commpy_b200.channelcoding.convcode import _trellis_handle
    lib = _lib.load()
    N = 64
    perm = torch.arange(N, dtype=torch.int32, device="cuda")
    msg = torch.empty((2, N), dtype=torch.uint8, device="cuda")
    y, h = (torch.empty((3, 2, N), dtype=torch.complex64, device="cuda") for _ in range(2))
    st = _lib.stream_ptr(torch)

    def call(tr, nlos=1.0, mean=(0.0, 0.0), sigma=0.5, yp=None, hp=None, pp=None):
        return lib.cpb_turbo_link_tx_fading(_trellis_handle(tr), _lib.ptr(perm) if pp is None else pp, C.c_int64(2),
                                            C.c_int64(N), C.c_uint64(5), C.c_int64(0), C.c_float(sigma), C.c_float(mean[0]),
                                            C.c_float(mean[1]), C.c_float(nlos), _lib.ptr(msg),
                                            _lib.ptr(y) if yp is None else yp, _lib.ptr(h) if hp is None else hp, st)
    rsc = helpers.rsc_k4()
    assert call(rsc) == _lib.CPB_OK
    assert call(rsc, yp=C.c_void_p(0)) == _lib.CPB_EINVAL
    assert call(rsc, hp=C.c_void_p(0)) == _lib.CPB_EINVAL
    assert call(rsc, pp=C.c_void_p(0)) == _lib.CPB_EINVAL
    assert call(rsc, nlos=-0.25) == _lib.CPB_EINVAL
    assert call(rsc, nlos=math.inf) == _lib.CPB_EINVAL
    assert call(rsc, mean=(math.nan, 0.0)) == _lib.CPB_EINVAL
    assert call(rsc, sigma=math.nan) == _lib.CPB_EINVAL
    assert call(helpers.k7()) == _lib.CPB_EUNSUPPORTED                     # feed-forward: not systematic
    torch.cuda.synchronize()


# ---------------------------------------------------------------- decoding
def _oracle_point(link, ebn0):
    """Batch 0 of `link` decoded on the GPU (TurboLinkGPU.decode_count) and by the fp64 oracle from the same channel output,
    combined in float64: (gpu bits, oracle bits, msg, s as combined in float64, sigma^2).  The GPU side must have run the
    combiner kernel."""
    import torch
    from oracle import oracle
    batch = link.make_batch(ebn0, 0)
    msg, y, h, s2 = batch
    cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
    dec = _ran(lambda: link.decode_count(*batch, cnt, torch), "turbolink::bpsk_combine_kernel").cpu().numpy()
    yn, hn = y.cpu().numpy().astype(np.complex128), h.cpu().numpy().astype(np.complex128)
    s = (np.conj(hn) * yn).real
    want = oracle.turbo_decode_batch(s[0], s[1], s[2], link.trellis, s2, link.iterations, link.interleaver, threads=8)
    msg = msg.cpu().numpy()
    return dec, want, msg, s, s2


@gpu
def test_turbo_fading_link_decodes_like_the_fp64_oracle():
    """TurboLinkGPU over Rayleigh (1,024 frames of N = 1,024, 6 iterations) at two Eb/N0 points in the waterfall, and over a
    strongly Rician channel at high Eb/N0 (channel LLRs 2 s / sigma^2 beyond 25; over Rayleigh |s| passes 10): the oracle
    decodes y, h combined in float64 at the same sigma^2.  At least 99.9 % of the bits agree, and the GPU BER equals the
    oracle's within 3 standard errors of the oracle's per-frame error counts."""
    N = 1024
    il = RandInterlv(N, 7)
    smax = 0.0
    for fp, ebn0 in ((RAYLEIGH, 1.5), (RAYLEIGH, 2.0), (STRONG_RICIAN, 8.0)):
        link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=1024, iterations=6, seed=31, fading_param=fp)
        dec, want, msg, s, s2 = _oracle_point(link, ebn0)
        agree = float((dec == want).mean())
        e_gpu, e_or = (dec != msg).sum(axis=1), (want != msg).sum(axis=1)
        se = max(float(np.std(e_or, ddof=1)), 1.0) / math.sqrt(len(e_or)) / N
        ber_gpu, ber_or = e_gpu.sum() / msg.size, e_or.sum() / msg.size
        llr = 2 * float(np.abs(s).max()) / s2
        smax = max(smax, float(np.abs(s).max()))
        print("%s %.1f dB: GPU BER %.4e, oracle %.4e (se %.1e), agreement %.6f, max |s| %.1f, max |LLR| %.1f"
              % (fp, ebn0, ber_gpu, ber_or, se, agree, np.abs(s).max(), llr))
        assert agree >= 0.999, (fp, ebn0, agree)
        assert abs(ber_gpu - ber_or) <= 3 * se, (fp, ebn0, ber_gpu, ber_or, se)
        if fp == RAYLEIGH:
            assert 1e-4 < ber_or < 0.2, (ebn0, ber_or)          # inside the waterfall
        else:
            assert llr > 25, llr
    assert smax >= 10.0, smax


@gpu
def test_turbo_fading_link_matches_reference_golden():
    """TurboLinkGPU over Rayleigh and Rician fading against the unmodified reference (turbo_encode, SISOFlatChannel, the
    coherent combiner and turbo_decode per frame, oracle/make_turbo_fading_golden.py): the GPU BER over 8,192 frames is within
    4 SE + 15 % + 1e-3 (absolute floor) of the reference's BER at every golden point, SE from the reference's per-frame
    error counts."""
    g = np.load(os.path.join(GOLD, "turbo_fading_ber.npz"))
    N, iters = int(g["N"]), int(g["iterations"])
    il = RandInterlv(N, int(g["interleaver_seed"]))
    for name in ("rayleigh", "rician"):
        m, nlos = g[name + "_fading_param"]
        fp = (complex(m), float(nlos.real))
        fe = g[name + "_frame_errors"].astype(np.float64)
        ref = fe.sum(axis=1) / (N * fe.shape[1])
        se = fe.std(axis=1, ddof=1) / N / np.sqrt(fe.shape[1])
        link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=2048, iterations=iters, seed=5, fading_param=fp)
        got = link.link_performance([float(e) for e in g[name + "_ebn0"]], send_max=4 * 2048 * N, err_min=10 ** 9)
        print("%s: reference %s (se %s), GPU %s" % (name, list(ref), list(se), list(got)))
        for b_ref, s_ref, b_gpu in zip(ref, se, got):
            assert abs(b_gpu - b_ref) <= 4 * s_ref + 0.15 * b_ref + 1e-3, (name, list(ref), list(se), list(got))
        assert min(ref) > 1e-3 and max(ref) < 0.2


@gpu
def test_turbo_fading_counters_identical_for_1_2_4_8_ranks(monkeypatch):
    """Same seed => same error counters over fading, whatever the number of (emulated) ranks."""
    import torch
    N = 1024
    il = RandInterlv(N, 1)
    totals = {}
    for world in (1, 2, 4, 8):
        link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=256 // world, iterations=6, seed=77,
                            fading_param=RAYLEIGH)
        tot = torch.zeros(3, dtype=torch.int64, device="cuda")
        for rank in range(world):
            monkeypatch.setenv("RANK", str(rank))
            monkeypatch.setenv("WORLD_SIZE", str(world))
            for b in range(3):
                link.decode_count(*link.make_batch(1.5, b), tot, torch)
        totals[world] = tot.cpu().numpy().copy()
    monkeypatch.delenv("RANK")
    monkeypatch.delenv("WORLD_SIZE")
    assert totals[1][0] > 0, "the test point must have bit errors to compare"
    for world in (2, 4, 8):
        assert np.array_equal(totals[world], totals[1]), (world, totals)


@gpu
def test_fading_tx_kernel_is_the_one_that_ran():
    """turbo_link_tx_fading launches the FADING instance of the encode kernel; turbo_link_tx the AWGN one."""
    tr, il = helpers.rsc_k4(), RandInterlv(256, 1)
    _ran(lambda: turbo_link_tx_fading(tr, il, 8, 256, 1, 0, 0.5, RAYLEIGH), "turbolink::encode_kernel<true>")
    _ran(lambda: turbo_link_tx(tr, il, 8, 256, 1, 0, 0.5), "turbolink::encode_kernel<false>")

"""Turbo-coded links over PSK/QAM modems: the parity kernel and the shared code-word modulator behind
cpb_turbo_link_tx_modem[_fading], and TurboLinkGPU with modem=, against a float64 model of the TX streams, the BPSK link,
the fp64 oracle's turbo decoder and the unmodified reference (tests/golden/turbo_modem_ber.npz, written by
oracle/make_turbo_modem_golden.py)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import helpers
from commpy_b200 import _lib
from commpy_b200.channelcoding import RandInterlv
from commpy_b200.links import TurboLinkGPU, turbo_link_tx, turbo_link_tx_modem, turbo_link_tx_modem_fading
from commpy_b200.modulation import PSKModem, QAMModem

gpu = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RAYLEIGH = (0j, 1)
RICIAN = (0.6 + 0j, 0.64)
UNIT = (1 + 0j, 0)
LLR_MAX = 600.0


def modems():
    """(name, modem, N): every modem with a frame length whose 3N code bits fill whole symbols"""
    return [("qpsk", QAMModem(4), 256), ("qam16", QAMModem(16), 1024), ("qam64", QAMModem(64), 1000),
            ("qam256", QAMModem(256), 512), ("psk8", PSKModem(8), 203)]


# ---------------------------------------------------------------- float64 model of the TX
def code_words(trellis, interleaver, msg):
    """[sys | par1 | par2] per row of msg: np.concatenate of turbo_encode's three streams, each cut to N"""
    from commpy_b200.channelcoding import turbo_encode
    N = msg.shape[1]
    return np.stack([np.concatenate([np.asarray(s[:N]) for s in turbo_encode(m.astype(int), trellis, trellis, interleaver)])
                     for m in msg]).astype(np.uint8)


def tx_model(trellis, interleaver, modem, frames, N, seed, first_frame, fading_param=None):
    """(msg, c, points, z, h) as cpb_turbo_link_tx_modem[_fading] define them: Philox message bits (word 0), the host
    turbo_encode mirror's code word, Modem.modulate's points (MSB first), float64 Box-Muller noise of word 1 and gains of
    word 5 (one per symbol, symbols 2q and 2q+1 from counter q).  y = h * points + noise_sigma * z."""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    nb = int(modem.num_bits_symbol)
    nsym = 3 * N // nb
    msg = np.stack([helpers.philox_bits(first_frame + f, N, key) for f in range(frames)]).astype(np.uint8)
    c = code_words(trellis, interleaver, msg)
    idx = c.reshape(frames, nsym, nb).astype(np.int64) @ (1 << np.arange(nb - 1, -1, -1))
    points = np.asarray(modem.constellation)[idx]
    z = np.stack([helpers.philox_normals(first_frame + f, -(-nsym // 2), 1, key).reshape(-1)[:nsym] for f in range(frames)])
    h = np.ones((frames, nsym), dtype=np.complex128)
    if fading_param is not None:
        mean, nlos = complex(fading_param[0]), float(np.real(fading_param[1]))
        g = np.stack([helpers.philox_normals(first_frame + f, -(-nsym // 2), 5, key).reshape(-1)[:nsym] for f in range(frames)])
        h = mean + math.sqrt(nlos / 2) * g
    return msg, c, points, z, h


def test_model_code_word_is_the_reference_layout():
    """No GPU: the model's code word is [msg | par1 | par2] with the message bits of the BPSK link's model, and its points
    are Modem.modulate of the code word."""
    tr = helpers.rsc_k4()
    seed, first = 0xabcdef0123, (1 << 32) - 1
    for _, modem, N in modems():
        il = RandInterlv(N, 4)
        msg, c, points, z, h = tx_model(tr, il, modem, 2, N, seed, first)
        want = helpers.turbo_link_tx_model(tr, il, 2, N, seed, first, 0.0)
        assert np.array_equal(msg, want[0])
        for j in range(3):
            assert np.array_equal(2.0 * c[:, j * N:(j + 1) * N] - 1.0, want[1 + j])
        assert np.array_equal(points[0], modem.modulate(c[0]))
        assert (h == 1).all() and abs(z.real.std() - 1) < 0.2


# ---------------------------------------------------------------- input errors (no GPU)
def test_python_layer_rejects_ragged_code_words_and_bad_fading():
    tr = helpers.rsc_k4()
    il = RandInterlv(203, 1)
    with pytest.raises(ValueError):
        TurboLinkGPU(tr, il, 203, modem=QAMModem(16))                   # 609 bits are not whole 16-QAM symbols
    with pytest.raises(ValueError):
        turbo_link_tx_modem(tr, il, QAMModem(4), 2, 203, 0, 0, 0.1)
    with pytest.raises(ValueError):
        turbo_link_tx_modem_fading(tr, il, QAMModem(4), 2, 203, 0, 0, 0.1, RAYLEIGH)
    with pytest.raises(ValueError):
        TurboLinkGPU(tr, il, 203, modem=PSKModem(8), fading_param=(0.5 + 0j, 0.5))
    with pytest.raises(NotImplementedError):
        TurboLinkGPU(tr, il, 203, modem=PSKModem(8), fading_param=(0.0, 1.0))
    link = TurboLinkGPU(tr, il, 203, modem=PSKModem(8), fading_param=RAYLEIGH)
    nb, Es = 3, PSKModem(8).Es
    assert math.isclose(link.noise_variance(4.0), Es / (2 * nb / 3 * 10 ** 0.4), rel_tol=1e-15)
    qpsk, bpsk = TurboLinkGPU(tr, RandInterlv(256, 1), 256, modem=QAMModem(4)), TurboLinkGPU(tr, RandInterlv(256, 1), 256)
    assert math.isclose(qpsk.noise_variance(1.5), bpsk.noise_variance(1.5), rel_tol=1e-15)      # QPSK: Es = 2, nb = 2


def test_c_entry_points_reject_null_handles_before_any_device_call():
    lib = _lib.load()
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)
    null = C.c_void_p(0)
    args = (C.c_int64(2), C.c_int64(64), C.c_uint64(1), C.c_int64(0), C.c_float(0.5))
    assert lib.cpb_turbo_link_tx_modem(null, p, p, *args, p, p, null) == _lib.CPB_EINVAL
    assert lib.cpb_turbo_link_tx_modem(p, null, p, *args, p, p, null) == _lib.CPB_EINVAL
    assert lib.cpb_turbo_link_tx_modem_fading(null, p, p, *args, C.c_float(0.0), C.c_float(0.0), C.c_float(1.0), p, p, p,
                                              null) == _lib.CPB_EINVAL


# ---------------------------------------------------------------- TX
@gpu
@pytest.mark.parametrize("name", [m[0] for m in modems()])
def test_tx_matches_float64_model(name):
    """Frames across first_frame = 2^32: the message equals the model and turbo_link_tx's message; at noise_sigma = 0, y is
    exactly Modem.modulate of the code word (this pins the parity kernel bit for bit, N % 16 == 0 on its 16-byte path and
    otherwise on its byte path); y - c is within 2e-3 of the model's noise, and over Rayleigh fading y - h c and h are too.
    At (1 + 0j, 0) the fading TX equals the AWGN TX bit for bit.  Two calls covering a batch give what one call gives."""
    import torch
    _, modem, N = next(m for m in modems() if m[0] == name)
    tr, il = helpers.rsc_k4(), RandInterlv(N, 2)
    frames, seed, first, sigma = 5, 0x1234567890abcdef, (1 << 32) - 3, 0.6
    msg_m, c, points, z, _ = tx_model(tr, il, modem, frames, N, seed, first)
    msg0, y0 = turbo_link_tx_modem(tr, il, modem, frames, N, seed, first, 0.0)
    assert np.array_equal(msg0.cpu().numpy(), msg_m)
    assert torch.equal(msg0, turbo_link_tx(tr, il, frames, N, seed, first, 0.5)[0])
    assert y0.shape == (frames, 3 * N // modem.num_bits_symbol) and y0.dtype == torch.complex64
    assert np.array_equal(y0.cpu().numpy(), points.astype(np.complex64))
    msg, y = turbo_link_tx_modem(tr, il, modem, frames, N, seed, first, sigma)
    assert torch.equal(msg, msg0)
    noise = y.cpu().numpy().astype(np.complex128) - points
    assert np.abs(noise - sigma * z).max() < 2e-3
    msg_u, y_u, h_u = turbo_link_tx_modem_fading(tr, il, modem, frames, N, seed, first, sigma, UNIT)
    assert torch.equal(msg_u, msg) and helpers.same(y_u, y) and (h_u == 1).all()
    for fp in (RAYLEIGH, RICIAN):
        _, _, _, _, want_h = tx_model(tr, il, modem, frames, N, seed, first, fp)
        msg_f, y_f, h_f = turbo_link_tx_modem_fading(tr, il, modem, frames, N, seed, first, sigma, fp)
        assert torch.equal(msg_f, msg) and h_f.shape == y_f.shape == y.shape
        hn = h_f.cpu().numpy().astype(np.complex128)
        assert np.abs(hn - want_h).max() < 2e-3, fp
        assert np.abs(y_f.cpu().numpy() - hn * points - sigma * z).max() < 2e-3, fp
        m2, y2, h2 = turbo_link_tx_modem_fading(tr, il, modem, 2, N, seed, first, sigma, fp)
        m3, y3, h3 = turbo_link_tx_modem_fading(tr, il, modem, 3, N, seed, first + 2, sigma, fp)
        assert torch.equal(torch.cat([m2, m3]), msg_f)
        assert helpers.same(torch.cat([y2, y3]), y_f) and helpers.same(torch.cat([h2, h3]), h_f)
    m2, y2 = turbo_link_tx_modem(tr, il, modem, 2, N, seed, first, sigma)
    m3, y3 = turbo_link_tx_modem(tr, il, modem, 3, N, seed, first + 2, sigma)
    assert torch.equal(torch.cat([m2, m3]), msg) and helpers.same(torch.cat([y2, y3]), y)


@gpu
def test_tx_unaligned_and_chunked_shapes():
    """A batch of more frames than one pass of the parity scratch (N = 6144: 8,192 frames per pass) and an N whose rows are
    not 16-byte aligned give the model's code words at noise_sigma = 0 (checked on a sample of frames)."""
    tr = helpers.rsc_k4()
    modem = QAMModem(16)
    for N, frames in ((6144, 8200), (1000, 33)):
        il = RandInterlv(N, 5)
        msg, y = turbo_link_tx_modem(tr, il, modem, frames, N, 99, 7, 0.0)
        rows = np.unique(np.array([0, 1, frames // 2, frames - 9, frames - 1]))
        msg_n, y_n = msg.cpu().numpy()[rows], y.cpu().numpy()[rows]
        c = code_words(tr, il, msg_n)
        nb = modem.num_bits_symbol
        idx = c.reshape(len(rows), -1, nb).astype(np.int64) @ (1 << np.arange(nb - 1, -1, -1))
        assert np.array_equal(y_n, np.asarray(modem.constellation)[idx].astype(np.complex64)), N
        key = (99, 0)
        for r, m in zip(rows, msg_n):
            assert np.array_equal(m, helpers.philox_bits(7 + int(r), N, key))


@gpu
def test_c_entry_points_reject_bad_arguments():
    """CPB_EINVAL for null pointers, 3N % bits_per_symbol, N < 1, first_frame < 0, nlos < 0 and non-finite fading parameters;
    CPB_EUNSUPPORTED for a trellis the turbo TX refuses; frames = 0 is a no-op."""
    import torch
    from commpy_b200.channelcoding.convcode import _trellis_handle
    lib = _lib.load()
    N = 64
    modem = QAMModem(16)
    perm = torch.arange(N, dtype=torch.int32, device="cuda")
    msg = torch.empty((2, N), dtype=torch.uint8, device="cuda")
    y, h = (torch.empty((2, 3 * N // 4), dtype=torch.complex64, device="cuda") for _ in range(2))
    st = _lib.stream_ptr(torch)
    null = C.c_void_p(0)
    rsc, k7 = helpers.rsc_k4(), helpers.k7()          # the handles live as long as their trellis objects

    def awgn(tr=rsc, frames=2, n=N, first=0, mp=None, yp=None, pp=None):
        return lib.cpb_turbo_link_tx_modem(_trellis_handle(tr), modem._handle(),
                                           _lib.ptr(perm) if pp is None else pp, C.c_int64(frames), C.c_int64(n), C.c_uint64(5),
                                           C.c_int64(first), C.c_float(0.5), _lib.ptr(msg) if mp is None else mp,
                                           _lib.ptr(y) if yp is None else yp, st)

    def fading(nlos=1.0, mean=(0.0, 0.0), sigma=0.5, hp=None, yp=None):
        return lib.cpb_turbo_link_tx_modem_fading(_trellis_handle(rsc), modem._handle(), _lib.ptr(perm),
                                                  C.c_int64(2), C.c_int64(N), C.c_uint64(5), C.c_int64(0), C.c_float(sigma),
                                                  C.c_float(mean[0]), C.c_float(mean[1]), C.c_float(nlos), _lib.ptr(msg),
                                                  _lib.ptr(y) if yp is None else yp, _lib.ptr(h) if hp is None else hp, st)
    assert awgn() == _lib.CPB_OK and fading() == _lib.CPB_OK
    assert awgn(mp=null) == _lib.CPB_EINVAL
    assert awgn(yp=null) == _lib.CPB_EINVAL
    assert awgn(pp=null) == _lib.CPB_EINVAL
    assert awgn(n=62) == _lib.CPB_EINVAL                                    # 186 bits are not whole 16-QAM symbols
    assert awgn(n=0) == _lib.CPB_EINVAL
    assert awgn(first=-1) == _lib.CPB_EINVAL
    assert awgn(frames=-1) == _lib.CPB_EINVAL
    assert awgn(frames=0, mp=null, yp=null, pp=null) == _lib.CPB_OK
    assert awgn(tr=k7) == _lib.CPB_EUNSUPPORTED                   # feed-forward: not systematic
    assert fading(hp=null) == _lib.CPB_EINVAL
    assert fading(yp=null) == _lib.CPB_EINVAL
    assert fading(nlos=-0.25) == _lib.CPB_EINVAL
    assert fading(nlos=math.inf) == _lib.CPB_EINVAL
    assert fading(mean=(math.nan, 0.0)) == _lib.CPB_EINVAL
    assert fading(mean=(0.0, math.inf)) == _lib.CPB_EINVAL
    assert fading(sigma=math.nan) == _lib.CPB_EINVAL
    torch.cuda.synchronize()


def _ran(fn, want):
    """fn() under the profiler; asserts that kernels whose normalised names contain each string of `want` ran"""
    for _ in range(5):
        box = []
        names = helpers.launched_kernels(lambda: box.append(fn()))
        if all(any(w in n for n in names) for w in want):
            break
    for w in want:
        assert any(w in n for n in names), (w, sorted(names))
    return box[0]


@gpu
def test_kernels_that_ran():
    """The modem TX launches the message, parity and shared modulate kernels (the fading instance over fading); the receiver
    the demapper and the turbo decoder; the LDPC TX still launches the shared modulator."""
    import torch
    tr, il = helpers.rsc_k4(), RandInterlv(256, 1)
    _ran(lambda: turbo_link_tx_modem(tr, il, QAMModem(16), 8, 256, 1, 0, 0.5),
         ["turbolink::msg_kernel", "turbolink::parity_kernel", "cwtx::modulate_kernel<false>"])
    _ran(lambda: turbo_link_tx_modem_fading(tr, il, QAMModem(16), 8, 256, 1, 0, 0.5, RAYLEIGH),
         ["turbolink::parity_kernel", "cwtx::modulate_kernel<true>"])
    link = TurboLinkGPU(tr, il, 256, frames_per_batch=8, modem=QAMModem(16), fading_param=RAYLEIGH)
    batch = link.make_batch(3.0, 0)
    cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
    _ran(lambda: link.decode_count(*batch, cnt, torch), ["demod_soft", "map_"])
    from commpy_b200.links import ldpc_link_tx
    from test_ldpc_encode_model import small_staircase
    import scipy.sparse as sp
    H = small_staircase(720, 360, 5)
    params = {"parity_check_matrix": sp.csc_matrix(H), "n_vnodes": 720, "n_cnodes": 360}
    _ran(lambda: ldpc_link_tx(params, QAMModem(16), 8, 1, 0, 0.5), ["cwtx::modulate_kernel<false>"])


# ---------------------------------------------------------------- link
def _frame_errors(link, ebn0, batches=1):
    """per-frame bit errors of `batches` batches of `link`, from its own decode_count"""
    import torch
    errs = []
    for b in range(batches):
        batch = link.make_batch(ebn0, b)
        cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
        dec = link.decode_count(*batch, cnt, torch)
        e = (dec != batch[0]).sum(dim=1).cpu().numpy()
        assert int(cnt[0]) == int(e.sum())
        errs.append(e)
    return np.concatenate(errs)


@gpu
def test_qpsk_link_equals_bpsk_link_statistically():
    """Gray QPSK with exact LLRs is two BPSK channels at the same Eb/N0: TurboLinkGPU(modem=QAMModem(4)) and the BPSK link
    (modem=None), 4,096 frames of N = 1,024 each at two waterfall points, have BERs within 4 standard errors of the
    difference of their per-frame error counts.  This pins the noise formula and the LLR scale."""
    N = 1024
    il = RandInterlv(N, 3)
    for ebn0 in (0.75, 1.0):
        e = {}
        for name, md in (("qpsk", QAMModem(4)), ("bpsk", None)):
            link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=2048, iterations=6, seed=17, modem=md)
            e[name] = _frame_errors(link, ebn0, batches=2).astype(np.float64)
        b = {k: v.sum() / (v.size * N) for k, v in e.items()}
        se = math.sqrt(sum(v.var(ddof=1) / v.size for v in e.values())) / N
        print("Eb/N0 %.2f dB: QPSK BER %.4e, BPSK %.4e, se %.1e" % (ebn0, b["qpsk"], b["bpsk"], se))
        assert 1e-4 < b["bpsk"] < 0.2, b
        assert abs(b["qpsk"] - b["bpsk"]) <= 4 * se, (ebn0, b, se)


@gpu
def test_high_snr_links_decode_without_errors():
    """16-, 64- and 256-QAM and 8-PSK over AWGN and Rayleigh far above the waterfall: zero bit errors, finite LLRs and 0/1
    decisions (this pins the LLR sign).  One point (16-QAM, AWGN, 30 dB) has channel LLRs beyond 1e3, which the turbo
    decoder takes unclamped."""
    import torch
    N = 1024
    il = RandInterlv(N, 9)
    cases = [(QAMModem(16), None, 8.0), (QAMModem(64), None, 12.0), (QAMModem(256), None, 16.0), (PSKModem(8), None, 10.0),
             (QAMModem(16), RAYLEIGH, 14.0), (QAMModem(64), RAYLEIGH, 18.0), (QAMModem(256), RAYLEIGH, 22.0),
             (PSKModem(8), RAYLEIGH, 16.0), (QAMModem(16), None, 30.0)]
    big = 0.0
    for modem, fp, ebn0 in cases:
        link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=256, iterations=6, seed=23, modem=modem, fading_param=fp)
        batch = link.make_batch(ebn0, 0)
        llr = torch.cat(link.llr_streams(*batch[1:]), dim=1)
        assert bool(torch.isfinite(llr).all())
        amax = float(llr.abs().max())
        cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
        dec = link.decode_count(*batch, cnt, torch)
        print("%d-point %s %.1f dB: errors %d, max |LLR| %.1f" % (len(modem.constellation), fp, ebn0, int(cnt[0]), amax))
        assert bool(((dec == 0) | (dec == 1)).all())
        assert int(cnt[0]) == 0 and int(cnt[1]) == 0, (len(modem.constellation), fp, ebn0, cnt.tolist())
        if ebn0 == 30.0:
            big = amax
    assert big > 1e3, big


def oracle_inputs(L):
    """(r, nv) with 2 r / nv == L and |r| <= 1: the fp64 oracle's probability-domain BCJR takes exact LLRs this way without
    its branch probabilities underflowing"""
    L = np.asarray(L, dtype=np.float64)
    amax = float(np.abs(L).max())
    assert np.isfinite(L).all() and amax <= LLR_MAX, amax
    nv = 2.0 / max(1.0, amax)
    return L * (nv / 2.0), nv


@gpu
def test_link_decodes_like_the_fp64_oracle():
    """1,024 frames of N = 1,024 in the waterfall, 16-QAM over AWGN and 64-QAM over Rayleigh: the fp64 oracle decodes the
    link's own float32 LLRs.  At least 99.9 % of the bits agree, and the BERs are equal within 3 standard errors of the
    oracle's per-frame error counts."""
    import torch
    from oracle import oracle
    N = 1024
    il = RandInterlv(N, 7)
    for modem, fp, ebn0 in ((QAMModem(16), None, 2.75), (QAMModem(64), RAYLEIGH, 6.5)):
        link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=1024, iterations=6, seed=31, modem=modem, fading_param=fp)
        batch = link.make_batch(ebn0, 0)
        cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
        dec = _ran(lambda: link.decode_count(*batch, cnt, torch), ["demod_soft"]).cpu().numpy()
        L = [s.cpu().numpy() for s in link.llr_streams(*batch[1:])]
        r, nv = oracle_inputs(np.stack(L))
        want = oracle.turbo_decode_batch(r[0], r[1], r[2], link.trellis, nv, link.iterations, il, threads=8)
        msg = batch[0].cpu().numpy()
        agree = float((dec == want).mean())
        e_gpu, e_or = (dec != msg).sum(axis=1), (want != msg).sum(axis=1)
        se = max(float(np.std(e_or, ddof=1)), 1.0) / math.sqrt(len(e_or)) / N
        ber_gpu, ber_or = e_gpu.sum() / msg.size, e_or.sum() / msg.size
        print("%d-QAM %s %.2f dB: GPU BER %.4e, oracle %.4e (se %.1e), agreement %.6f, max |LLR| %.1f"
              % (len(modem.constellation), fp, ebn0, ber_gpu, ber_or, se, agree, 2 / nv))
        assert 1e-4 < ber_or < 0.2, ber_or
        assert agree >= 0.999, agree
        assert abs(ber_gpu - ber_or) <= 3 * se, (ber_gpu, ber_or, se)


@gpu
def test_link_matches_reference_golden():
    """TurboLinkGPU(modem=QAMModem(M)) over AWGN and Rayleigh against the unmodified reference (turbo_encode, Modem.modulate,
    SISOFlatChannel, the exact demapper and turbo_decode per frame): the GPU BER over 8,192 frames is within 4 SE + 15 % +
    1e-3 of the reference's BER at every golden point, SE from the reference's per-frame error counts."""
    g = np.load(os.path.join(GOLD, "turbo_modem_ber.npz"))
    N, iters = int(g["N"]), int(g["iterations"])
    il = RandInterlv(N, int(g["interleaver_seed"]))
    for name in ("qam4_awgn", "qam16_awgn", "qam16_rayleigh", "qam64_rayleigh"):
        m, nlos = g[name + "_fading_param"]
        fp = None if nlos == 0 else (complex(m), float(nlos.real))
        fe = g[name + "_frame_errors"].astype(np.float64)
        ref = fe.sum(axis=1) / (N * fe.shape[1])
        se = fe.std(axis=1, ddof=1) / N / np.sqrt(fe.shape[1])
        link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=2048, iterations=iters, seed=5,
                            modem=QAMModem(int(g[name + "_M"])), fading_param=fp)
        got = link.link_performance([float(e) for e in g[name + "_ebn0"]], send_max=4 * 2048 * N, err_min=10 ** 9)
        print("%s: reference %s (se %s), GPU %s" % (name, list(ref), list(se), list(got)))
        for b_ref, s_ref, b_gpu in zip(ref, se, got):
            assert abs(b_gpu - b_ref) <= 4 * s_ref + 0.15 * b_ref + 1e-3, (name, list(ref), list(se), list(got))
        assert min(ref) > 1e-3 and max(ref) < 0.2


@gpu
@pytest.mark.parametrize("fp", [None, RAYLEIGH])
def test_counters_identical_for_1_2_4_8_ranks(monkeypatch, fp):
    """Same seed => same error counters over a modem, whatever the number of (emulated) ranks."""
    import torch
    N = 1024
    il = RandInterlv(N, 1)
    totals = {}
    for world in (1, 2, 4, 8):
        link = TurboLinkGPU(helpers.rsc_k4(), il, N, frames_per_batch=256 // world, iterations=6, seed=77, modem=QAMModem(16),
                            fading_param=fp)
        tot = torch.zeros(3, dtype=torch.int64, device="cuda")
        for rank in range(world):
            monkeypatch.setenv("RANK", str(rank))
            monkeypatch.setenv("WORLD_SIZE", str(world))
            for b in range(3):
                link.decode_count(*link.make_batch(2.75 if fp is None else 4.0, b), tot, torch)
        totals[world] = tot.cpu().numpy().copy()
    monkeypatch.delenv("RANK")
    monkeypatch.delenv("WORLD_SIZE")
    assert totals[1][0] > 0, "the test point must have bit errors to compare"
    for world in (2, 4, 8):
        assert np.array_equal(totals[world], totals[1]), (world, totals)

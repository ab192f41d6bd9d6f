"""LDPC-coded links on the GPU: the systematic encoder planned from H (cpb_ldpc_encode), the LDPC TX chain over AWGN and flat
fading (cpb_ldpc_link_tx[_fading]) and LdpcLinkGPU, against the NumPy GF(2) model (tests/model_ldpc_encode.py), the
float64 Philox model of the TX streams, the fp64 C oracle and the unmodified reference (tests/golden/ldpc_link_ber.npz,
written by oracle/make_ldpc_link_golden.py)."""
import math
import os

import numpy as np
import pytest
import scipy.sparse as sp

import helpers
import model_ldpc_encode as mle
from test_ldpc_encode_model import design_H, small_staircase

gpu = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RAYLEIGH = (0j, 1)


def params_of(H):
    """a code dict given only as a parity-check matrix (no generator is ever computed for it by the GPU paths)"""
    return {"parity_check_matrix": sp.csc_matrix(H), "n_vnodes": H.shape[1], "n_cnodes": H.shape[0]}


def wimax(name):
    return params_of(design_H(name))


def syndrome_zero(H, cw):
    return not ((sp.csr_matrix(H) @ np.asarray(cw, dtype=np.int64).T) % 2).any()


def _ran(fn, want):
    """fn() under the profiler; asserts that a kernel whose name contains `want` ran and `want` is not a kernel of the
    other encoder form"""
    for _ in range(5):
        box = []
        names = helpers.launched_kernels(lambda: box.append(fn()))
        if any(want in n for n in names):
            break
    assert any(want in n for n in names), (want, sorted(names))
    return box[0], names


# ---------------------------------------------------------------- encoder
@gpu
@pytest.mark.parametrize("name", ["1440_720", "960_720_a"])
def test_encoder_equals_reference_encodings(name):
    """Batches of 1, 3, 33 and 4,097: equal to the stored reference encodings and to the host triang_ldpc_systematic_encode,
    bit for bit."""
    import torch
    from commpy_b200.channelcoding import ldpc_encode_batch, triang_ldpc_systematic_encode
    g = np.load(os.path.join(GOLD, "ldpc_link_ber.npz"))
    msg0, cw0 = g["wimax_%s_msg" % name], g["wimax_%s_cw" % name]
    params = wimax(name)
    k = msg0.shape[1]
    rs = np.random.RandomState(7)
    host = dict(params)
    for batch in (1, 3, 33, 4097):
        msg = np.concatenate([msg0, rs.randint(0, 2, (max(batch - len(msg0), 0), k)).astype(np.uint8)])[:batch]
        got = ldpc_encode_batch(torch.from_numpy(msg).cuda(), params).cpu().numpy()
        m0 = min(batch, len(msg0))
        assert np.array_equal(got[:m0], cw0[:m0]), (name, batch)
        want = np.asarray(triang_ldpc_systematic_encode(msg.reshape(-1), host, False)).reshape(-1, batch).T
        assert np.array_equal(got, want.astype(np.uint8)), (name, batch)


@gpu
def test_encoder_code_words():
    """H c = 0 on every frame: Gallager 96.33.964 (where the reference's encoding is not a code word, DESIGN.md section 7),
    both WiMax codes, the full DVB-S2-shaped code and a small one; each equals the GF(2) model.  Gallager 96.3.963 (singular
    H_p) raises ValueError, a code that neither peels nor fits the dense bound raises NotImplementedError."""
    from commpy_b200.channelcoding import ldpc_encode_batch
    rs = np.random.RandomState(3)
    for H, batch in ((design_H("96_33_964"), 65), (design_H("1440_720"), 70), (design_H("960_720_a"), 31),
                     (helpers.dvbs2_like_H(), 40), (small_staircase(), 100)):
        m, n = H.shape
        msg = rs.randint(0, 2, (batch, n - m)).astype(np.uint8)
        cw = ldpc_encode_batch(msg, params_of(H)).cpu().numpy()
        assert np.array_equal(cw[:, :n - m], msg)
        assert syndrome_zero(H, cw), H.shape
        if n < 10000:
            assert np.array_equal(cw, mle.encode(H, msg)), H.shape
    with pytest.raises(ValueError):
        ldpc_encode_batch(np.zeros((2, 48), np.uint8), params_of(design_H("96_3_963")))
    big = helpers.mixed_degree_H([6] * 9000, 18000, seed=4)
    with pytest.raises(NotImplementedError):
        ldpc_encode_batch(np.zeros((2, 9000), np.uint8), params_of(big))


@gpu
def test_peeled_and_dense_forms_agree():
    """On a small staircase code the peeled and the forced-dense forms give identical code words; the profiler shows the
    peeled solve kernel, resp. the dense parity kernel, ran."""
    from commpy_b200 import _lib
    from commpy_b200.channelcoding import ldpc_encode_batch
    H = small_staircase(720, 360, 5)
    params = params_of(H)
    msg = np.random.RandomState(9).randint(0, 2, (300, 360)).astype(np.uint8)
    peeled, names = _ran(lambda: ldpc_encode_batch(msg, params), "ldpclink::peel_solve_kernel")
    assert not any("dense_parity_kernel" in s for s in names)
    _lib.set_option(_lib.OPT_LDPC_ENC_FORCE_DENSE, 1)
    try:
        dense, names = _ran(lambda: ldpc_encode_batch(msg, params), "ldpclink::dense_parity_kernel")
    finally:
        _lib.set_option(_lib.OPT_LDPC_ENC_FORCE_DENSE, 0)
    assert not any("peel_solve_kernel" in s for s in names)
    assert np.array_equal(peeled.cpu().numpy(), dense.cpu().numpy())
    assert syndrome_zero(H, peeled.cpu().numpy())


# ---------------------------------------------------------------- TX chain
def tx_model(H, modem, frames, seed, first, sigma):
    """(msg, code words, points, noise) as cpb_ldpc_link_tx defines them: Philox message bits (word 0), the GF(2) model's
    code word, Modem.modulate's points (MSB first), float64 Box-Muller noise of word 1"""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    m, n = H.shape
    nb = modem.num_bits_symbol
    msg = np.stack([helpers.philox_bits(first + f, n - m, key) for f in range(frames)]).astype(np.uint8)
    cw = mle.encode(H, msg)
    cst = np.asarray(modem.constellation)
    idx = cw.reshape(frames, -1, nb).astype(np.int64) @ (1 << np.arange(nb - 1, -1, -1))
    nsym = n // nb
    z = np.stack([helpers.philox_normals(first + f, -(-nsym // 2), 1, key).reshape(-1)[:nsym] for f in range(frames)])
    return msg, cw, cst[idx], sigma * z


@gpu
@pytest.mark.parametrize("code,M", [("1440_720", 16), ("960_720_a", 4), ("staircase", 256), ("96_33_964", 64)])
def test_tx_matches_model(code, M):
    """Messages equal the Philox model exactly; noiseless symbols equal Modem.modulate(code word); y - c matches the model
    noise within 2e-3; frames do not depend on the split across first_frame = 2^32; the fading TX at (1 + 0j, 0) equals the
    AWGN TX bit for bit, and its gains and noise match the model."""
    import torch
    from commpy_b200.links import ldpc_link_tx, ldpc_link_tx_fading
    from commpy_b200.modulation import QAMModem
    H = small_staircase(800, 400, 2) if code == "staircase" else design_H(code)
    params, modem = params_of(H), QAMModem(M)
    frames, seed, first, sigma = 6, 0x1234567890abcdef, (1 << 32) - 3, 0.7
    msg_m, cw_m, pts, noise = tx_model(H, modem, frames, seed, first, sigma)
    msg, y0 = ldpc_link_tx(params, modem, frames, seed, first, 0.0)
    assert np.array_equal(msg.cpu().numpy(), msg_m)
    assert np.array_equal(y0.cpu().numpy(), pts.astype(np.complex64))
    assert np.array_equal(modem.modulate(cw_m.reshape(-1)).astype(np.complex64).reshape(frames, -1), y0.cpu().numpy())
    msg, y = ldpc_link_tx(params, modem, frames, seed, first, sigma)
    assert np.abs(y.cpu().numpy() - pts - noise).max() < 2e-3
    msg3, y3 = ldpc_link_tx(params, modem, 3, seed, first + 3, sigma)
    assert torch.equal(msg3, msg[3:]) and helpers.same(y3, y[3:])
    fm, fy, fh = ldpc_link_tx_fading(params, modem, frames, seed, first, sigma, (1 + 0j, 0))
    assert torch.equal(fm, msg) and helpers.same(fy, y) and bool((fh == 1).all())
    fm, fy, fh = ldpc_link_tx_fading(params, modem, frames, seed, first, sigma, RAYLEIGH)
    key = (seed & 0xFFFFFFFF, seed >> 32)
    nsym = pts.shape[1]
    hm = np.stack([helpers.philox_normals(first + f, -(-nsym // 2), 5, key).reshape(-1)[:nsym] for f in range(frames)])
    hn = fh.cpu().numpy()
    assert torch.equal(fm, msg) and np.abs(hn - hm / math.sqrt(2)).max() < 2e-3
    assert np.abs(fy.cpu().numpy() - hn * pts - noise).max() < 2e-3


@gpu
def test_tx_gain_statistics():
    """> 1e6 Rayleigh gains: mean 0 and mean power 1 (5 sigma), |h|^2 ~ Exp(1) (Kolmogorov-Smirnov, p > 1e-3)."""
    from scipy import stats
    from commpy_b200.links import ldpc_link_tx_fading
    from commpy_b200.modulation import QAMModem
    _, _, h = ldpc_link_tx_fading(wimax("1440_720"), QAMModem(4), 1500, 11, 0, 0.5, RAYLEIGH)
    h = h.cpu().numpy().reshape(-1).astype(np.complex128)
    n = h.size
    assert n >= 1_000_000
    assert abs(h.real.mean()) < 5 * math.sqrt(0.5 / n) and abs(h.imag.mean()) < 5 * math.sqrt(0.5 / n)
    p = np.abs(h) ** 2
    assert abs(p.mean() - 1.0) < 5 * p.std() / math.sqrt(n)
    assert stats.kstest(p, stats.expon().cdf).pvalue > 1e-3


# ---------------------------------------------------------------- link
@gpu
def test_link_high_snr_has_no_errors():
    """At a high SNR every frame decodes: the decoder gets the demapper's LLRs negated (with the demapper's own sign every
    frame would fail)."""
    from commpy_b200.links import LdpcLinkGPU
    from commpy_b200.modulation import QAMModem
    for fp in (None, RAYLEIGH):
        link = LdpcLinkGPU(wimax("1440_720"), QAMModem(16), 512, seed=5, fading_param=fp)
        ber, cnt = link.link_performance([25.0], send_max=5e5, err_min=10 ** 9, return_counters=True, stop_early=False)
        assert ber[0] == 0 and int(cnt[2]) >= 5e5, (fp, ber, cnt)


@gpu
@pytest.mark.parametrize("fp", [None, RAYLEIGH])
def test_link_fp64_decisions_equal_oracle(fp):
    """1,024 frames at fp64: the link's decisions equal the fp64 oracle's ldpc_bp_decode on the link's own LLRs, exactly, and
    the counters count the message bits of those decisions."""
    import torch
    from oracle import oracle
    from commpy_b200.links import LdpcLinkGPU
    from commpy_b200.modulation import QAMModem
    params = wimax("1440_720")
    link = LdpcLinkGPU(params, QAMModem(16), 1024, precision="fp64", seed=21, fading_param=fp)
    snr = 10.0 if fp is None else 12.0
    msg, y, nv, *h = link.make_batch(snr, 0)
    llr = link.llrs(y, nv, *h).cpu().numpy()
    cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
    dec = link.receive_decode_count(msg, y, nv, cnt, torch, *h).cpu().numpy()
    want, _ = oracle.ldpc_bp_decode(llr.reshape(-1).copy(), params, "MSA", 15, threads=8)
    want = want.T.astype(np.uint8)
    assert np.array_equal(dec, want)
    err = want[:, :720] != msg.cpu().numpy()
    assert int(cnt[0]) == err.sum() > 0 and int(cnt[1]) == err.any(axis=1).sum()


@gpu
@pytest.mark.parametrize("case", ["qam4_awgn", "qam16_awgn", "qam4_rayleigh", "qam16_rayleigh"])
def test_link_ber_matches_reference(case):
    """LdpcLinkGPU's BER within 4 SE + 15 % of the reference LinkModel's (WiMax 1440.720, MSA 15 iterations) at every point."""
    from commpy_b200.links import LdpcLinkGPU
    from commpy_b200.modulation import QAMModem
    g = np.load(os.path.join(GOLD, "ldpc_link_ber.npz"))
    snrs, fe = g[case + "_snr"], g[case + "_block_errors"].astype(np.float64)
    K = int(g["k"])
    ref = fe.mean(axis=1) / K
    se = fe.std(axis=1, ddof=1) / K / np.sqrt(fe.shape[1])
    M = int(case.split("_")[0][3:])
    link = LdpcLinkGPU(wimax("1440_720"), QAMModem(M), 2048, seed=8, fading_param=RAYLEIGH if "rayleigh" in case else None)
    got = link.link_performance([float(s) for s in snrs], send_max=8192 * K, err_min=10 ** 9, stop_early=False)
    print("%s: reference %s (se %s), GPU %s" % (case, list(ref), list(se), list(got)))
    for b_ref, s_ref, b_gpu in zip(ref, se, got):
        assert abs(b_gpu - b_ref) <= 4 * s_ref + 0.15 * b_ref, (case, list(snrs), list(ref), list(se), list(got))


@gpu
def test_link_counters_identical_for_1_2_4_8_ranks(monkeypatch):
    import torch
    from commpy_b200.links import LdpcLinkGPU
    from commpy_b200.modulation import QAMModem
    totals = {}
    for world in (1, 2, 4, 8):
        link = LdpcLinkGPU(wimax("1440_720"), QAMModem(16), 1024 // world, seed=77, fading_param=RAYLEIGH)
        tot = torch.zeros(3, dtype=torch.int64, device="cuda")
        for rank in range(world):
            monkeypatch.setenv("RANK", str(rank))
            monkeypatch.setenv("WORLD_SIZE", str(world))
            for b in range(3):
                msg, y, nv, h = link.make_batch(12.0, b)
                link.receive_decode_count(msg, y, nv, tot, torch, h)
        totals[world] = tot.cpu().numpy().copy()
    monkeypatch.delenv("RANK")
    monkeypatch.delenv("WORLD_SIZE")
    assert totals[1][0] > 0
    for world in (2, 4, 8):
        assert np.array_equal(totals[world], totals[1]), (world, totals)


@gpu
def test_input_errors():
    """Wrong shapes and non-0/1 messages (ValueError), invalid fading_param (ValueError / NotImplementedError), code words
    that do not fill whole symbols (ValueError in Python, CPB_EINVAL from the C ABI), bad decoder settings."""
    import ctypes as C
    import torch
    from commpy_b200 import _lib
    from commpy_b200.channelcoding import ldpc_encode_batch
    from commpy_b200.channelcoding.ldpc import _ldpc_handle
    from commpy_b200.links import LdpcLinkGPU, ldpc_link_tx, ldpc_link_tx_fading
    from commpy_b200.modulation import QAMModem
    params = wimax("1440_720")
    for bad in (np.zeros((3, 721), np.uint8), np.zeros(720, np.uint8), np.zeros((2, 3, 720), np.uint8)):
        with pytest.raises(ValueError):
            ldpc_encode_batch(bad, params)
    two = np.zeros((2, 720), np.uint8)
    two[1, 5] = 2
    with pytest.raises(ValueError):
        ldpc_encode_batch(two, params)
    with pytest.raises(ValueError):
        ldpc_encode_batch(-torch.ones((1, 720), dtype=torch.int32), params)
    with pytest.raises(ValueError):
        LdpcLinkGPU(params, QAMModem(4), 64, fading_param=(0.5 + 0j, 0.5))
    with pytest.raises(NotImplementedError):
        LdpcLinkGPU(params, QAMModem(4), 64, fading_param=(0.0, 1.0))
    with pytest.raises(ValueError):
        ldpc_link_tx_fading(params, QAMModem(4), 2, 0, 0, 0.1, (0.5 + 0j, 0.7))
    with pytest.raises(ValueError):
        LdpcLinkGPU(params, QAMModem(4), 64, decoder_algorithm="BP")
    with pytest.raises(ValueError):
        LdpcLinkGPU(params, QAMModem(4), 64, precision="fp16")
    odd = params_of(small_staircase(200, 100, 2))
    with pytest.raises(ValueError):
        LdpcLinkGPU(odd, QAMModem(64), 64)
    with pytest.raises(ValueError):
        ldpc_link_tx(odd, QAMModem(64), 4, 0, 0, 0.1)
    handle, _ = _ldpc_handle(odd)
    msg = torch.empty((4, 100), dtype=torch.uint8, device="cuda")
    y = torch.empty((4, 40), dtype=torch.complex64, device="cuda")
    lib = _lib.load()
    head = (handle, QAMModem(64)._handle(), C.c_int64(4), C.c_uint64(0), C.c_int64(0), C.c_float(0.1))
    assert lib.cpb_ldpc_link_tx(*head, _lib.ptr(msg), _lib.ptr(y), _lib.stream_ptr(torch)) == _lib.CPB_EINVAL
    assert lib.cpb_ldpc_link_tx_fading(*head, C.c_float(0), C.c_float(0), C.c_float(1), _lib.ptr(msg), _lib.ptr(y), _lib.ptr(y),
                                       _lib.stream_ptr(torch)) == _lib.CPB_EINVAL
    head = (handle, QAMModem(4)._handle(), C.c_int64(4), C.c_uint64(0), C.c_int64(0), C.c_float(0.1))
    assert lib.cpb_ldpc_link_tx_fading(*head, C.c_float(0), C.c_float(0), C.c_float(-1), _lib.ptr(msg), _lib.ptr(y), _lib.ptr(y),
                                       _lib.stream_ptr(torch)) == _lib.CPB_EINVAL
    assert lib.cpb_ldpc_encode(handle, _lib.ptr(msg), C.c_int64(-1), _lib.ptr(msg), _lib.stream_ptr(torch)) == _lib.CPB_EINVAL

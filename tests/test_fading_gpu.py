"""Flat-fading SISO links: the fading TX kernels (cpb_conv_link_tx_fading), the channel-aware demapper (cpb_demod_soft_csi /
cpb_demod_hard_csi) and ConvLinkGPU / Wifi80211.link_performance_gpu with fading_param, against NumPy models, theory and the
reference (tests/golden/fading_ber.npz, written by oracle/make_fading_golden.py)."""
import math
import os

import numpy as np
import pytest

import helpers
from commpy_b200.links import ConvLinkGPU, conv_link_tx_fading

gpu = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ATOL, RTOL = 5e-4, 5e-4
RAYLEIGH = (0j, 1)
RICIAN = (0.6 + 0j, 0.64)            # passes the reference's exact energy check (0.64 + 0.6^2 == 1 in binary64)
WIFI_34 = [1, 1, 1, 0, 0, 1]


# ---------------------------------------------------------------- fp64 models
def csi_llr(y, h, cst, nv):
    """fp64 log-sum-exp LLRs of y = h c + noise (MSB first, positive favours 1): log sum_{bit=1} exp(-|y-hc|^2/nv) - log
    sum_{bit=0} ..., the reference's demodulate(y/h, 'soft', nv/|h|^2) per symbol, and 0 where h = 0."""
    from scipy.special import logsumexp
    M = len(cst)
    nb = int(np.log2(M))
    out = np.empty((len(y), nb))
    for lo in range(0, len(y), 256):
        e = -np.abs(y[lo:lo + 256, None] - h[lo:lo + 256, None] * cst[None, :]) ** 2 / nv
        for b in range(nb):
            one = ((np.arange(M) >> (nb - 1 - b)) & 1) == 1
            out[lo:lo + 256, b] = logsumexp(e[:, one], axis=1) - logsumexp(e[:, ~one], axis=1)
    return out.reshape(-1)


def gains_model(frames, nsym, seed, first_frame, fading_param):
    """h exactly as cpb_conv_link_tx_fading defines it: Philox counter word 5, float64 Box-Muller."""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    mean, nlos = complex(fading_param[0]), float(np.real(fading_param[1]))
    h = np.zeros((frames, nsym), dtype=np.complex128)
    for fl in range(frames):
        g = helpers.philox_normals(first_frame + fl, -(-nsym // 2), 5, key)
        h[fl] = mean + math.sqrt(nlos / 2) * g.reshape(-1)[:nsym]
    return h


class _ScaledModem:
    """duck-typed modem whose constellation is h * c: what oracle.demodulate sees for one symbol of gain h"""

    def __init__(self, cst, h):
        self.constellation = np.asarray(cst) * h


def test_csi_llr_model_matches_oracle_on_scaled_constellations():
    """The fp64 CSI restatement the GPU tests compare with equals the C oracle's demapper run on the constellation h * c,
    symbol by symbol (Rayleigh gains, QAM16 and PSK8)."""
    from oracle import oracle
    from commpy_b200.modulation import PSKModem, QAMModem
    rs = np.random.RandomState(5)
    for md, nv in ((QAMModem(16), 2.0), (PSKModem(8), 0.3)):
        cst = np.asarray(md.constellation, dtype=np.complex128)
        n = 150
        h = (rs.randn(n) + 1j * rs.randn(n)) / math.sqrt(2)
        y = h * cst[rs.randint(0, len(cst), n)] + math.sqrt(nv / 2) * (rs.randn(n) + 1j * rs.randn(n))
        want = np.concatenate([oracle.demodulate(_ScaledModem(cst, h[i]), y[i:i + 1], "soft", nv) for i in range(n)])
        got = csi_llr(y, h, cst, nv)
        assert np.allclose(got, want, rtol=1e-9, atol=1e-9), np.abs(got - want).max()


def test_fading_param_is_validated_like_the_reference():
    from commpy_b200.modulation import QAMModem
    with pytest.raises(ValueError):
        ConvLinkGPU(helpers.k7(), QAMModem(4), fading_param=(0.5 + 0j, 0.5))          # adds energy: 0.5 + 0.25 != 1
    with pytest.raises(ValueError):
        conv_link_tx_fading(helpers.k7(), QAMModem(4), 2, 128, 0, 0, 0.1, (0.5 + 0j, 0.7))
    with pytest.raises(NotImplementedError):
        ConvLinkGPU(helpers.k7(), QAMModem(4), fading_param=(0.0, 1.0))                # real channel
    ConvLinkGPU(helpers.k7(), QAMModem(4), fading_param=RICIAN)


# ---------------------------------------------------------------- TX kernels
def _tx_both(fn):
    """fn() with the word-parallel TX kernel allowed and with the bit-serial one forced"""
    from commpy_b200 import _lib
    out = {}
    for force in (1, 0):
        _lib.set_option(_lib.OPT_TX_FORCE_GENERIC, force)
        try:
            out[force] = fn()
        finally:
            _lib.set_option(_lib.OPT_TX_FORCE_GENERIC, 0)
    return out


@gpu
def test_unit_gain_equals_awgn_link_bit_for_bit():
    """fading_param = (1 + 0j, 0): msg and y equal cpb_conv_link_tx[_punctured] bit for bit and h == 1, for the word-parallel
    kernel, the bit-serial kernel and a punctured 802.11 pattern."""
    from commpy_b200.links import conv_link_tx
    from commpy_b200.modulation import QAMModem
    seed, first = 0x5eed0123456789, (1 << 32) - 3
    for tr, modem, fb, punct in ((helpers.k7(), QAMModem(16), 1024, None), (helpers.k7(), QAMModem(256), 4096, None),
                                 (helpers.k7_wifi_quirk(), QAMModem(16), 1536, WIFI_34)):
        awgn = _tx_both(lambda: conv_link_tx(tr, modem, 9, fb, seed, first, 0.6, punct))
        fad = _tx_both(lambda: conv_link_tx_fading(tr, modem, 9, fb, seed, first, 0.6, (1 + 0j, 0), punct))
        for force in (0, 1):
            assert helpers.same(fad[force][0], awgn[force][0]), (fb, punct, force)
            assert helpers.same(fad[force][1], awgn[force][1]), (fb, punct, force)
            h = fad[force][2].cpu().numpy()
            assert h.shape == awgn[force][1].shape and (h == 1).all()


@gpu
@pytest.mark.parametrize("modem_m", [4, 16, 256])
def test_fading_word_parallel_kernel_equals_bit_serial(modem_m):
    """With Rayleigh fading the word-parallel and the bit-serial TX kernels give the same msg, y and h bit for bit (the cases of
    test_conv_link_tx_word_parallel_kernel_equals_bit_serial)."""
    from commpy_b200.channelcoding import Trellis
    from commpy_b200.modulation import QAMModem
    modem = QAMModem(modem_m)
    k3 = Trellis(np.array([2]), np.array([[5, 7]]))
    for tr, frame_bits in ((helpers.k7(), 1024), (helpers.k7_wifi_quirk(), 128), (helpers.k7(), 4096), (k3, 256)):
        out = _tx_both(lambda: conv_link_tx_fading(tr, modem, 37, frame_bits, 0xfeedbeef12345, (1 << 32) - 5, 0.6, RAYLEIGH))
        for a, b in zip(out[0], out[1]):
            assert helpers.same(a, b), (modem_m, frame_bits)


@gpu
@pytest.mark.parametrize("modem_m,frame_bits,punct", [(4, 200, None), (16, 1024, None), (256, 4096, None), (64, 1536, [1, 1, 1, 0]),
                                                     (16, 1536, WIFI_34)])
def test_fading_tx_matches_numpy_model(modem_m, frame_bits, punct):
    """h equals the float64 model (Philox counter word 5), y - h c equals the AWGN link's noise, and the frames do not depend on
    how they are split over calls, beyond first_frame = 2^32."""
    import torch
    from commpy_b200.modulation import QAMModem
    tr = helpers.k7() if punct is None else helpers.k7_wifi_quirk()
    modem = QAMModem(modem_m)
    frames, seed, first, sigma = 5, 0x1234567890abcdef, (1 << 32) - 2, 0.75
    want_msg, points = helpers.conv_link_tx_model(tr, modem, frames, frame_bits, seed, first, 0.0, punct)
    _, y_awgn = helpers.conv_link_tx_model(tr, modem, frames, frame_bits, seed, first, sigma, punct)
    for fp in (RAYLEIGH, RICIAN):
        msg, y, h = conv_link_tx_fading(tr, modem, frames, frame_bits, seed, first, sigma, fp, punct)
        assert np.array_equal(msg.cpu().numpy(), want_msg)
        hn = h.cpu().numpy()
        assert np.abs(hn - gains_model(frames, points.shape[1], seed, first, fp)).max() < 2e-3
        noise = y.cpu().numpy() - hn.astype(np.complex128) * points
        assert np.abs(noise - (y_awgn - points)).max() < 2e-3
        msg3, y3, h3 = conv_link_tx_fading(tr, modem, 3, frame_bits, seed, first + 2, sigma, fp, punct)
        assert torch.equal(msg3, msg[2:]) and helpers.same(y3, y[2:]) and helpers.same(h3, h[2:])


@gpu
def test_fading_gain_statistics():
    """>= 1e6 gains: Rayleigh (0j, 1) and Rician (0.6 + 0j, 0.64) have the right mean and mean power (5 sigma) and |h|^2 follows
    Exp(1), resp. (nlos/2) * ncx2(2, |m|^2 / (nlos/2)) (Kolmogorov-Smirnov, p > 1e-3)."""
    from scipy import stats
    from commpy_b200.modulation import QAMModem
    for fp in (RAYLEIGH, RICIAN):
        _, _, h = conv_link_tx_fading(helpers.k7(), QAMModem(4), 260, 4096, 2024, 0, 0.5, fp)
        h = h.cpu().numpy().reshape(-1).astype(np.complex128)
        n = h.size
        assert n >= 1_000_000
        m, nlos = complex(fp[0]), float(fp[1])
        assert abs(h.real.mean() - m.real) < 5 * math.sqrt(nlos / 2 / n)
        assert abs(h.imag.mean() - m.imag) < 5 * math.sqrt(nlos / 2 / n)
        p = np.abs(h) ** 2
        assert abs(p.mean() - 1.0) < 5 * p.std() / math.sqrt(n), (fp, p.mean())
        if m == 0:
            dist = stats.expon()
        else:
            dist = stats.ncx2(2, abs(m) ** 2 / (nlos / 2), scale=nlos / 2)
        pv = stats.kstest(p, dist.cdf).pvalue
        assert pv > 1e-3, (fp, pv)


# ---------------------------------------------------------------- CSI demapper
def _custom16():
    from commpy_b200.modulation import Modem
    ring = np.concatenate([np.exp(2j * np.pi * (np.arange(4) + 0.5) / 4), 2.5 * np.exp(2j * np.pi * np.arange(12) / 12)])
    return Modem(ring)


def _cases():
    from commpy_b200.modulation import PSKModem, QAMModem
    c = {"qam%d" % m: (lambda m=m: QAMModem(m), "demod_soft_separable_csi<%d>" % (int(np.log2(m)) // 2))
         for m in (4, 16, 64, 256, 1024, 4096)}
    c["psk8"] = (lambda: PSKModem(8), "demod_soft_general_csi<3>")
    c["psk16"] = (lambda: PSKModem(16), "demod_soft_general_csi<4>")
    c["custom16"] = (_custom16, "demod_soft_general_csi<4>")
    return c


CSI_CASES = sorted(["qam4", "qam16", "qam64", "qam256", "qam1024", "qam4096", "psk8", "psk16", "custom16"])


def _ran(fn, want):
    """fn() under the profiler; asserts that a kernel whose normalised name contains `want` ran (a profiling session that
    recorded the API calls but no kernel activity is repeated, at most four times)"""
    for _ in range(5):
        box = []
        names = helpers.launched_kernels(lambda: box.append(fn()))
        if any(want in n for n in names):
            break
    assert any(want in n for n in names), (want, sorted(names))
    return box[0]


def _gain_sets(cst, rs):
    """(h, noise variance) sets: Rayleigh draws with a few exact zeros; |h| fixed at 1e-6 .. 10 with random phases, the
    noise scaled with |h|^2 (the same effective SNR, so that fp32 keeps the LLRs to the tolerance); deep fades at a
    unit-gain noise variance."""
    d = np.abs(cst[:, None] - cst[None, :])
    dmin2 = float(np.min(d[d > 0])) ** 2
    n = 600
    ph = lambda: np.exp(2j * np.pi * rs.rand(n))
    ray = (rs.randn(n) + 1j * rs.randn(n)) / math.sqrt(2)
    ray[::97] = 0
    sets = [(ray, dmin2), (ray, 4 * dmin2)]
    for mag in (1e-6, 1e-3, 0.1, 3.0, 10.0):
        sets.append((mag * ph(), 0.3 * dmin2 * mag ** 2))
    sets.append((10 ** rs.uniform(-6, -2, n) * ph(), dmin2))
    return sets


@gpu
@pytest.mark.parametrize("case", CSI_CASES)
def test_csi_demapper_vs_fp64(case):
    """Soft: every LLR within 5e-4 + 5e-4 |L| of the fp64 restatement, LLR exactly 0 where h = 0.  Hard: the fp64 first-minimum
    argmin of |y - h c|^2 except on near ties, index 0 where h = 0.  The separable / general CSI kernels are the ones that ran."""
    import torch
    make, kern = _cases()[case]
    md = make()
    cst = np.asarray(md.constellation).astype(np.complex64).astype(np.complex128)
    nb = md.num_bits_symbol
    rs = np.random.RandomState(100 + CSI_CASES.index(case))
    for h, nv in _gain_sets(cst, rs):
        h = h.astype(np.complex64)
        n = len(h)
        y = (h.astype(np.complex128) * cst[rs.randint(0, len(cst), n)] +
             math.sqrt(nv / 2) * rs.uniform(0.3, 3, n) * (rs.randn(n) + 1j * rs.randn(n))).astype(np.complex64)
        yt, ht = torch.from_numpy(y).cuda(), torch.from_numpy(h).cuda()
        got = _ran(lambda: md.demodulate_batch(yt, "soft", nv, channel_gains=ht), "demap::" + kern).cpu().numpy()
        ref = csi_llr(y.astype(np.complex128), h.astype(np.complex128), cst, nv)
        err = np.abs(got - ref) - RTOL * np.abs(ref)
        assert (err <= ATOL).all(), (case, nv, float(err.max()), float(ref[np.argmax(err)]))
        zero = np.repeat(h == 0, nb)
        assert (got[zero] == 0).all()
        hard = _ran(lambda: md.demodulate_batch(yt, "hard", channel_gains=ht), "demap::demod_hard_csi_kernel")
        hard = hard.cpu().numpy().reshape(-1, nb)
        dist = np.abs(y.astype(np.complex128)[:, None] - h.astype(np.complex128)[:, None] * cst[None, :]) ** 2
        two = np.sort(dist, axis=1)[:, :2]
        ok = ((two[:, 1] - two[:, 0]) > 1e-5 * np.maximum(two[:, 1], 1e-300)) & (h != 0)
        want = (np.argmin(dist, axis=1)[:, None] >> np.arange(nb - 1, -1, -1)) & 1
        assert np.array_equal(hard[ok], want[ok]), (case, nv)
        assert not hard[h == 0].any()


@gpu
@pytest.mark.parametrize("case", CSI_CASES)
def test_csi_demapper_at_unit_gain_equals_awgn_demapper(case):
    """h = 1: cpb_demod_soft_csi / cpb_demod_hard_csi return exactly what cpb_demod_soft / cpb_demod_hard return."""
    import torch
    md = _cases()[case][0]()
    rs = np.random.RandomState(3)
    cst = np.asarray(md.constellation)
    y = cst[rs.randint(0, len(cst), 3000)] + 0.7 * (rs.randn(3000) + 1j * rs.randn(3000))
    yt = torch.from_numpy(y.astype(np.complex64)).cuda()
    for nv in (0.05, 1.0, 20.0):
        a = md.demodulate_batch(yt, "soft", nv, channel_gains=1.0).cpu().numpy()
        b = md.demodulate_batch(yt, "soft", nv).cpu().numpy()
        assert np.array_equal(a.view(np.int32), b.view(np.int32)), (case, nv)
    ones = torch.ones(3000, dtype=torch.complex64, device="cuda")
    assert torch.equal(md.demodulate_batch(yt, "hard", channel_gains=ones), md.demodulate_batch(yt, "hard"))


@gpu
def test_channel_gains_shape_must_match():
    import torch
    from commpy_b200.modulation import QAMModem
    md = QAMModem(16)
    y = torch.zeros((4, 10), dtype=torch.complex64, device="cuda")
    with pytest.raises(ValueError):
        md.demodulate_batch(y, "soft", 1.0, channel_gains=torch.ones(7, dtype=torch.complex64))
    with pytest.raises(ValueError):
        md.demodulate(np.zeros(10, complex), "hard", channel_gains=np.ones(9))
    # broadcasting: one gain per row
    h = torch.full((4, 1), 2.0 + 0j, dtype=torch.complex64, device="cuda")
    a = md.demodulate_batch(y + 1, "soft", 1.0, channel_gains=h)
    b = md.demodulate_batch(y + 1, "soft", 1.0, channel_gains=torch.full((4, 10), 2.0 + 0j, dtype=torch.complex64))
    assert torch.equal(a, b)


# ---------------------------------------------------------------- links
@gpu
def test_uncoded_qpsk_rayleigh_matches_theory():
    """Hard CSI decisions on the TX output (QPSK on +-1 +-j, Rayleigh) against the host conv_encode of msg: the channel-bit error
    rate is within 4 standard errors of 1/2 (1 - sqrt(g / (1 + g))) with g = E|h|^2 / (2 sigma^2) = 1 / (2 sigma^2), the
    mean SNR per bit when each real component carries amplitude |h| and noise of std sigma.  > 1e7 bits per point."""
    from commpy_b200.modulation import QAMModem
    tr = helpers.k7()
    md = QAMModem(4)
    frames, fb = 1280, 4096
    for i, sigma in enumerate((0.5, 0.2)):
        msg, y, h = conv_link_tx_fading(tr, md, frames, fb, 99 + i, 0, sigma, RAYLEIGH)
        coded = helpers.encode_batch(msg.cpu().numpy().astype(np.int64), tr).astype(np.uint8)
        errs = np.zeros(coded.size, np.uint8)
        for lo in range(0, frames, 128):                     # frames in slices: keeps the host memory small
            bits = md.demodulate_batch(y[lo:lo + 128], "hard", channel_gains=h[lo:lo + 128]).cpu().numpy()
            errs[lo * 2 * fb:(lo + 128) * 2 * fb] = (bits != coded[lo:lo + 128]).reshape(-1)
        assert errs.size >= 1e7
        per_sym = errs.reshape(-1, 2).sum(axis=1)           # the two bits of a symbol share h: count symbols as the unit
        ber = per_sym.mean() / 2
        se = per_sym.std() / 2 / math.sqrt(per_sym.size)
        g = 1 / (2 * sigma ** 2)
        want = 0.5 * (1 - math.sqrt(g / (1 + g)))
        print("uncoded QPSK Rayleigh sigma %.2f: %.5e (theory %.5e, se %.1e)" % (sigma, ber, want, se))
        assert abs(ber - want) < 4 * se, (sigma, ber, want, se)


@gpu
@pytest.mark.parametrize("mcs", [1, 4])
def test_wifi80211_gpu_fading_link_matches_reference_golden(mcs):
    """Wifi80211.link_performance_gpu over Rayleigh fading against the reference's Wifi80211.link_performance with
    SISOFlatChannel(None, (0j, 1)) and a receiver that equalises each symbol (oracle/make_fading_golden.py): within
    4 SE + 15 % + 2e-3 of the reference's BER at every point."""
    from commpy_b200.wifi80211 import Wifi80211
    g = np.load(os.path.join(GOLD, "fading_ber.npz"))
    snrs, fe, chunk = g["mcs%d_snr" % mcs], g["mcs%d_frame_errors" % mcs].astype(np.float64), int(g["chunk"])
    ref = fe.mean(axis=1) / chunk
    se = fe.std(axis=1, ddof=1) / chunk / np.sqrt(fe.shape[1])
    w = Wifi80211(mcs)
    got = [w.link_performance_gpu([float(s)], send_max=6e6, err_min=10 ** 9, send_chunk=chunk, frames_per_batch=2048, seed=3,
                                  stop_early=False, fading_param=RAYLEIGH)[0] for s in snrs]
    assert w.gpu_link.frame_bits == chunk
    print("mcs %d over Rayleigh: reference %s, GPU %s" % (mcs, list(ref), got))
    for b_ref, s_ref, b_gpu in zip(ref, se, got):
        assert abs(b_gpu - b_ref) <= 4 * s_ref + 0.15 * b_ref + 2e-3, (mcs, list(snrs), list(ref), list(se), got)
    assert min(ref) > 3e-3 and max(ref) < 0.1


@gpu
def test_host_linkmodel_with_csi_receiver_reproduces_reference_counts():
    """The host drop-in: with the golden's seed, LinkModel + SISOFlatChannel(None, (0j, 1)) + demodulate(y, 'hard',
    channel_gains=h) gives the reference's per-transmission error counts (the reference divides by h; at most one
    transmission may differ by an fp32 near-tie)."""
    from commpy_b200.channels import SISOFlatChannel
    from commpy_b200.links import LinkModel
    from commpy_b200.modulation import PSKModem
    g = np.load(os.path.join(GOLD, "fading_ber.npz"))
    chunk = int(g["chunk"])
    differ = 0
    for snr, want in zip(g["uncoded_snr"], g["uncoded_frame_errors"]):
        np.random.seed(int(g["uncoded_seed"]))
        modem = PSKModem(4)
        model = LinkModel(modem.modulate, SISOFlatChannel(None, RAYLEIGH),
                          lambda y, h, c, nv: modem.demodulate(y, "hard", channel_gains=h), modem.num_bits_symbol,
                          modem.constellation, modem.Es)
        _, bes, _, _ = model.link_performance_full_metrics([float(snr)], len(want), 10 ** 9, chunk, stop_on_surpass_error=False)
        differ += int((np.asarray(bes[0]) != want).sum())
    print("transmissions differing from the reference: %d" % differ)
    assert differ <= 1, differ


@gpu
def test_fading_counters_identical_for_1_2_4_8_ranks(monkeypatch):
    """Same seed => same error counters with fading, whatever the number of (emulated) ranks."""
    import torch
    from commpy_b200.modulation import QAMModem
    tr = helpers.k7()
    snr = 10.0 + 10 * np.log10(4)
    totals = {}
    for world in (1, 2, 4, 8):
        link = ConvLinkGPU(tr, QAMModem(16), frame_bits=1024, frames_per_batch=1024 // world, decoding_type="soft", seed=77,
                           fading_param=RAYLEIGH)
        tot = torch.zeros(3, dtype=torch.int64, device="cuda")
        for rank in range(world):
            monkeypatch.setenv("RANK", str(rank))
            monkeypatch.setenv("WORLD_SIZE", str(world))
            for b in range(3):
                msg, y, nv, h = link.make_batch(snr, b, torch)
                link.receive_decode_count(msg, y, nv, tot, torch, h)
        totals[world] = tot.cpu().numpy().copy()
    monkeypatch.delenv("RANK")
    monkeypatch.delenv("WORLD_SIZE")
    assert totals[1][0] > 0, "the test point must have bit errors to compare"
    for world in (2, 4, 8):
        assert np.array_equal(totals[world], totals[1]), (world, totals)


@gpu
def test_conv_link_gpu_fading_link_performance_runs():
    """ConvLinkGPU.link_performance with fading: hard and soft decoding, BER falls with SNR and soft beats hard; the Rayleigh
    BER is far above the AWGN one at the same SNR."""
    from commpy_b200.modulation import QAMModem
    tr = helpers.k7()
    snr = np.array([8.0, 14.0])
    res = {}
    for dt in ("soft", "hard"):
        link = ConvLinkGPU(tr, QAMModem(4), frame_bits=1024, frames_per_batch=256, decoding_type=dt, seed=4, fading_param=RAYLEIGH)
        res[dt] = link.link_performance(snr, send_max=2e6, err_min=10 ** 9, stop_early=False)
    awgn = ConvLinkGPU(tr, QAMModem(4), frame_bits=1024, frames_per_batch=256, seed=4).link_performance(
        snr[:1], send_max=2e6, err_min=10 ** 9, stop_early=False)
    assert res["soft"][0] > res["soft"][1] and res["hard"][0] > res["hard"][1], res
    assert res["soft"][0] < res["hard"][0], res
    assert res["soft"][0] > 10 * max(awgn[0], 1e-6), (res, awgn)

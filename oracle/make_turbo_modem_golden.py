"""BER of the UNMODIFIED reference's turbo code over QAM, AWGN and SISO flat fading, replayed by
tests/test_turbo_modem_gpu.py against TurboLinkGPU(modem=QAMModem(M)) with the same fading_param.

Per frame and point: c = np.concatenate of the three streams of turbo_encode(msg, rsc_k4, rsc_k4, RandInterlv(N, 1)), each
cut to N (commpy/channelcoding/turbo.py:14-59), QAMModem(M).modulate(c) (MSB first), SISOFlatChannel(None, fading_param)
with set_SNR_dB(EbN0 + 10 log10 nb, code_rate=1/3, Es) (channels.py:37-93, :176-221).  The receiver demaps with the true
complex noise variance N0 = noise_std^2 / 2: demodulate(y, 'soft', N0) over AWGN, demodulate(y_i / h_i, 'soft', N0 / |h_i|^2)
symbol by symbol over fading (what the CSI demapper computes), giving exact LLRs L = log P(1) / P(0).  L is the channel term
of turbo_decode's probability-domain BCJR at noise variance nv when fed as r = L nv / 2 (turbo.py:74: the channel term is
2 r / nv); nv = 2 / max(1, max |L|) keeps |r| <= 1, so no branch probability underflows (|L| <= 600 is asserted; the
points lie far below).  The decoder is the reference's turbo_decode(r_sys, r_par1, r_par2, trellis, nv, ITERATIONS, il).

    python oracle/make_turbo_modem_golden.py     # writes tests/golden/turbo_modem_ber.npz
                                                 # (3.5 minutes on 8 cores)
TEST INFRASTRUCTURE ONLY."""
import math
import os
import sys
import time
from multiprocessing import Pool

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path = [p for p in sys.path if os.path.abspath(p or ".") != HERE]
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np

import refimport

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
N, FRAMES, ITERATIONS, INTERLEAVER_SEED = 512, 100, 6, 1
LLR_MAX = 600.0
# name -> (QAM order, fading_param, Eb/N0 points in dB inside the waterfall: reference BER ~1e-3 .. 0.2)
# (far above the waterfall, e.g. 64-QAM over Rayleigh at 12.5 dB, the reference's probability-domain turbo loop fails on
# some frames as its extrinsic LLRs grow: those points measure that, not the channel)
CASES = {"qam4_awgn": (4, (1 + 0j, 0), [0.5, 0.75, 1.0]),
         "qam16_awgn": (16, (1 + 0j, 0), [2.5, 2.75, 3.0]),
         "qam16_rayleigh": (16, (0j, 1), [3.5, 4.0, 4.5]),
         "qam64_rayleigh": (64, (0j, 1), [6.0, 6.5, 7.0])}


def _ref():
    refimport.import_reference()
    import importlib
    return (importlib.import_module("commpy.channelcoding"), importlib.import_module("commpy.modulation"),
            importlib.import_module("commpy.channels"))


def receive(modem, y, h, N0, awgn):
    """exact LLRs log P(1) / P(0) of the received symbols (the reference's demapper, with CSI over fading)"""
    if awgn:
        return modem.demodulate(y, "soft", N0)
    return np.concatenate([modem.demodulate(y[i:i + 1] / h[i], "soft", N0 / abs(h[i]) ** 2) for i in range(len(y))])


def decoder_inputs(L):
    """(r, nv) with 2 r / nv == L and |r| <= 1: what the reference's probability-domain turbo_decode takes without
    underflow"""
    L = np.asarray(L, dtype=np.float64)
    amax = float(np.abs(L).max())
    assert np.isfinite(L).all() and amax <= LLR_MAX, amax
    nv = 2.0 / max(1.0, amax)
    return L * (nv / 2.0), nv


def point(args):
    (name, M, fp, ebn0), seed = args
    cc, rm, rch = _ref()
    trellis = cc.Trellis(np.array([3]), np.array([[1, 0o15]]), np.array([[0o13]]), "rsc")     # tests/helpers.py rsc_k4
    il = cc.RandInterlv(N, INTERLEAVER_SEED)
    modem = rm.QAMModem(M)
    nb = modem.num_bits_symbol
    np.random.seed(seed)
    errs = np.zeros(FRAMES, dtype=np.int64)
    ch = rch.SISOFlatChannel(None, fp)
    ch.set_SNR_dB(ebn0 + 10 * math.log10(nb), 1 / 3, modem.Es)
    N0 = ch.noise_std ** 2 / 2
    # TurboLinkGPU.noise_variance with a modem: sigma^2 = Es / (2 R nb Eb/N0) per real component
    assert abs(N0 / 2 - modem.Es / (2 * nb / 3 * 10 ** (ebn0 / 10))) <= 1e-12 * N0
    for f in range(FRAMES):
        msg = np.random.randint(0, 2, N)
        c = np.concatenate([np.asarray(s[:N]) for s in cc.turbo_encode(msg, trellis, trellis, il)])
        y = ch.propagate(modem.modulate(c))
        L = receive(modem, y, ch.channel_gains, N0, fp[1] == 0)
        r, nv = decoder_inputs(L)
        dec = cc.turbo_decode(r[:N], r[N:2 * N], r[2 * N:], trellis, nv, ITERATIONS, il)
        errs[f] = int(np.sum(np.asarray(dec[:N]) != msg))
    print(name, ebn0, errs.sum() / (N * FRAMES), flush=True)
    return errs


def main():
    jobs = []
    for c, (name, (M, fp, ebn0s)) in enumerate(CASES.items()):
        for i, e in enumerate(ebn0s):
            jobs.append(((name, M, fp, e), 7000 + 100 * c + i))
    t0 = time.time()
    with Pool(min(len(jobs), os.cpu_count() or 1)) as pool:
        res = pool.map(point, jobs, chunksize=1)
    out = {"N": np.array(N), "frames": np.array(FRAMES), "iterations": np.array(ITERATIONS),
           "interleaver_seed": np.array(INTERLEAVER_SEED)}
    for c, (name, (M, fp, ebn0s)) in enumerate(CASES.items()):
        out[name + "_M"] = np.array(M)
        out[name + "_fading_param"] = np.array([complex(fp[0]), complex(fp[1])])
        out[name + "_ebn0"] = np.array(ebn0s, dtype=np.float64)
        out[name + "_frame_errors"] = np.stack(res[3 * c:3 * c + 3])          # bit errors of every frame (N bits)
        out[name + "_ber"] = out[name + "_frame_errors"].sum(axis=1) / float(N * FRAMES)
    np.savez_compressed(os.path.join(GOLD, "turbo_modem_ber.npz"), **out)
    print("done in %.1f min" % ((time.time() - t0) / 60))


if __name__ == "__main__":
    main()

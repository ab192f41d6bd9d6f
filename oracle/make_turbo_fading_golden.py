"""BER of the UNMODIFIED reference's turbo code over SISO flat fading, replayed by tests/test_turbo_fading_gpu.py against
TurboLinkGPU with the same fading_param.

Per frame and point: turbo_encode(msg, rsc_k4, rsc_k4, RandInterlv(N, 1)) (commpy/channelcoding/turbo.py:14-59), BPSK 2x-1,
then each of the three streams through its own SISOFlatChannel(None, fading_param) with set_SNR_dB(EbN0, code_rate=1/3)
(channels.py:37-93, :176-221).  The receiver knows the channel: s = Re(conj(h) y) per value, decoded by the reference's
turbo_decode(s_sys, s_par1, s_par2, trellis, sigma^2, ITERATIONS, interleaver) (turbo.py:254-333) with sigma^2 the noise
variance per real component -- the exact MAP channel term 2 s / sigma^2 of y = h x + noise.

    python oracle/make_turbo_fading_golden.py     # writes tests/golden/turbo_fading_ber.npz
                                                  # (2.4 minutes on one core: 0.24 s per frame and point)
TEST INFRASTRUCTURE ONLY."""
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path = [p for p in sys.path if os.path.abspath(p or ".") != HERE]
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np

import refimport

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
N, FRAMES, ITERATIONS, INTERLEAVER_SEED = 512, 100, 6, 1
# name -> (fading_param, Eb/N0 points in dB inside the waterfall: BER ~3e-3 .. 0.1 with this code and N)
CASES = {"rayleigh": ((0j, 1), [1.5, 2.0, 2.5]),
         "rician": ((0.6 + 0j, 0.64), [1.0, 1.5, 2.0])}     # 0.64 + 0.6^2 == 1 passes the reference's energy check


def noise_variance(ebn0_db):
    """TurboLinkGPU.noise_variance: sigma^2 = 1 / (2 R Eb/N0), R = 1/3, E|h|^2 = 1"""
    return 1.0 / (2.0 * (1.0 / 3.0) * 10 ** (ebn0_db / 10.0))


def point(cc, rch, trellis, il, fading_param, ebn0, seed):
    np.random.seed(seed)
    s2 = noise_variance(ebn0)
    errs = np.zeros(FRAMES, dtype=np.int64)
    for f in range(FRAMES):
        msg = np.random.randint(0, 2, N)
        streams = cc.turbo_encode(msg, trellis, trellis, il)
        s = []
        for x in streams:
            ch = rch.SISOFlatChannel(None, fading_param)
            ch.set_SNR_dB(ebn0, code_rate=1 / 3)
            # the reference's complex noise is (N(0,1) + jN(0,1)) * noise_std / 2: sigma^2 per real component
            assert abs((ch.noise_std / 2) ** 2 - s2) <= 1e-12 * s2
            y = ch.propagate(2.0 * np.asarray(x[:N], dtype=np.float64) - 1.0)
            s.append(np.real(np.conj(ch.channel_gains) * y))
        dec = cc.turbo_decode(s[0], s[1], s[2], trellis, s2, ITERATIONS, il)
        errs[f] = int(np.sum(np.asarray(dec[:N]) != msg))
    return errs


def main():
    refimport.import_reference()
    import importlib
    cc = importlib.import_module("commpy.channelcoding")
    rch = importlib.import_module("commpy.channels")
    trellis = cc.Trellis(np.array([3]), np.array([[1, 0o15]]), np.array([[0o13]]), "rsc")     # tests/helpers.py rsc_k4
    il = cc.RandInterlv(N, INTERLEAVER_SEED)
    out = {"N": np.array(N), "frames": np.array(FRAMES), "iterations": np.array(ITERATIONS),
           "interleaver_seed": np.array(INTERLEAVER_SEED)}
    t0 = time.time()
    for k, (name, (fp, ebn0s)) in enumerate(CASES.items()):
        per_frame = []
        for i, e in enumerate(ebn0s):
            errs = point(cc, rch, trellis, il, fp, e, 5000 + 100 * k + i)
            per_frame.append(errs)
            print(name, e, errs.sum() / (N * FRAMES), errs.sum(), (errs > 0).sum(), "%.0f s" % (time.time() - t0), flush=True)
        out[name + "_fading_param"] = np.array([complex(fp[0]), complex(fp[1])])
        out[name + "_ebn0"] = np.array(ebn0s, dtype=np.float64)
        out[name + "_frame_errors"] = np.stack(per_frame)                  # bit errors of every frame (N bits)
        out[name + "_ber"] = out[name + "_frame_errors"].sum(axis=1) / float(N * FRAMES)
    np.savez_compressed(os.path.join(GOLD, "turbo_fading_ber.npz"), **out)
    print("done in %.1f min" % ((time.time() - t0) / 60))


if __name__ == "__main__":
    main()

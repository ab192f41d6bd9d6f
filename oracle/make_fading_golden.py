"""BER of the UNMODIFIED reference over Rayleigh flat fading, replayed by tests/test_fading_gpu.py against the batched GPU link
with fading_param = (0j, 1) (ConvLinkGPU / Wifi80211.link_performance_gpu) and against the host LinkModel drop-in.

* Coded: Wifi80211(mcs).link_performance(SISOFlatChannel(None, (0j, 1)), ...) (commpy/wifi80211.py:132-216) with a receiver
  that knows the channel: per symbol, demodulate(y / h, 'soft', nv / |h|^2) -- the reference's default receiver ignores h.
* Uncoded: LinkModel with PSKModem(4), the same channel and demodulate(y / h, 'hard'), per-transmission bit errors for a
  fixed np.random.seed.

    python oracle/make_fading_golden.py          # writes tests/golden/fading_ber.npz (about ten minutes on one core)
TEST INFRASTRUCTURE ONLY."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path = [p for p in sys.path if os.path.abspath(p or ".") != HERE]
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np

import refimport

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
CASES = {1: [12.0, 13.5], 4: [24.0, 26.0]}        # mcs -> SNR_dB points where the reference's BER is ~3e-3 .. 1e-1
UNCODED_SNRS = [6.0, 12.0]
FRAMES, CHUNK = 64, 600
UNCODED_SEED = 2718


def csi_receiver(modem):
    """what a CommPy user writes for a flat-fading SISO link: equalise each symbol and scale the noise variance"""
    def receive(y, h, constellation, noise_var):
        return np.concatenate([modem.demodulate(y[i:i + 1] / h[i], "soft", noise_var / abs(h[i]) ** 2)
                               for i in range(len(y))])
    return receive


def coded_point(rw, rch, mcs, snr, frames=FRAMES):
    np.random.seed(2000 + mcs)
    w = rw.Wifi80211(mcs)
    ch = rch.SISOFlatChannel(None, (0j, 1))
    b, bes, _, _ = w.link_performance(ch, [snr], frames, 10 ** 9, CHUNK, receiver=csi_receiver(w.get_modem()),
                                      stop_on_surpass_error=False)
    return float(b[0]), np.asarray(bes[0], dtype=np.int64).reshape(-1)


def uncoded_point(rl, rm, rch, snr, frames=FRAMES):
    np.random.seed(UNCODED_SEED)
    modem = rm.PSKModem(4)
    ch = rch.SISOFlatChannel(None, (0j, 1))
    model = rl.LinkModel(modem.modulate, ch, lambda y, h, c, nv: modem.demodulate(y / h, "hard"), modem.num_bits_symbol,
                         modem.constellation, modem.Es)
    b, bes, _, _ = model.link_performance_full_metrics([snr], frames, 10 ** 9, CHUNK, stop_on_surpass_error=False)
    return float(b[0]), np.asarray(bes[0], dtype=np.int64).reshape(-1)


def main():
    refimport.import_reference()
    import importlib
    rw = importlib.import_module("commpy.wifi80211")
    rch = importlib.import_module("commpy.channels")
    rl = importlib.import_module("commpy.links")
    rm = importlib.import_module("commpy.modulation")
    out = {}
    for mcs, snrs in CASES.items():
        bers, per_frame = [], []
        for snr in snrs:                       # one call per point, each from its own seed
            b, bes = coded_point(rw, rch, mcs, snr)
            bers.append(b)
            per_frame.append(bes)
            print(mcs, snr, b, bes.sum(), len(bes), flush=True)
        out["mcs%d_snr" % mcs] = np.array(snrs)
        out["mcs%d_ber" % mcs] = np.array(bers, dtype=np.float64)
        out["mcs%d_frame_errors" % mcs] = np.stack(per_frame)          # bit errors of every transmission (CHUNK bits)
    errs = []
    for snr in UNCODED_SNRS:
        b, bes = uncoded_point(rl, rm, rch, snr)
        errs.append(bes)
        print("uncoded", snr, b, bes.sum(), flush=True)
    out["uncoded_snr"] = np.array(UNCODED_SNRS)
    out["uncoded_frame_errors"] = np.stack(errs)
    out["uncoded_seed"] = np.array(UNCODED_SEED)
    out["chunk"] = np.array(CHUNK)
    np.savez_compressed(os.path.join(GOLD, "fading_ber.npz"), **out)


if __name__ == "__main__":
    main()

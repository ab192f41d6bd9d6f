"""Cost of flat fading on one GPU: the fading TX kernels against the AWGN ones, the channel-aware demapper against the plain one,
and the config-5 link (256-QAM, K=7, 4096-bit frames, soft) with and without fading_param = (0j, 1).  CUDA events, a warm-up
of every shape, and at least 1e8 symbols per timed window.  Prints the card and its power limit first.

    python scripts/exp_fading.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import helpers
from commpy_b200.links import ConvLinkGPU, conv_link_tx, conv_link_tx_fading
from commpy_b200.modulation import Modem, PSKModem, QAMModem

MIN_SYMBOLS = 1e8


def timed(fn, per_call, warmup=2):
    """seconds per call of fn() over a window of at least MIN_SYMBOLS symbols (per_call symbols per call)"""
    for _ in range(warmup):
        fn()
    calls = max(3, int(np.ceil(MIN_SYMBOLS / per_call)))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / calls


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q), flush=True)
    tr = helpers.k7()
    # -- TX
    for m in (4, 256):
        modem = QAMModem(m)
        nsym = 4096 * 2 // modem.num_bits_symbol
        frames = (1 << 24) // nsym
        n = frames * nsym
        t_awgn = timed(lambda: conv_link_tx(tr, modem, frames, 4096, 1, 0, 0.3), n)
        t_fad = timed(lambda: conv_link_tx_fading(tr, modem, frames, 4096, 1, 0, 0.3, (0j, 1)), n)
        print("TX %d-QAM K=7 4096-bit frames: AWGN %.3e sym/s, Rayleigh %.3e sym/s (%.2fx time)"
              % (m, n / t_awgn, n / t_fad, t_fad / t_awgn), flush=True)
    # -- demapper
    rs = np.random.RandomState(0)
    n = 1 << 25
    y = torch.view_as_complex(torch.randn(n, 2, device="cuda") * 4)
    h = torch.view_as_complex(torch.randn(n, 2, device="cuda") * 0.7071)
    for name, md in (("256-QAM separable", QAMModem(256)), ("16-QAM separable", QAMModem(16)),
                     ("256-point general", Modem(rs.randn(256) * 8 + 8j * rs.randn(256))),
                     ("16-PSK general", PSKModem(16))):
        nb = md.num_bits_symbol
        t_plain = timed(lambda: md.demodulate_batch(y, "soft", 2.0), n)
        t_csi = timed(lambda: md.demodulate_batch(y, "soft", 2.0, channel_gains=h), n)
        print("demap %s: plain %.3e sym/s (%.2f TB/s), CSI %.3e sym/s (%.2f TB/s), CSI/plain time %.2f"
              % (name, n / t_plain, n * (8 + 4 * nb) / t_plain * 1e-12, n / t_csi, n * (16 + 4 * nb) / t_csi * 1e-12,
                 t_csi / t_plain), flush=True)
    del y, h
    # -- config-5 link step: TX -> demap -> soft Viterbi -> error count, frames_per_batch 4096
    snr = 13.0 + 10 * np.log10(8)
    for fp in (None, (0j, 1)):
        link = ConvLinkGPU(tr, QAMModem(256), frame_bits=4096, frames_per_batch=4096, decoding_type="soft", seed=5,
                           fading_param=fp)
        cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
        state = {"b": 0}

        def step():
            msg, y, nv, *g = link.make_batch(snr, state["b"], torch)
            state["b"] += 1
            link.receive_decode_count(msg, y, nv, cnt, torch, *g)
        per = 4096 * 4096 * 2 // 8
        t = timed(step, per)
        print("link C5 (256-QAM, K=7, 4096-bit frames, soft) %s: %.3e sym/s, %.3e info bits/s"
              % ("AWGN" if fp is None else "Rayleigh (0j, 1)", per / t, 4096 * 4096 / t), flush=True)


if __name__ == "__main__":
    main()

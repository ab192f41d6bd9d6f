"""Where the time of an LDPC link step goes at the C4 shape on one GPU: the DVB-S2-shaped surrogate code (tests/helpers.py
dvbs2_like_H, 64,800 x 32,400, staircase parity part), 256-QAM, min-sum fp32 with 50 iterations, 128 and 1,024 frames.
Stages, each timed alone with CUDA events over device-resident calls after a warm-up: encode (cpb_ldpc_encode of
caller-supplied messages), TX (cpb_ldpc_link_tx: message + encode + modulate + AWGN), demap (soft, 256-QAM), decode (50
iterations, no early stop at a low SNR) and count (cpb_count_errors).  Per-kernel device times of the TX from one
torch.profiler pass of its own.  Prints the card and its power limit first.

    python scripts/exp_ldpc_link.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import helpers
from commpy_b200.channelcoding import ldpc_bp_decode_batch, ldpc_encode_batch
from commpy_b200.links import LdpcLinkGPU, _count_errors
from commpy_b200.modulation import QAMModem

ITERS = 50
SNR_DB = 8.0          # well below the waterfall: no frame stops early, every call runs all 50 iterations


def timed(fn, calls, warmup=2):
    """seconds per call of fn(), CUDA events around `calls` back-to-back calls"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / calls


def kernel_times(fn, calls=5):
    """mean device time (s) per launch of each ldpclink kernel, and of the shared code-word modulator (cwtx::), over `calls`
    calls of fn(), from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if ("ldpclink::" in e.key or "cwtx::" in e.key) and e.count:
            t = getattr(e, "device_time_total", None)
            t = e.cuda_time_total if t is None else t
            out[e.key.split("(")[0]] = t * 1e-6 / e.count
    return out


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q), flush=True)
    H = helpers.dvbs2_like_H()
    m, n = H.shape
    k = n - m
    params = {"parity_check_matrix": H.tocsc(), "n_vnodes": n, "n_cnodes": m}
    modem = QAMModem(256)
    for frames in (128, 1024):
        link = LdpcLinkGPU(params, modem, frames, n_iters=ITERS, seed=1)
        msg, y, nv = link.make_batch(SNR_DB, 0)
        llr = link.llrs(y, nv)
        dec = ldpc_bp_decode_batch(llr.clone(), params, ITERS, return_llrs=False)
        counters = torch.zeros(3, dtype=torch.int64, device="cuda")
        t = {
            "encode": timed(lambda: ldpc_encode_batch(msg, params), 20),
            "tx": timed(lambda: link.make_batch(SNR_DB, 0), 20),
            "demap": timed(lambda: link.llrs(y, nv), 20),
            "decode": timed(lambda: ldpc_bp_decode_batch(llr.clone(), params, ITERS, return_llrs=False), 3, warmup=1),
            "count": timed(lambda: _count_errors(dec, msg, counters, torch), 50),
        }
        tot = sum(v for s, v in t.items() if s != "encode")
        print("C4 shape (dvbs2_like_H, 256-QAM, %d iterations), %d frames:" % (ITERS, frames))
        for s, v in t.items():
            print("  %-7s %9.3f ms  %5.1f %% of the decode" % (s, v * 1e3, 100 * v / t["decode"]))
        print("  link step (tx + demap + decode + count) %.3f ms; tx / decode = %.2f %%, encode / decode = %.2f %%"
              % (tot * 1e3, 100 * t["tx"] / t["decode"], 100 * t["encode"] / t["decode"]))
        ndec = (dec[:, :k] != msg).any(dim=1).sum().item()
        print("  frames not decoded at %.1f dB: %d of %d (all must run every iteration)" % (SNR_DB, ndec, frames))
        for name, v in sorted(kernel_times(lambda: link.make_batch(SNR_DB, 0)).items()):
            print("  kernel %s: %.3f ms per launch" % (name, v * 1e3))
        # algorithmic bytes of the TX per frame: k message bytes written, packed message written and read once per H_s
        # edge (L2), syndrome and parity words, m parity bytes written and read, n bytes read by the mapper, 8 B per symbol
        nsym = n // modem.num_bits_symbol
        tx_bytes = frames * (k + m + n + 8 * nsym)
        print("  tx: %.1f MB of message, parity and symbol bytes per call, %.2f TB/s achieved"
              % (tx_bytes / 1e6, tx_bytes / t["tx"] / 1e12), flush=True)


if __name__ == "__main__":
    main()

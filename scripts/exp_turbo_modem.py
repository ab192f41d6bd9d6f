"""Cost of a modem for the turbo link on one GPU: the modem TX (message, parity and shared modulate kernels), the receiver's
demapper, LLR stream split and turbo decode, per kernel; and a config-3-shaped link step (rsc_k4, N = 6144, 8,192 codewords,
6 iterations: TX -> demap -> split -> turbo decode -> error count) for 16-QAM and 256-QAM over AWGN and Rayleigh (0j, 1),
against the BPSK TurboLinkGPU step, alternated.  CUDA events around device-resident calls, every shape warmed up; per-kernel
device times from torch.profiler passes of their own.  Prints the card and its power limit first.

    python scripts/exp_turbo_modem.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import helpers
from commpy_b200.channelcoding import RandInterlv, turbo_decode_batch
from commpy_b200.links import TurboLinkGPU
from commpy_b200.modulation import QAMModem

N, FRAMES, ITERS = 6144, 8192, 6
RAYLEIGH = (0j, 1)


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


def kernel_times(fn, calls=3):
    """{kernel: mean device seconds per call of fn()} over `calls` calls, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if e.count and t > 0 and not e.key.startswith(("cuda", "Memcpy", "Memset")):
            out[e.key.split("(")[0]] = t * 1e-6 / calls
    return out


def stage(name):
    """the receiver stage a kernel belongs to"""
    if "demod" in name:
        return "demap"
    if "count_errors" in name:
        return "count"
    if "turbolink::" in name or "cwtx::" in name:
        return "tx"
    if "map_" in name or "bcjr" in name or "_sub_kernel" in name or "bits" in name or "step_major" in name:
        return "decode"
    return "split (torch copies)"


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q), flush=True)
    tr, il = helpers.rsc_k4(), RandInterlv(N, 1)
    cnt = torch.zeros(3, dtype=torch.int64, device="cuda")

    # -- per kernel: TX, then receiver (demap, split, decode, count), one configuration at a time
    for M, fp, ebn0 in ((16, None, 3.0), (16, RAYLEIGH, 4.5), (256, None, 9.0), (256, RAYLEIGH, 12.0)):
        link = TurboLinkGPU(tr, il, N, frames_per_batch=FRAMES, iterations=ITERS, seed=5, modem=QAMModem(M), fading_param=fp)
        kt = kernel_times(lambda: link.make_batch(ebn0, 0))
        batch = link.make_batch(ebn0, 0)
        kr = kernel_times(lambda: link.decode_count(*batch, cnt, torch))
        print("%d-QAM %s, %.1f dB, %d codewords of N=%d:" % (M, "AWGN" if fp is None else fp, ebn0, FRAMES, N), flush=True)
        for name, t in sorted(kt.items()):
            print("  TX kernel %s: %.3f ms" % (name, t * 1e3))
        stages = {}
        for name, t in sorted(kr.items()):
            s = stage(name)
            stages[s] = stages.get(s, 0.0) + t
            print("  RX kernel [%s] %s: %.3f ms" % (s, name, t * 1e3))
        tx = sum(kt.values())
        dec = stages.get("decode", 0.0)
        extra = tx + stages.get("demap", 0.0) + stages.get("split (torch copies)", 0.0)
        print("  stages: TX %.3f ms, %s; TX + demap + split = %.1f %% of the decode"
              % (tx * 1e3, ", ".join("%s %.3f ms" % (k, v * 1e3) for k, v in sorted(stages.items())), 100 * extra / dec),
              flush=True)
        del batch
    # the decoder alone on the split streams, as a cross-check of the profiler's decode stage
    link = TurboLinkGPU(tr, il, N, frames_per_batch=FRAMES, iterations=ITERS, seed=5, modem=QAMModem(16))
    batch = link.make_batch(3.0, 0)
    streams = link.llr_streams(*batch[1:])
    t_dec = timed(lambda: turbo_decode_batch(*streams, tr, 2.0, ITERS, il), 5)
    print("turbo_decode_batch alone on the split 16-QAM LLR streams: %.2f ms" % (t_dec * 1e3), flush=True)
    del batch, streams
    torch.cuda.empty_cache()

    # -- link step: make_batch + decode_count, alternated
    links = {"BPSK AWGN": (TurboLinkGPU(tr, il, N, FRAMES, ITERS, 5), 1.0),
             "16-QAM AWGN": (TurboLinkGPU(tr, il, N, FRAMES, ITERS, 5, modem=QAMModem(16)), 3.0),
             "16-QAM Rayleigh": (TurboLinkGPU(tr, il, N, FRAMES, ITERS, 5, RAYLEIGH, QAMModem(16)), 4.5),
             "256-QAM AWGN": (TurboLinkGPU(tr, il, N, FRAMES, ITERS, 5, modem=QAMModem(256)), 9.0),
             "256-QAM Rayleigh": (TurboLinkGPU(tr, il, N, FRAMES, ITERS, 5, RAYLEIGH, QAMModem(256)), 12.0)}
    res = {k: [] for k in links}
    for rnd in range(3):
        for name, (link, ebn0) in links.items():
            state = {"b": 0}

            def step():
                b = link.make_batch(ebn0, state["b"])
                state["b"] += 1
                link.decode_count(*b, cnt, torch)
            t = timed(step, 6)
            res[name].append(t)
            print("link step (rsc_k4, N=%d, %d codewords, %d iterations) %s, round %d: %.2f ms, %.3e codewords/s"
                  % (N, FRAMES, ITERS, name, rnd, t * 1e3, FRAMES / t), flush=True)
    base = np.array(res["BPSK AWGN"])
    for name, ts in res.items():
        ts = np.array(ts)
        print("link step %s: mean %.2f ms, %.3f x the BPSK step" % (name, ts.mean() * 1e3, ts.mean() / base.mean()), flush=True)


if __name__ == "__main__":
    main()

"""Cost of flat fading for the turbo link on one GPU: the fading turbo TX against the AWGN one, the coherent BPSK combiner, and
a config-3-shaped link step (rsc_k4, N = 6144, 8,192 codewords, 6 iterations: TX -> [combine] -> turbo decode -> error count)
over Rayleigh (0j, 1) against AWGN, alternated.  CUDA events around device-resident calls, every shape warmed up; per-kernel
device times from one torch.profiler pass of its own.  Prints the card and its power limit first.

    python scripts/exp_turbo_fading.py"""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import helpers
from commpy_b200 import _lib
from commpy_b200.channelcoding import RandInterlv
from commpy_b200.channelcoding.convcode import _trellis_handle
from commpy_b200.links import TurboLinkGPU, bpsk_combine

N, FRAMES, ITERS = 6144, 8192, 6


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
    """mean device time (s) per launch of each turbolink kernel over `calls` calls of fn(), from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "turbolink::" in e.key and e.count:
            t = getattr(e, "device_time_total", None)
            t = e.cuda_time_total if t is None else t
            out[e.key.split("(")[0]] = t * 1e-6 / e.count
    return out


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(0), q), flush=True)
    lib = _lib.load()
    tr, il = helpers.rsc_k4(), RandInterlv(N, 1)
    th = _trellis_handle(tr)
    perm = torch.from_numpy(np.asarray(il.p_array, dtype=np.int32)).cuda()
    msg = torch.empty((FRAMES, N), dtype=torch.uint8, device="cuda")
    streams = torch.empty((3, FRAMES, N), dtype=torch.float32, device="cuda")
    y, h = (torch.empty((3, FRAMES, N), dtype=torch.complex64, device="cuda") for _ in range(2))
    st = _lib.stream_ptr(torch)
    sigma = float(np.sqrt(TurboLinkGPU(tr, il, N).noise_variance(1.0)))
    values = 3 * FRAMES * N

    def tx_awgn():
        _lib.check(lib.cpb_turbo_link_tx(th, _lib.ptr(perm), C.c_int64(FRAMES), C.c_int64(N), C.c_uint64(1), C.c_int64(0),
                                         C.c_float(sigma), _lib.ptr(msg), _lib.ptr(streams[0]), _lib.ptr(streams[1]),
                                         _lib.ptr(streams[2]), st), "turbo_link_tx")

    def tx_fading():
        _lib.check(lib.cpb_turbo_link_tx_fading(th, _lib.ptr(perm), C.c_int64(FRAMES), C.c_int64(N), C.c_uint64(1),
                                                C.c_int64(0), C.c_float(sigma), C.c_float(0.0), C.c_float(0.0),
                                                C.c_float(1.0), _lib.ptr(msg), _lib.ptr(y), _lib.ptr(h), st),
                   "turbo_link_tx_fading")

    # -- TX: call time (message kernel + encode kernel) alternated, then per-kernel device time
    for rnd in range(2):
        t_a = timed(tx_awgn, 10)
        t_f = timed(tx_fading, 10)
        print("TX call, %d codewords of N=%d (round %d): AWGN %.3f ms, Rayleigh %.3f ms (%.2fx time); %.3e vs %.3e values/s"
              % (FRAMES, N, rnd, t_a * 1e3, t_f * 1e3, t_f / t_a, values / t_a, values / t_f), flush=True)
    ka, kf = kernel_times(tx_awgn), kernel_times(tx_fading)
    for name, t in sorted(ka.items()) + sorted(kf.items()):
        print("  kernel %s: %.3f ms per launch" % (name, t * 1e3), flush=True)
    enc_a = [t for k, t in ka.items() if "encode_kernel" in k]
    enc_f = [t for k, t in kf.items() if "encode_kernel" in k]
    if enc_a and enc_f:
        print("encode kernel: Rayleigh / AWGN time %.2fx" % (enc_f[0] / enc_a[0]), flush=True)

    # -- combiner: y, h complex64 in, s float32 out (20 B per value)
    tx_fading()
    s = torch.empty((3, FRAMES, N), dtype=torch.float32, device="cuda")

    def combine():
        _lib.check(lib.cpb_bpsk_combine(_lib.ptr(y), _lib.ptr(h), C.c_int64(values), _lib.ptr(s), st), "bpsk_combine")
    combine()
    assert torch.equal(s, bpsk_combine(y, h))
    t_c = timed(combine, 20)
    print("combine %d values: %.3f ms, %.3e values/s, %.2f TB/s achieved (20 B per value)"
          % (values, t_c * 1e3, values / t_c, 20.0 * values / t_c * 1e-12), flush=True)
    del streams, y, h, s
    torch.cuda.empty_cache()

    # -- config-3-shaped link step: make_batch + decode_count, AWGN and Rayleigh alternated
    links = {"AWGN": TurboLinkGPU(tr, il, N, frames_per_batch=FRAMES, iterations=ITERS, seed=5),
             "Rayleigh (0j, 1)": TurboLinkGPU(tr, il, N, frames_per_batch=FRAMES, iterations=ITERS, seed=5,
                                              fading_param=(0j, 1))}
    cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
    res = {k: [] for k in links}
    for rnd in range(3):
        for name, link in links.items():
            state = {"b": 0}

            def step():
                batch = link.make_batch(1.0, state["b"])
                state["b"] += 1
                link.decode_count(*batch, cnt, torch)
            t = timed(step, 8)
            res[name].append(t)
            print("link step (rsc_k4, N=%d, %d codewords, %d iterations) %s, round %d: %.2f ms, %.3e codewords/s"
                  % (N, FRAMES, ITERS, name, rnd, t * 1e3, FRAMES / t), flush=True)
    a, f = np.array(res["AWGN"]), np.array(res["Rayleigh (0j, 1)"])
    print("link step Rayleigh / AWGN time: %.3f (rounds %s)" % (f.mean() / a.mean(), ", ".join("%.3f" % r for r in f / a)),
          flush=True)


if __name__ == "__main__":
    main()

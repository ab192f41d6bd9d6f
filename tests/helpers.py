"""Shared helpers for the parity tests: trellises, seeded channel inputs."""
import warnings

import numpy as np

from commpy_b200.channelcoding.convcode import Trellis, conv_encode


def k7():
    return Trellis(np.array([6]), np.array([[0o133, 0o171]]))


def k7_wifi_quirk():
    """Trellis of DECIMAL (133, 171) as commpy/wifi80211.py:49 builds it (taps 5, 43)."""
    return Trellis(np.array([6]), np.array([[133, 171]]))


def k7_171_133():
    """The K=7 code with its two generators swapped (octal 171, 133)."""
    return Trellis(np.array([6]), np.array([[0o171, 0o133]]))


def mem6_5_7():
    """Trellis([6], [[5, 7]]): the 64-state trellis of commpy/channelcoding/README.md:81-84."""
    return Trellis(np.array([6]), np.array([[5, 7]]))


def reference_test_trellises():
    """The five trellises of commpy/channelcoding/tests/test_convcode.py:23-111."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return [
            Trellis(np.array([2]), np.array([[5, 7]]), code_type="default"),
            Trellis(np.array([2]), np.array([[1, 7]]), 5, "rsc"),
            Trellis(np.array([2, 1]), np.array([[5, 7, 0], [0, 2, 3]]), code_type="default"),
            Trellis(np.array([2, 1]), np.array([[5, 7, 0], [0, 2, 6]]), code_type="default", polynomial_format="LSB"),
            Trellis(np.array([1, 1]), np.array([[1, 0, 0], [0, 1, 3]]), np.array([[2, 2], [3, 1]]), "rsc"),
        ]


def rsc_k4():
    """K=4 RSC (8 states) of SURVEY.md section 8c: Trellis([3], [[1, 0o15]], [[0o13]], 'rsc')."""
    return Trellis(np.array([3]), np.array([[1, 0o15]]), np.array([[0o13]]), "rsc")


def encode_batch(msgs, trellis, termination="cont"):
    """conv_encode for a (batch, nbits) array of messages: the table walk of convcode.py:535-540 vectorised over
    frames (checked against conv_encode in tests/test_host_mirror.py)."""
    msgs = np.asarray(msgs)
    k, n, M = trellis.k, trellis.n, trellis.total_memory
    if termination == "term":
        if trellis.code_type == "rsc":
            return np.stack([conv_encode(m, trellis, termination) for m in msgs])
        msgs = np.concatenate([msgs, np.zeros((msgs.shape[0], M + M % k), msgs.dtype)], axis=1)
    batch, nin = msgs.shape
    steps = nin // k
    nst = np.asarray(trellis.next_state_table)
    otab = np.asarray(trellis.output_table)
    words = msgs[:, :steps * k].reshape(batch, steps, k) @ (1 << np.arange(k - 1, -1, -1))
    state = np.zeros(batch, dtype=np.int64)
    out = np.zeros((batch, int(nin / (k / n))), dtype=np.int64)
    shifts = np.arange(n - 1, -1, -1)
    for t in range(steps):
        w = words[:, t]
        o = otab[state, w]
        out[:, t * n:(t + 1) * n] = (o[:, None] >> shifts) & 1
        state = nst[state, w]
    return out


def channel_frames(trellis, rs, batch, nbits, mode, termination="cont", flip=0.03, ebn0_db=4.0):
    """Encode `batch` random messages and pass them through BSC (hard) or BPSK-AWGN (soft: LLR = 2y/sigma^2,
    positive favours 1; unquantized: y).  Returns (msgs, channel_values)."""
    msgs = rs.randint(0, 2, (batch, nbits))
    coded = encode_batch(msgs, trellis, termination).astype(np.float64)
    rate = trellis.k / trellis.n
    if mode == "hard":
        x = np.abs(coded - (rs.rand(*coded.shape) < flip))
    else:
        sigma2 = 1.0 / (2.0 * rate * 10 ** (ebn0_db / 10.0))
        y = (2 * coded - 1) + np.sqrt(sigma2) * rs.randn(*coded.shape)
        x = 2 * y / sigma2 if mode == "soft" else y
    return msgs, x


def dvbs2_like_H(seed=3, n=64800, m=32400, n8=12960, n3=19440):
    """DVB-S2-SHAPED surrogate parity-check matrix (the reference ships no DVB-S2 design and there is no network,
    SURVEY.md section 7-3): same size (32400 x 64800), same degree profile as the rate-1/2 normal frame
    (12,960 information columns of degree 8, 19,440 of degree 3, dual-diagonal staircase parity part, every
    check of degree 7 except the first: 226,799 edges), information edges placed pseudo-randomly from `seed`.
    It is NOT the ETSI EN 302 307 address table.  Returns a scipy CSR int8 matrix."""
    import scipy.sparse as sp
    rs = np.random.RandomState(seed)
    k = n - m
    assert n8 + n3 == k
    deg = np.concatenate([np.full(n8, 8), np.full(n3, 3)])
    slots = np.repeat(np.arange(m), (deg.sum() + m - 1) // m)[:deg.sum()]       # 5 information edges per check
    for _ in range(200):
        rs.shuffle(slots)
        cols = np.repeat(np.arange(k), deg)
        key = cols.astype(np.int64) * m + slots
        order = np.argsort(key, kind="stable")
        dup = np.zeros(len(key), bool)
        dup[order[1:]] = key[order][1:] == key[order][:-1]
        if not dup.any():
            break
        # repair duplicates by swapping the offending slots with random other positions
        bad = np.nonzero(dup)[0]
        other = rs.randint(0, len(slots), len(bad))
        slots[bad], slots[other] = slots[other].copy(), slots[bad].copy()
        key = cols.astype(np.int64) * m + slots
        if len(np.unique(key)) == len(key):
            break
    rows = [slots, np.arange(m), np.arange(1, m)]
    colsl = [np.repeat(np.arange(k), deg), k + np.arange(m), k + np.arange(m - 1)]
    r = np.concatenate(rows)
    c = np.concatenate(colsl)
    H = sp.csr_matrix((np.ones(len(r), np.int8), (r, c)), shape=(m, n))
    H.data[:] = 1
    H.sort_indices()
    return H


def mixed_degree_H(row_degrees, n, seed=0):
    """Parity-check matrix with the given row degrees (one row per entry) over n columns, edges placed at random without
    repeats; every column gets at least one edge when the degrees allow it.  Returns a scipy CSR int8 matrix."""
    import scipy.sparse as sp
    rs = np.random.RandomState(seed)
    rows, cols = [], []
    unused = list(rs.permutation(n))
    for i, d in enumerate(row_degrees):
        take = [unused.pop() for _ in range(min(d, len(unused)))]
        rest = np.setdiff1d(np.arange(n), take)
        take += list(rs.choice(rest, d - len(take), replace=False))
        rows += [i] * d
        cols += take
    H = sp.csr_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(len(row_degrees), n))
    H.sort_indices()
    return H


def normalize_kernel_name(name):
    """Kernel name without spaces, integer casts and integer suffixes, so that the profiler's demangling
    ('FFCode<6, 5u, 7u>') and cu++filt's ('FFCode<(int)6, (unsigned int)5, (unsigned int)7>') compare equal."""
    import re
    s = re.sub(r"\((?:unsigned |signed )?(?:int|long long|long|short|char)\)", "", name)
    s = s.replace(" ", "")
    return re.sub(r"(?<=\d)(?:ull|ll|ul|u|l)(?=[,>)])", "", s)


def launched_kernels(fn):
    """Run fn() under torch.profiler (CUDA activity only: CUPTI sees every kernel of the process, including the ones the
    ctypes library launches on its own pipeline streams) and return the normalised names of what it recorded: the
    kernels launched, plus the runtime API calls (cudaLaunchKernel, ...) that made them.

    Kineto maps CUPTI's GPU timestamps onto the host clock from a sync taken when CUPTI starts, and drops every GPU record
    whose mapped time falls outside the profiling window.  On some hosts that mapping drifts by more than a second within
    a minute of the first session, and the kernel records are then lost ("Out-of-range" in Kineto's record counts).
    TEARDOWN_CUPTI=1 finalises CUPTI after each session, so that every session starts it, and its clock sync, afresh.
    The teardown runs on a thread of its own and a session started before it ends records nothing: hence the pause."""
    import os
    import time

    import torch
    from torch.profiler import ProfilerActivity, profile
    os.environ["TEARDOWN_CUPTI"] = "1"
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    time.sleep(0.1)
    names = {e.name for e in prof.events()}
    raw = getattr(prof.profiler, "kineto_results", None)                     # the raw activity records, when exposed
    if raw is not None:
        names |= {e.name() for e in raw.events()}
    return {normalize_kernel_name(s) for s in names if not s.startswith(("Memcpy", "Memset"))}


# ---- NumPy model of the device-side TX chains (commpy_b200/csrc/txlink.cu, turbolink.cu) ---------------------------
def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., Random123).  ctr: (N, 4) uint32 counters, key: (k0, k1).  Returns (N, 4) uint32."""
    c = np.asarray(ctr, dtype=np.uint64).copy()
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[:, 0]
        p1 = np.uint64(0xCD9E8D57) * c[:, 2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask
        c = np.stack([hi1 ^ c[:, 1] ^ np.uint64(k0), lo1, hi0 ^ c[:, 3] ^ np.uint64(k1), lo0], axis=1)
        k0 = (k0 + 0x9E3779B9) & 0xFFFFFFFF
        k1 = (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c.astype(np.uint32)


def _philox_words(frame, count, word, key):
    """Philox of the counters (f_lo, f_hi, 0 .. count-1, word) of global frame `frame`: (count, 4) uint32"""
    ctr = np.zeros((count, 4), dtype=np.uint64)
    ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3] = frame & 0xFFFFFFFF, frame >> 32, np.arange(count), word
    return philox4x32_10(ctr, key)


def philox_bits(frame, nbits, key):
    """The first `nbits` message bits of global frame `frame` (counter word 0, 128 bits per counter, LSB first)."""
    words = _philox_words(frame, -(-nbits // 128), 0, key).reshape(-1)
    return ((words[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1).reshape(-1)[:nbits]


def philox_normals(frame, count, word, key):
    """Counters 0 .. count-1 of `word` through float64 Box-Muller: (count, 2) complex standard normals, g.x + j g.y of the
    two Box-Mullers of each counter (commpy_b200/csrc/philox.cuh lists which word feeds which stream)."""
    r = _philox_words(frame, count, word, key).astype(np.float64)
    za = np.sqrt(-2 * np.log(r[:, 0] * 2.0 ** -32 + 2.0 ** -33)) * np.exp(2j * np.pi * r[:, 1] * 2.0 ** -32)
    zb = np.sqrt(-2 * np.log(r[:, 2] * 2.0 ** -32 + 2.0 ** -33)) * np.exp(2j * np.pi * r[:, 3] * 2.0 ** -32)
    return np.stack([za, zb], axis=1)


def same(a, b):
    """torch.equal, complex tensors compared through their real views"""
    import torch
    if a.is_complex():
        a, b = torch.view_as_real(a), torch.view_as_real(b)
    return torch.equal(a, b)


def conv_link_tx_model(trellis, modem, frames, frame_bits, seed, first_frame, noise_sigma, puncture=None):
    """(msg, y) exactly as cpb_conv_link_tx defines them (float64 Box-Muller for the noise)."""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    from commpy_b200.channelcoding.convcode import puncturing
    n, nb = int(trellis.n), int(modem.num_bits_symbol)
    ncoded = n * frame_bits
    nkept = ncoded if puncture is None else int(np.sum(np.asarray(puncture)[np.arange(ncoded) % len(puncture)] == 1))
    nsym = nkept // nb
    msg = np.zeros((frames, frame_bits), dtype=np.uint8)
    y = np.zeros((frames, nsym), dtype=np.complex128)
    cst = np.asarray(modem.constellation)
    for fl in range(frames):
        f = first_frame + fl
        bits = philox_bits(f, frame_bits, key)
        msg[fl] = bits
        coded = conv_encode(bits.astype(int), trellis, "cont")
        if puncture is not None:
            coded = puncturing(coded, puncture)
        idx = coded.reshape(-1, nb).dot(1 << np.arange(nb - 1, -1, -1))
        z = philox_normals(f, -(-nsym // 2), 1, key).reshape(-1)[:nsym]
        y[fl] = cst[idx] + noise_sigma * z
    return msg, y


def turbo_link_tx_model(trellis, interleaver, frames, frame_bits, seed, first_frame, noise_sigma):
    """(msg, sys, par1, par2) exactly as cpb_turbo_link_tx defines them: Philox message bits, the host turbo_encode mirror
    (commpy/channelcoding/turbo.py:14-59), BPSK 2x-1, float64 Box-Muller noise (stream j uses Philox counter word 2 + j)."""
    from commpy_b200.channelcoding import turbo_encode
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    N = frame_bits
    msg = np.zeros((frames, N), dtype=np.uint8)
    ys = np.zeros((frames, 3, N))
    for fl in range(frames):
        f = first_frame + fl
        bits = philox_bits(f, N, key)
        msg[fl] = bits
        streams = turbo_encode(bits.astype(int), trellis, trellis, interleaver)
        for j in range(3):
            z = philox_normals(f, -(-N // 4), 2 + j, key)
            z = np.stack([z.real, z.imag], axis=2).reshape(-1)[:N]
            ys[fl, j] = (2.0 * np.asarray(streams[j][:N], dtype=np.float64) - 1.0) + noise_sigma * z
    return msg, ys[:, 0], ys[:, 1], ys[:, 2]


# (noise variance, amplitude, prior std) of the "contradicted" MAP test frames: random +-amplitude symbols (not code words)
# plus noise and Gaussian priors.  Branch weights fall to 2^-19 .. 2^-40 per step, so 4-step blocks of map_lin2_kernel decay
# below its 2^-20 rescaling floor and take the per-step fallback, while every LLR below 40 stays representable in fp32.
CONTRADICTED_MAP_CASES = ((0.15, 1.0, 6.0), (0.3, 1.5, 8.0), (1.0, 1.0, 1.0))

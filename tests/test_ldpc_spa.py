"""Sum-product LDPC decoding ('SPA', commpy/channelcoding/ldpc.py:209-227, ldpc::cn_spa_kernel) against fp64.

References: the fp64 C oracle (oracle.ldpc_bp_decode(..., 'SPA', ..., return_iters=True)) and reference outputs stored in
tests/golden/ldpc_spa.npz (oracle/make_ldpc_spa_golden.py).  fp32 runs get float32 LLRs and the oracle gets those same
values as float64, so both start from identical check-node inputs.

The check node is ill-conditioned near saturation: R = 2 atanh(x), x = prod_k tanh(Q_k / 2), and
dR/dx = 2 / (1 - x^2) = 2 cosh^2(R/2).  Once 1 - |x| falls to a few units of 2^-53, x rounds to +-1 in double, atanh is
infinite and R is clipped to 500.  Two correct fp64 implementations that round differently may therefore send ~37 and 500
for the same edge, and after several iterations that one difference can change a whole frame.  So element-wise
assertions are made after ONE iteration, against the bound derived in `_one_iteration_bound`, and runs of many
iterations are compared only statistically (decisions and iteration counts of nearly every frame, frame error rates)."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import helpers
from oracle import oracle
from commpy_b200.channelcoding import ldpc_bp_decode_batch
from commpy_b200.channelcoding.ldpc import ldpc_bp_decode_batch_host
from test_dispatch_paths import _ran

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
EPS = 2.0 ** -53                                  # unit roundoff of double: the check node's arithmetic
UNIT = {"fp64": 2.0 ** -53, "fp32": 2.0 ** -24}   # unit roundoff of the message type: stored R, posterior sums
DTYPE = {"fp64": np.float64, "fp32": np.float32}
KNEE32, KNEE64 = 2 * np.arctanh(np.float64(1 - 2.0 ** -24)), 2 * np.arctanh(np.float64(1 - 2.0 ** -53))


# ---------------------------------------------------------------- fixtures
def _params(H):
    H = sp.csr_matrix(H)
    H.sort_indices()
    return {"n_vnodes": H.shape[1], "n_cnodes": H.shape[0], "parity_check_matrix": H.tocsc()}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLD, "ldpc_spa.npz"))


def _golden_H(g, tag):
    m, n = (int(v) for v in g[tag + "_shape"])
    return sp.csr_matrix((np.ones(len(g[tag + "_indices"]), np.int8), g[tag + "_indices"], g[tag + "_indptr"]),
                         shape=(m, n))


def _matrices():
    g = np.load(os.path.join(GOLD, "ldpc_spa.npz"))
    return {"g96": _golden_H(g, "g96"), "w960": _golden_H(g, "w960"),
            "mixed2_40": helpers.mixed_degree_H(list(range(2, 41)) * 4, 1200, seed=40)}


def _spread_llr(rs, batch, n):
    """All-zero code word; |LLR| log-uniform over [0.1, 80] (incoming messages on both sides of both saturation
    knees), a wrong sign with probability 1 / (1 + e^|LLR|)."""
    mag = np.exp(rs.uniform(np.log(0.1), np.log(80.0), (batch, n)))
    return np.where(rs.rand(batch, n) * (1.0 + np.exp(mag)) < 1.0, -mag, mag)


def _gpu(llr, params, iters, precision):
    x = np.ascontiguousarray(llr, dtype=DTYPE[precision])
    dec, out, it = ldpc_bp_decode_batch(x, params, iters, precision, return_iters=True, decoder_algorithm="SPA")
    return dec.cpu().numpy(), out.cpu().numpy().astype(np.float64), it.cpu().numpy()


def _oracle(llr64, params, iters):
    n = llr64.shape[1]
    d, o, it = oracle.ldpc_bp_decode(np.ascontiguousarray(llr64, np.float64).reshape(-1).copy(), params, "SPA", iters,
                                     return_iters=True, threads=8)
    return d.reshape(n, -1).T, o.reshape(n, -1).T, it


# ---------------------------------------------------------------- the one-iteration bound
def _one_iteration_bound(llr64, H, precision):
    """Per-element bound on |out_gpu - out_oracle| after one iteration, and the mask of variables with an edge where
    either a finite message or the +-500 clip is a correct result.

    Both decoders see the same Q = LLR.  Per edge e of a row of degree d, x_e = prod_{k != e} t_k, t_k = tanh(Q_k / 2):
      * the kernel forms it in double from d tanh values (<= 1 ulp = 2 EPS relative each), d - 1 products, one
        division and one product (EPS each): relative error <= (3 d + 3) EPS;
      * the oracle forms exp2(sum_k log2 |t_k|): the tanh errors pass through unchanged (2 d EPS), each log2 adds
        2 EPS |log2 t_k| absolute in the exponent, the sum adds at most d EPS sum_k |log2 t_k|, and exp2 multiplies the
        exponent error by ln 2 and adds 2 EPS, plus 4 EPS for its own 1/t_e and product;
    so |x_gpu - x_oracle| <= rho |x| with rho = (5 d + 9 + (d + 2) L) EPS, L = sum_k |log2 |t_k||.  The message error
    is then dR_e = 2 atanh(|x|(1 + rho)) - 2 atanh(|x|) ~ 2 rho |x| cosh^2(R_e/2): the conditioning term.  An edge whose
    |x|(1 + rho) reaches 1 may come out as any value from its finite message up to the 500 clip: "either value".
    The posterior is llr + sum_e R_e in ascending check order in the message type: storing each R (fp32) and the
    d_v + 1 additions add at most (d_v + 2) u (|llr| + sum_e |R_e|), u = 2^-53 (fp64) or 2^-24 (fp32).  So
        |dout| <= a + r S + sum_e dR_e,   a = 0,  r = (d_v + 2) u,  S = |llr| + sum_e |R_e|,
    with S in place of |out| because the messages of a variable may cancel."""
    H = sp.csr_matrix(H)
    H.sort_indices()
    rows = np.repeat(np.arange(H.shape[0]), np.diff(H.indptr))
    cols = H.indices
    deg = np.diff(H.indptr)[rows].astype(np.float64)
    dv = np.bincount(cols, minlength=H.shape[1]).astype(np.float64)
    Q = np.clip(llr64, -500, 500)[:, cols]                                   # (frames, edges)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.tanh(0.5 * Q)
        lg = np.where(t == 0, 0.0, np.abs(np.log2(np.abs(t))))        # an exact zero makes its own edge NaN, the others 0
        Lsum = np.add.reduceat(lg, H.indptr[:-1], axis=1)[:, rows]
        prod = np.multiply.reduceat(t, H.indptr[:-1], axis=1)[:, rows]
        x = np.abs(prod / t)
        rho = (5 * deg + 9 + (deg + 2) * Lsum) * EPS
        R = np.minimum(2 * np.arctanh(np.minimum(x, 1.0)), 500.0)
        hi = x * (1 + rho)
        either = hi >= 1.0
        dR = np.where(either, 500.0 - np.minimum(2 * np.arctanh(np.minimum(x * (1 - rho), 1.0)), 500.0),
                      2 * np.arctanh(np.minimum(hi, 1.0)) - 2 * np.arctanh(x))
    n = H.shape[1]
    frames = llr64.shape[0]
    sum_dR = np.zeros((frames, n))
    S = np.abs(np.clip(llr64, -500, 500))
    any_either = np.zeros((frames, n), bool)
    for j_e in range(len(cols)):                                             # scatter edges onto their variables
        sum_dR[:, cols[j_e]] += dR[:, j_e]
        S[:, cols[j_e]] += np.abs(R[:, j_e])
        any_either[:, cols[j_e]] |= either[:, j_e]
    bound = (dv + 2) * UNIT[precision] * S + sum_dR
    return bound, any_either


def _assert_one_iteration(llr, H, params, precision, got=None):
    """One iteration of `precision` against the oracle: out_llrs element-wise within `_one_iteration_bound`, iteration
    counts exact, decisions exact wherever the bound does not reach across zero."""
    llr = np.ascontiguousarray(llr, dtype=DTYPE[precision])
    llr64 = llr.astype(np.float64)
    d_o, o_o, it_o = _oracle(llr64, params, 1)
    dec, out, it = _gpu(llr, params, 1, precision) if got is None else got
    bound, _ = _one_iteration_bound(llr64, H, precision)
    bound[it_o == 0] = 0.0                         # syndrome met before the first iteration: out_llrs = the clipped LLRs
    err = np.abs(out - o_o)
    bad = ~(err <= bound)
    assert not bad.any(), ("out_llrs outside the conditioning bound", int(bad.sum()),
                           [(int(f), int(j), float(out[f, j]), float(o_o[f, j]), float(bound[f, j]))
                            for f, j in zip(*np.nonzero(bad))][:8])
    assert np.array_equal(it, it_o)
    sure = np.abs(o_o) > bound
    assert (~sure).sum() <= 1 + 0.001 * sure.size, int((~sure).sum())
    assert np.array_equal(dec[sure], d_o[sure]), int((dec[sure] != d_o[sure]).sum())
    return dec, out, it


# ---------------------------------------------------------------- single-message probe
def _probe_case(precision):
    """One row per degree d in {2, 3, 7, 15, 32}, every column of degree 1.  Column 0 of a row is the probe (LLR 0.25);
    the other d - 1 LLRs share one magnitude s, swept from 5 to 60 over the frames, and one of them is negative, so the
    check fails and one iteration runs.  Then out - llr at the probe is R = -2 atanh(tanh(s/2)^(d-1))."""
    degs = (2, 3, 7, 15, 32)
    starts = np.concatenate([[0], np.cumsum(degs)])
    H = sp.csr_matrix((np.ones(starts[-1], np.int8), np.arange(starts[-1]), starts), shape=(len(degs), starts[-1]))
    s = np.linspace(5.0, 60.0, 4096)
    llr = np.repeat(s[:, None], starts[-1], axis=1)
    llr[:, starts[:-1]] = 0.25
    llr[:, starts[:-1] + 1] *= -1.0
    return degs, starts, H, s, np.ascontiguousarray(llr, DTYPE[precision])


@pytest.mark.parametrize("precision", ["fp32", "fp64"])
def test_spa_single_message_probe(precision):
    degs, starts, H, s, llr = _probe_case(precision)
    params = _params(H)
    dec, out, it = _gpu(llr, params, 1, precision)
    assert (it == 1).all()
    R = out[:, starts[:-1]] - llr[:, starts[:-1]].astype(np.float64)     # exact in double: both are values of T
    # fp64 formula and its conditioning (see _one_iteration_bound): x = tanh(s/2)^(d-1)
    for i, d in enumerate(degs):
        t = np.tanh(llr[:, starts[i] + 2 if d > 2 else starts[i] + 1].astype(np.float64) * 0.5)
        x = np.abs(t) ** (d - 1)
        want = -np.minimum(2 * np.arctanh(np.minimum(x, 1.0)), 500.0)
        rho = (5 * d + 9) * EPS + 4 * EPS
        hi = np.minimum(x * (1 + rho), 1.0)
        tol = 2 * np.arctanh(hi) - 2 * np.arctanh(np.minimum(x, 1.0)) + 2 * UNIT[precision] * (np.abs(want) + 0.25)
        either = x * (1 + rho) >= 1.0                 # any value from the finite message up to the clip is correct
        lo = 2 * np.arctanh(np.minimum(x * (1 - rho), 1.0)) - 2 * UNIT[precision] * (np.abs(want) + 0.25)
        ok = np.where(either, -R[:, i] >= lo, np.abs(R[:, i] - want) <= tol)
        assert ok.all(), (precision, d, [(float(s[f]), float(R[f, i]), float(want[f])) for f in np.nonzero(~ok)[0][:6]])
        # 500 only where the fp64 formula itself saturates (or is within its rounding of doing so)
        sat = R[:, i] == -500.0
        assert not (sat & ~either & (want != -500.0)).any(), (precision, d, float(s[sat & ~either][0]))
    # an fp32 message reaches the values between the fp32 knee (~17.3) and the fp64 knee (~37.4)
    mid = (np.abs(R) > KNEE32 + 0.5) & (np.abs(R) < KNEE64 - 0.5)
    assert mid.sum() > 1000, int(mid.sum())


def test_spa_probe_fp32_saturates_where_fp64_does():
    """fp32 and fp64 see the same Q in the first iteration and the check node computes in double for both, so the
    messages are the same double rounded to float: +-500 at exactly the same frames."""
    degs, starts, H, s, llr32 = _probe_case("fp32")
    params = _params(H)
    _, o32, _ = _gpu(llr32, params, 1, "fp32")
    _, o64, _ = _gpu(llr32.astype(np.float64), params, 1, "fp64")
    p = starts[:-1]
    R32 = o32[:, p] - llr32[:, p].astype(np.float64)
    R64 = o64[:, p] - llr32[:, p].astype(np.float64)
    assert np.array_equal(R32 == -500.0, R64 == -500.0), [(d, float(s[(R32[:, i] == -500) != (R64[:, i] == -500)][0]))
                                                          for i, d in enumerate(degs)
                                                          if ((R32[:, i] == -500) != (R64[:, i] == -500)).any()]


# ---------------------------------------------------------------- one full iteration at scale
@pytest.mark.parametrize("precision", ["fp32", "fp64"])
@pytest.mark.parametrize("code", ["g96", "w960", "mixed2_40"])
def test_spa_one_iteration_vs_oracle(code, precision):
    H = _matrices()[code]
    params = _params(H)
    rs = np.random.RandomState({"g96": 1, "w960": 2, "mixed2_40": 3}[code])
    batch = {"g96": 4096, "w960": 2048, "mixed2_40": 2048}[code]
    llr = _spread_llr(rs, batch, H.shape[1])
    llr[rs.rand(*llr.shape) < 0.01] *= 40.0                                  # some beyond the +-500 clip
    dec, out, it = _assert_one_iteration(llr, H, params, precision)
    assert (it == 1).mean() > 0.5
    Q = np.abs(np.clip(llr, -500, 500))
    assert ((Q > KNEE32) & (Q < KNEE64)).any() and (Q > KNEE64).any()


# ---------------------------------------------------------------- dispatch paths
@pytest.mark.parametrize("precision", ["fp32", "fp64"])
def test_spa_batch_sizes_and_kernels(precision):
    """Batches of 1, 3, 31, 32, 33 and 4,097 frames (padding to 32 frames; vectors of 4 floats or 2 doubles): one
    iteration against the oracle, and eight iterations bit for bit equal to the same frames inside the 4,097 batch.
    cn_spa_kernel and vn_spa_kernel run; neither the min-sum check pass nor the min-sum variable pass does."""
    H = _matrices()["g96"]
    params = _params(H)
    rs = np.random.RandomState(5)
    llr = np.ascontiguousarray(_spread_llr(rs, 4097, 96), DTYPE[precision])
    T = "double" if precision == "fp64" else "float"
    full = _ran(lambda: _gpu(llr, params, 8, precision), ["ldpc::cn_spa_kernel<%s>" % T, "ldpc::vn_spa_kernel<%s>" % T],
                ["cn_bulk_kernel", "ldpc::cn_kernel<", "ldpc::vn_kernel<"])
    for b in (1, 3, 31, 32, 33, 4097):
        _assert_one_iteration(llr[:b], H, params, precision)
        got = _gpu(llr[:b], params, 8, precision)
        assert np.array_equal(got[0], full[0][:b]) and np.array_equal(got[2], full[2][:b])
        assert np.array_equal(got[1].view(np.uint64), full[1][:b].view(np.uint64))


def test_spa_frozen_frames_iteration_counts():
    """Frames that meet the syndrome before the first iteration (a clean code word) next to frames that need several
    iterations: the converged ones freeze (done / act) while the others go on; iteration counts equal the oracle's."""
    H = _matrices()["w960"]
    params = _params(H)
    rs = np.random.RandomState(6)
    batch = 512
    sigma = 1.0 / np.sqrt(2 * 0.75 * 10 ** (np.linspace(2.5, 5.0, batch) / 10))[:, None]
    llr = 2.0 * (1.0 + sigma * rs.randn(batch, 960)) / sigma ** 2
    llr[::4] = np.abs(llr[::4])                                             # every fourth frame: no error at all
    d_o, _, it_o = _oracle(llr, params, 30)
    assert (it_o == 0).sum() == batch // 4 and (it_o >= 3).sum() > batch // 4 and (it_o == 30).sum() < batch // 8
    for precision in ("fp64", "fp32"):
        dec, _, it = _gpu(llr, params, 30, precision)
        same = (it == it_o) & (dec == d_o).all(axis=1)
        assert same.mean() >= 0.995, (precision, np.nonzero(~same)[0].tolist()[:10])
        assert np.array_equal(it[::4], it_o[::4])


@pytest.mark.parametrize("precision", ["fp32", "fp64"])
def test_spa_host_pipeline_across_chunks(precision):
    """cpb_ldpc_decode_host with algorithm 1 (SPA), 1,000 frames of WiMax 960: chunks of 128 and a ragged 104.
    Decisions, out_llrs and iterations equal the device call bit for bit."""
    H = _matrices()["w960"]
    params = _params(H)
    rs = np.random.RandomState(7)
    llr = _spread_llr(rs, 1000, 960)
    llr[::7, ::5] *= 40.0
    x = np.ascontiguousarray(llr, DTYPE[precision])
    x0 = x.copy()
    T = "double" if precision == "fp64" else "float"
    dh, oh, ih = _ran(lambda: ldpc_bp_decode_batch_host(x, params, 6, precision, return_iters=True,
                                                        decoder_algorithm="SPA"), "ldpc::cn_spa_kernel<%s>" % T,
                      "cn_bulk_kernel")
    assert np.array_equal(x, np.clip(x0, -500, 500))
    dd, od, idd = (t.cpu().numpy() for t in ldpc_bp_decode_batch(x0.copy(), params, 6, precision, return_iters=True,
                                                                  decoder_algorithm="SPA"))
    assert np.array_equal(dh, dd) and np.array_equal(ih, idd)
    assert np.array_equal(oh.view(np.uint8), od.view(np.uint8))


# ---------------------------------------------------------------- reference goldens
def _golden_case(g, code, case, K):
    """(decisions, iteration counts, NaN mask of out_llrs) of the reference after K iterations, unpacked."""
    pre = "%s_%s_it%d_" % (code, case, K)
    n = int(g[code + "_shape"][1])
    return (np.unpackbits(g[pre + "dec"], axis=1, count=n), g[pre + "iters"],
            np.unpackbits(g[pre + "nan"], axis=1, count=n).astype(bool))


@pytest.mark.parametrize("code", ["g96", "w960"])
@pytest.mark.parametrize("case", ["spread", "big", "zero"])
def test_spa_reference_golden(golden, code, case):
    """fp64 against the reference's own outputs.  1, 2 and 20 iterations: decisions and iteration counts equal on every
    frame, NaN exactly where the reference has NaN.  One iteration: out_llrs within the conditioning bound, of the
    reference's out_llrs on the zero set and of the oracle's on the others.  Zero LLRs make NaN messages; the
    reference's decision of such a NaN is its sign bit (set for the NaN of (1/0) * 0 on x86), which the kernels
    reproduce."""
    H = _golden_H(golden, code)
    params = _params(H)
    llr = golden["%s_%s_llr" % (code, case)].astype(np.float64)
    for K in (1, 2, 20):
        dec, out, it = _gpu(llr, params, K, "fp64")
        d_ref, it_ref, nan_ref = _golden_case(golden, code, case, K)
        print(code, case, K, "frames with other iteration counts:", np.nonzero(it != it_ref)[0].tolist(),
              "other decisions:", np.nonzero((dec != d_ref).any(axis=1))[0].tolist())
        assert np.array_equal(dec, d_ref), K
        assert np.array_equal(it, it_ref), K
        assert np.array_equal(np.isnan(out), nan_ref), K
    if case == "zero":
        dec, out, it = _gpu(llr, params, 1, "fp64")
        ref = golden["%s_zero_it1_out" % code]
        assert np.isnan(ref).any() and np.array_equal(np.isnan(out), np.isnan(ref))
        bound, _ = _one_iteration_bound(llr, H, "fp64")
        bound[it == 0] = 0.0
        fin = ~np.isnan(ref)
        assert (np.abs(out - ref)[fin] <= bound[fin]).all()
    else:
        _assert_one_iteration(llr, H, params, "fp64")


def test_spa_zero_llrs_fp32_decisions(golden):
    """fp32 on the frames with +0.0 / -0.0 LLRs: NaN where the reference has NaN, with the reference's decision."""
    for code in ("g96", "w960"):
        H = _golden_H(golden, code)
        llr = golden["%s_zero_llr" % code].astype(np.float32)
        dec, out, it = _gpu(llr, _params(H), 1, "fp32")
        d_ref, it_ref, nan = _golden_case(golden, code, "zero", 1)
        assert nan.any() and np.array_equal(np.isnan(out), nan)
        assert np.array_equal(it, it_ref)
        assert np.array_equal(dec[nan], d_ref[nan])


# ---------------------------------------------------------------- many iterations: statistics only
def test_spa_many_iterations_statistics():
    """8,192 Gallager frames at 1.5, 2.0 and 2.5 dB, 50 iterations.  At least 99.5 % of the frames have the oracle's
    decisions and iteration count, in fp64 and in fp32; fp32 FER equals fp64 FER within 3 standard errors."""
    H = _matrices()["g96"]
    params = _params(H)
    rs = np.random.RandomState(8)
    N = 8192
    for ebno in (1.5, 2.0, 2.5):
        sigma = 1 / np.sqrt(10 ** (ebno / 10.0) * 0.5 * 2)
        llr = (2.0 * (1.0 + sigma * rs.randn(N, 96)) / sigma ** 2).astype(np.float32).astype(np.float64)
        d_o, _, it_o = _oracle(llr, params, 50)
        fer = {}
        for precision in ("fp64", "fp32"):
            dec, _, it = _gpu(llr, params, 50, precision)
            same = (it == it_o) & (dec == d_o).all(axis=1)
            if not same.all():
                print("SPA %s at %.1f dB: %d frames differ from the oracle: %s" % (
                    precision, ebno, int((~same).sum()), np.nonzero(~same)[0].tolist()[:20]))
            assert same.mean() >= 0.995, (precision, ebno, same.mean())
            fer[precision] = float((dec.sum(axis=1) > 0).mean())
        p = fer["fp64"]
        se = np.sqrt(max(p * (1 - p), 1.0 / N) / N)
        assert abs(fer["fp32"] - p) <= 3 * se, (ebno, fer)

"""CPU: the NumPy GF(2) model of the LDPC encoder plan (tests/model_ldpc_encode.py) against the facts that decide how each
code is encoded, and against the plan the library builds (cpb_ldpc_encoder_plan runs on the host; no device is used).
The reference's design files enter as the parity-check matrices stored in tests/golden/ldpc_link_ber.npz."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import helpers
import model_ldpc_encode as mle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CODES = ("96_3_963", "96_33_964", "1440_720", "960_720_a")


def design_H(name):
    g = np.load(os.path.join(GOLD, "ldpc_link_ber.npz"))
    r, c, shape = g["H_%s_rows" % name], g["H_%s_cols" % name], tuple(g["H_%s_shape" % name])
    H = sp.csr_matrix((np.ones(len(r), np.int8), (r, c)), shape=shape)
    H.sort_indices()
    return H


def small_staircase(n=720, m=360, seed=5):
    k = n - m
    return helpers.dvbs2_like_H(seed=seed, n=n, m=m, n8=k * 2 // 5, n3=k - k * 2 // 5)


def mirror_encodings_valid(H, count=50, seed=0):
    """how many of `count` random messages the host mirror of triang_ldpc_systematic_encode (the reference's real-valued
    generator) turns into code words"""
    import warnings
    from commpy_b200.channelcoding import triang_ldpc_systematic_encode
    m, n = H.shape
    params = {"parity_check_matrix": H.tocsc(), "n_cnodes": m, "n_vnodes": n}
    rs = np.random.RandomState(seed)
    ok = 0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for _ in range(count):
            cw = triang_ldpc_systematic_encode(rs.randint(0, 2, n - m), params, False).astype(np.int64)
            ok += int(not ((H @ cw) % 2).any())
    return ok


def test_model_reproduces_the_code_table():
    """GF(2) ranks, peeling and the validity of the reference's generator encoding (through the host mirror), per code:
    96.3.963 has a singular H_p (rank 45 of 48, H rank 46); 96.33.964 an invertible one, but its real-valued generator
    encodes no message to a code word; both WiMax codes are invertible, encode validly and do not peel; the DVB-S2-shaped
    staircase peels completely."""
    want = {"96_3_963": (45, 46, 0), "96_33_964": (48, None, 0), "1440_720": (720, None, 50), "960_720_a": (240, None, 50)}
    for name in CODES:
        H = design_H(name)
        m, n = H.shape
        Hd = np.asarray(H.todense())
        rank_p, rank_h, valid = want[name]
        assert mle.gf2_rank(Hd[:, n - m:]) == rank_p, name
        if rank_h is not None:
            assert mle.gf2_rank(Hd) == rank_h, name
        assert mle.peel(H) is None, name
        assert mirror_encodings_valid(H) == valid, name
    order, pivot = mle.peel(helpers.dvbs2_like_H())
    assert np.array_equal(order, np.arange(32400)) and np.array_equal(pivot, np.arange(32400))


def test_model_encodings_are_code_words_and_equal_the_reference():
    g = np.load(os.path.join(GOLD, "ldpc_link_ber.npz"))
    rs = np.random.RandomState(1)
    for name in ("96_33_964", "1440_720", "960_720_a"):
        H = design_H(name)
        m, n = H.shape
        msg = rs.randint(0, 2, (7, n - m))
        cw = mle.encode(H, msg)
        assert not ((H @ cw.T.astype(np.int64)) % 2).any(), name
    for name in ("1440_720", "960_720_a"):
        msg, want = g["wimax_%s_msg" % name], g["wimax_%s_cw" % name]
        assert np.array_equal(mle.encode(design_H(name), msg), want), name
    H = small_staircase()
    msg = rs.randint(0, 2, (9, 360))
    a, b = mle.encode(H, msg), mle.encode(H, msg, force_dense=True)
    assert np.array_equal(a, b) and not ((H @ a.T.astype(np.int64)) % 2).any()


@pytest.mark.parametrize("n,m,seed", [(720, 360, 5), (96, 48, 1), (200, 100, 2)])
def test_library_plan_equals_model_on_staircase_codes(n, m, seed):
    """Same peel order and pivots, and with the dense form forced the same P, as the model."""
    H = small_staircase(n, m, seed)
    form, order, pivot, _ = mle.library_plan(H)
    mform, morder, mpivot, _ = mle.plan(H)
    assert form == mform == mle.PEELED
    assert np.array_equal(order, morder) and np.array_equal(pivot, mpivot)
    form, _, _, P = mle.library_plan(H, force_dense=True)
    assert form == mle.DENSE and np.array_equal(P, mle.plan(H, force_dense=True)[3])


def test_library_plan_on_design_codes_and_bounds():
    """WiMax codes: dense form with the model's P; 96.3.963: ValueError (singular H_p); the full-size DVB-S2-shaped code
    peels even when the dense form is asked for (it exceeds the bound); a code that neither peels nor fits the bound:
    NotImplementedError."""
    for name in ("1440_720", "960_720_a", "96_33_964"):
        H = design_H(name)
        form, _, _, P = mle.library_plan(H)
        assert form == mle.DENSE and np.array_equal(P, mle.dense_P(H)), name
    with pytest.raises(ValueError):
        mle.library_plan(design_H("96_3_963"))
    with pytest.raises(ValueError):
        mle.plan(design_H("96_3_963"))
    form, order, pivot, _ = mle.library_plan(helpers.dvbs2_like_H(), force_dense=True)
    assert form == mle.PEELED and np.array_equal(order, np.arange(32400)) and np.array_equal(pivot, np.arange(32400))
    big = helpers.mixed_degree_H([6] * 9000, 18000, seed=4)        # random rows: k m = 8.1e7 > 2^26
    assert mle.peel(big) is None
    with pytest.raises(NotImplementedError):
        mle.library_plan(big)
    with pytest.raises(NotImplementedError):
        mle.plan(big)

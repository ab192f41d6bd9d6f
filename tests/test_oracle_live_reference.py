"""CPU: the oracle (oracle/commpy_oracle.c) and the host-side MIMO mirrors against outputs of the UNMODIFIED reference on
cases drawn from several fixed seeds (tests/golden/live_reference.npz, written by oracle/make_live_golden.py): bit-exact for
Viterbi, LDPC min-sum incl. out_llrs and the hard demapper, 1e-9 for the float outputs."""
import os

import numpy as np
import pytest
import scipy.sparse as sp

import helpers
from oracle import oracle

pytestmark = pytest.mark.filterwarnings("ignore")

GOLD = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "live_reference.npz"))
TAGS = ["s%d" % s for s in GOLD["seeds"]]


def test_viterbi_and_bcjr_fresh_cases():
    """Viterbi (every mode and termination) and BCJR with a prior on the stored cases of every seed.  ("fresh": cases other
    than those of tests/golden/viterbi.npz and bcjr_turbo.npz; they come from fixed seeds, not from each run.)"""
    for tag in TAGS:
        _viterbi_and_bcjr(GOLD, tag)


def _viterbi_and_bcjr(g, tag):
    k7 = helpers.k7()
    for mode in ("hard", "soft", "unquantized"):
        for term in ("cont", "term"):
            key = "%s_vit_%s_%s" % (tag, mode, term)
            tb = int(g[key + "_tb"]) or None
            assert np.array_equal(g[key + "_ref"], oracle.viterbi_decode(g[key + "_x"].copy(), k7, tb, mode)), key
    got = oracle.map_decode(g[tag + "_map_sys"], g[tag + "_map_par"], helpers.rsc_k4(), float(g[tag + "_map_s2"]),
                            g[tag + "_map_La"], "decode")
    assert np.allclose(g[tag + "_map_L"], got[0], rtol=1e-9, atol=1e-9) and np.array_equal(g[tag + "_map_bits"], got[1]), tag


def test_ldpc_and_demapper_fresh_cases():
    """LDPC min-sum on the gallager 96.33.964 design and the 16-QAM demapper on the stored cases of every seed (fixed seeds)"""
    for tag in TAGS:
        _ldpc_and_demapper(GOLD, tag)


def _ldpc_and_demapper(g, tag):
    from commpy_b200.modulation import QAMModem
    m, n = (int(v) for v in g["ldpc_H_shape"])
    H = sp.csr_matrix((np.ones(len(g["ldpc_H_indices"]), np.int8), g["ldpc_H_indices"], g["ldpc_H_indptr"]), shape=(m, n))
    params = {"n_vnodes": n, "parity_check_matrix": H}
    dec, out = oracle.ldpc_bp_decode(g[tag + "_ldpc_llr"].copy(), params, "MSA", 6)
    assert np.array_equal(g[tag + "_ldpc_dec"], dec) and np.array_equal(g[tag + "_ldpc_out"], out), tag
    modem = QAMModem(16)
    y = g[tag + "_demap_y"]
    want = g[tag + "_demap_soft"]
    got = oracle.demodulate(modem, y, "soft", 0.7)
    fin = np.isfinite(want)
    assert np.allclose(want[fin], got[fin], rtol=1e-9, atol=1e-9), tag
    assert np.array_equal(g[tag + "_demap_hard"], oracle.demodulate(modem, y, "hard")), tag


def test_mimo_mirrors_fresh_cases():
    """host-side MIMO mirrors (kbest, best_first_detector, idd_decoder) against the reference's outputs on the stored cases
    of every seed (fixed seeds)"""
    for tag in TAGS:
        _mimo_mirrors(GOLD, tag)


def _mimo_mirrors(g, tag):
    from commpy_b200 import modulation as mod
    from commpy_b200.links import idd_decoder
    for m, n in ((4, 2), (16, 3), (16, 4)):
        mq = mod.QAMModem(m)

        def demode(s):
            return oracle.demodulate(mq, s, "hard")
        key = "%s_mimo_q%d_n%d" % (tag, m, n)
        for c in range(len(g[key + "_y"])):
            y, h, nv = g[key + "_y"][c], g[key + "_h"][c], float(g[key + "_nv"][c])
            stack = tuple(int(s) for s in g[key + "_stack"][c])
            msg = "%s case %d" % (key, c)
            np.testing.assert_allclose(mod.kbest(y, h, mq.constellation, 6), g[key + "_kbest_hard"][c], atol=1e-12, err_msg=msg)
            np.testing.assert_allclose(mod.kbest(y, h, mq.constellation, 6, nv, "soft", demode), g[key + "_kbest_soft"][c],
                                       rtol=1e-9, atol=1e-9, err_msg=msg)
            np.testing.assert_allclose(mod.best_first_detector(y, h, mq.constellation, stack, nv, demode, 100),
                                       g[key + "_best_first"][c], rtol=1e-9, atol=1e-9, err_msg=msg)
    # idd_decoder: the reference's closures, with the mirrors' kbest, 3 iterations
    mq = mod.QAMModem(16)

    def detector(y, h, constellation, noise_var, a_priori):
        return mod.kbest(y, h, constellation, 8, noise_var, "soft", lambda s: oracle.demodulate(mq, s, "hard")) + 0.25 * a_priori

    def decoder(llr):
        return np.tanh(llr) * 3 + np.roll(llr, 1)

    def decision(llr):
        return (llr > 0).astype(int)
    n = 2
    got = idd_decoder(detector, decoder, decision, 3)(g[tag + "_idd_y"], g[tag + "_idd_h"], mq.constellation, 0.02,
                                                     g[tag + "_idd_ap"].copy(), n * 4)
    np.testing.assert_array_equal(got, g[tag + "_idd_ref"])

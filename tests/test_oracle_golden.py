"""CPU: the oracle (oracle/commpy_oracle.c) against the golden vectors generated from the UNMODIFIED reference
by oracle/validate_against_reference.py.  This is what pins the oracle without the reference checkout."""
import os

import numpy as np
import pytest

from oracle import oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class _T:
    """Trellis stand-in built from the golden tables."""

    def __init__(self, tabs, name):
        self.next_state_table = tabs[name + "_next"]
        self.output_table = tabs[name + "_out"]
        self.number_states, self.number_inputs = self.next_state_table.shape
        self.k = int(np.log2(self.number_inputs))
        self.n = int(np.ceil(np.log2(self.output_table.max() + 1)))
        self.total_memory = int(np.log2(self.number_states))


def golden_trellis(name):
    tabs = np.load(os.path.join(GOLD, "trellis_tables.npz"))
    t = _T(tabs, name)
    t.n = {"t57": 2, "rsc_legacy": 2, "r23": 3, "r23_lsb": 3, "r23_rsc": 3, "k7": 2, "k7_wifi_quirk": 2, "rsc_k4": 2}[name]
    return t


def test_viterbi_golden_bit_exact():
    g = np.load(os.path.join(GOLD, "viterbi.npz"))
    ncase = len([k for k in g.files if k.endswith("_meta")])
    assert ncase >= 100
    for c in range(ncase):
        name, mode, term, tb = g["c%03d_meta" % c]
        tb = None if tb == "None" else int(tb)
        out = oracle.viterbi_decode(g["c%03d_x" % c], golden_trellis(str(name)), tb, str(mode))
        assert np.array_equal(out, g["c%03d_ref" % c]), (c, name, mode, term, tb)


def test_map_and_turbo_golden():
    g = np.load(os.path.join(GOLD, "bcjr_turbo.npz"))
    for c in range(9):
        name, s2 = g["m%02d_meta" % c]
        L, bits = oracle.map_decode(g["m%02d_sys" % c], g["m%02d_par" % c], golden_trellis(str(name)), float(s2),
                                    g["m%02d_La" % c], "decode")
        assert np.allclose(L, g["m%02d_L" % c], rtol=1e-9, atol=1e-9)
        assert np.array_equal(bits, g["m%02d_bits" % c])

    class IL:
        pass
    for c in range(3):
        s2, iters = g["t%02d_meta" % c]
        il = IL()
        il.p_array = g["t%02d_perm" % c]
        bits = oracle.turbo_decode(g["t%02d_sys" % c], g["t%02d_p1" % c], g["t%02d_p2" % c], golden_trellis("rsc_k4"),
                                   float(s2), int(iters), il)
        assert np.array_equal(bits, g["t%02d_bits" % c])


def test_ldpc_golden_exact():
    import scipy.sparse as sp
    g = np.load(os.path.join(GOLD, "ldpc.npz"))
    for c in range(5):
        rel, nblk, iters, m, n = g["l%02d_meta" % c]
        indptr, indices = g["l%02d_indptr" % c], g["l%02d_indices" % c]
        H = sp.csr_matrix((np.ones(len(indices), np.int8), indices, indptr), shape=(int(m), int(n)))
        llr = g["l%02d_llr" % c].copy()
        dec, out = oracle.ldpc_bp_decode(llr, {"n_vnodes": int(n), "parity_check_matrix": H}, "MSA", int(iters))
        assert np.array_equal(dec, g["l%02d_dec" % c]), rel
        assert np.array_equal(out, g["l%02d_out" % c]), rel
        assert np.abs(llr).max() <= 500.0          # clipped in place


def test_demod_golden():
    g = np.load(os.path.join(GOLD, "demod.npz"))

    class M:
        pass
    for c in range(24):
        name, nv = g["d%02d_meta" % c]
        md = M()
        md.constellation = g[str(name) + "_constellation"]
        ref = g["d%02d_llr" % c]
        out = oracle.demodulate(md, g["d%02d_y" % c], "soft", float(nv))
        fin = np.isfinite(ref)
        assert np.allclose(out[fin], ref[fin], rtol=1e-9, atol=1e-9), name
        assert np.array_equal(oracle.demodulate(md, g["d%02d_y" % c], "hard"), g["d%02d_hard" % c])


def test_oracle_threads_agree():
    t = golden_trellis("k7")
    rs = np.random.RandomState(3)
    x = rs.randint(0, 2, (16, 400)).astype(float)
    a = oracle.viterbi_decode_batch(x, t, None, "hard", threads=1)
    b = oracle.viterbi_decode_batch(x, t, None, "hard", threads=4)
    assert np.array_equal(a, b)


def test_ldpc_spa_golden():
    import scipy.sparse as sp
    g = np.load(os.path.join(GOLD, "ldpc.npz"))
    for c in range(3):
        rel, nblk, iters, m, n = g["s%02d_meta" % c]
        H = sp.csr_matrix((np.ones(len(g["s%02d_indices" % c]), np.int8), g["s%02d_indices" % c], g["s%02d_indptr" % c]),
                          shape=(int(m), int(n)))
        dec, out = oracle.ldpc_bp_decode(g["s%02d_llr" % c].copy(), {"n_vnodes": int(n), "parity_check_matrix": H}, "SPA",
                                         int(iters))
        assert np.array_equal(dec, g["s%02d_dec" % c]), rel
        assert np.allclose(out, g["s%02d_out" % c], rtol=1e-9, atol=1e-9), rel

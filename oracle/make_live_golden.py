"""Outputs of the UNMODIFIED reference on the cases of tests/test_oracle_live_reference.py (Viterbi in every mode and
termination, BCJR with a prior, LDPC min-sum on the reference's gallager 96.33.964 design, the QAM demapper, the MIMO
detectors and idd_decoder), drawn from a few fixed seeds and replayed by that test against the oracle and the host-side
mirrors.

    python oracle/make_live_golden.py            # writes tests/golden/live_reference.npz (seconds)
TEST INFRASTRUCTURE ONLY."""
import os
import sys
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path = [p for p in sys.path if os.path.abspath(p or ".") != HERE]
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np

import refimport

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
SEEDS = (11, 12, 13, 14)


def viterbi_bcjr(rcc, rs, out, tag):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        k7 = rcc.Trellis(np.array([6]), np.array([[0o133, 0o171]]))
        rsc = rcc.Trellis(np.array([3]), np.array([[1, 0o15]]), np.array([[0o13]]), "rsc")
    for mode in ("hard", "soft", "unquantized"):
        for term, tb in (("cont", None), ("term", 9)):
            msg = rs.randint(0, 2, 48)
            c = rcc.conv_encode(msg, k7, term).astype(float)
            if mode == "hard":
                x = np.abs(c - (rs.rand(len(c)) < 0.1))
            elif mode == "soft":
                x = (2 * c - 1) * 2 + rs.randn(len(c)) * 2.5
            else:
                x = (2 * c - 1) + rs.randn(len(c))
            key = "%s_vit_%s_%s" % (tag, mode, term)
            out[key + "_x"] = x
            out[key + "_tb"] = np.array(tb or 0)
            out[key + "_ref"] = rcc.viterbi_decode(x.copy(), k7, tb, mode)
    N, s2 = 40, 0.9
    sys_, par, la = (-1 + np.sqrt(s2) * rs.randn(N) for _ in range(3))
    with np.errstate(all="ignore"):
        L, bits = rcc.map_decode(sys_, par, rsc, s2, 0.2 * la, "decode")
    out.update({tag + "_map_sys": sys_, tag + "_map_par": par, tag + "_map_La": 0.2 * la, tag + "_map_s2": np.array(s2),
                tag + "_map_L": L, tag + "_map_bits": bits})


def ldpc_demap(rcc, rmod, params, rs, out, tag):
    sigma = 0.9
    llr = 2.0 * (1.0 + sigma * rs.randn(2 * 96)) / sigma ** 2
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        dec, llr_out = rcc.ldpc_bp_decode(llr.copy(), params, "MSA", 6)
    out.update({tag + "_ldpc_llr": llr, tag + "_ldpc_dec": dec, tag + "_ldpc_out": llr_out})
    modem = rmod.QAMModem(16)
    y = modem.modulate(rs.randint(0, 2, 4 * 30)) + 0.4 * (rs.randn(30) + 1j * rs.randn(30))
    with np.errstate(all="ignore"):
        soft = modem.demodulate(y, "soft", 0.7)
    out.update({tag + "_demap_y": y, tag + "_demap_soft": soft, tag + "_demap_hard": modem.demodulate(y, "hard")})


def mimo(rmod, rlinks, rs, out, tag):
    for m, n in ((4, 2), (16, 3), (16, 4)):
        rq = rmod.QAMModem(m)

        def demode(s):
            return rq.demodulate(s, "hard")
        H, Y, NV, ST, KH, KS, BF = [], [], [], [], [], [], []
        for _ in range(10):
            nb = rq.num_bits_symbol
            h = (rs.randn(n, n) + 1j * rs.randn(n, n)) * np.sqrt(0.5)
            nv = n / 10 ** (rs.uniform(5, 25) / 10)
            y = h.dot(rq.modulate(rs.randint(0, 2, n * nb))) + (rs.randn(n) + 1j * rs.randn(n)) * np.sqrt(nv / 2)
            stack = tuple(rs.randint(1, 6, n - 1))
            H.append(h), Y.append(y), NV.append(nv), ST.append(stack)
            KH.append(rmod.kbest(y, h, rq.constellation, 6))
            KS.append(rmod.kbest(y, h, rq.constellation, 6, nv, "soft", demode))
            BF.append(rmod.best_first_detector(y, h, rq.constellation, stack, nv, demode, 100))
        key = "%s_mimo_q%d_n%d" % (tag, m, n)
        for name, v in (("h", H), ("y", Y), ("nv", NV), ("stack", ST), ("kbest_hard", KH), ("kbest_soft", KS), ("best_first", BF)):
            out[key + "_" + name] = np.array(v)
    rq = rmod.QAMModem(16)

    def detector(y, h, constellation, noise_var, a_priori):
        return rmod.kbest(y, h, constellation, 8, noise_var, "soft", lambda s: rq.demodulate(s, "hard")) + 0.25 * a_priori

    def decoder(llr):
        return np.tanh(llr) * 3 + np.roll(llr, 1)

    def decision(llr):
        return (llr > 0).astype(int)
    nvec, n = 5, 2
    h = (rs.randn(nvec, n, n) + 1j * rs.randn(nvec, n, n)) * np.sqrt(0.5)
    y = np.einsum("ijk,ik->ij", h, rq.modulate(rs.randint(0, 2, nvec * n * 4)).reshape(nvec, n)) + 0.1 * rs.randn(nvec, n)
    ap = rs.randn(nvec * n * 4)
    out.update({tag + "_idd_h": h, tag + "_idd_y": y, tag + "_idd_ap": ap,
                tag + "_idd_ref": rlinks.idd_decoder(detector, decoder, decision, 3)(y, h, rq.constellation, 0.02, ap.copy(), n * 4)})


def main():
    import importlib
    import scipy.sparse as sp
    refimport.import_reference()
    rcc = importlib.import_module("commpy.channelcoding")
    rmod = importlib.import_module("commpy.modulation")
    rlinks = importlib.import_module("commpy.links")
    params = rcc.get_ldpc_code_params(os.path.join(refimport.REF_ROOT, "commpy/channelcoding/designs/ldpc/gallager/96.33.964.txt"), True)
    H = sp.csr_matrix(params["parity_check_matrix"])
    out = {"ldpc_H_indptr": H.indptr, "ldpc_H_indices": H.indices, "ldpc_H_shape": np.array(H.shape),
           "seeds": np.array(SEEDS)}
    for seed in SEEDS:
        tag = "s%d" % seed
        rs = np.random.RandomState(seed)
        viterbi_bcjr(rcc, rs, out, tag)
        ldpc_demap(rcc, rmod, params, rs, out, tag)
        mimo(rmod, rlinks, rs, out, tag)
    np.savez_compressed(os.path.join(GOLD, "live_reference.npz"), **out)
    print("wrote %d arrays" % len(out))


if __name__ == "__main__":
    main()

"""BER of the UNMODIFIED reference on an LDPC-coded link, replayed by tests/test_ldpc_link_gpu.py against LdpcLinkGPU; and
a few reference encodings, which the GPU encoder must reproduce bit for bit.

* Link: the reference's LinkModel.link_performance_full_metrics with triang_ldpc_systematic_encode (WiMax 1440.720, rate
  1/2), QAMModem(16) or QAMModem(4), SISOFlatChannel(None, (1 + 0j, 0)) (AWGN) or SISOFlatChannel(None, (0j, 1))
  (Rayleigh), and ldpc_bp_decode(..., 'MSA', 15), as commpy/tests/test_links.py:62-86 builds its coded link.  One
  transmission is one 720-bit message block.  Over fading the receiver knows the channel and demaps each symbol as
  demodulate(y / h, 'soft', nv / |h|^2), as oracle/make_fading_golden.py does.  The demapper returns log P(1) / P(0) and
  the decoder decides bit = signbit(llr), so the receiver hands the decoder the negated LLRs.
* Encodings: random messages of WiMax 1440.720 and 960.720.a through triang_ldpc_systematic_encode.
* Codes: the parity-check matrices of the reference's four design files as coordinates (the files are not copied), for
  the tests of the encoder plan (tests/model_ldpc_encode.py).

    python oracle/make_ldpc_link_golden.py       # writes tests/golden/ldpc_link_ber.npz (6.3 minutes on 8 cores)
TEST INFRASTRUCTURE ONLY."""
import os
import sys
from fractions import Fraction
from multiprocessing import Pool

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path = [p for p in sys.path if os.path.abspath(p or ".") != HERE]
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np

import refimport

GOLD = os.path.join(os.path.dirname(HERE), "tests", "golden")
DESIGNS = os.path.join(refimport.REF_ROOT, "commpy", "channelcoding", "designs", "ldpc", "wimax")
# (modem order, channel) -> three SNR_dB points where the reference's BER lies between ~1e-3 and ~1e-1
CASES = {
    (4, "awgn"): [4.25, 4.5, 5.0],
    (16, "awgn"): [9.5, 10.0, 10.5],
    (4, "rayleigh"): [6.0, 6.5, 7.0],
    (16, "rayleigh"): [11.5, 12.0, 12.5],
}
BLOCKS = 400                 # transmissions (720-bit message blocks) per point
K = 720
ENCODINGS = 6                # reference encodings stored per code


def _ref():
    refimport.import_reference()
    import importlib
    return (importlib.import_module("commpy.links"), importlib.import_module("commpy.modulation"),
            importlib.import_module("commpy.channels"), importlib.import_module("commpy.channelcoding.ldpc"))


def point(args):
    (M, channel, snr), seed = args
    rl, rm, rch, rldpc = _ref()
    params = rldpc.get_ldpc_code_params(os.path.join(DESIGNS, "1440.720.txt"), True)
    modem = rm.QAMModem(M)
    fading = (0j, 1) if channel == "rayleigh" else (1 + 0j, 0)

    def modulate(bits):
        return modem.modulate(rldpc.triang_ldpc_systematic_encode(bits, params, False).reshape(-1, order="F"))

    def receive(y, h, constellation, nv):
        if channel == "awgn":
            return modem.demodulate(y, "soft", nv)
        return np.concatenate([modem.demodulate(y[i:i + 1] / h[i], "soft", nv / abs(h[i]) ** 2) for i in range(len(y))])

    def decoder(llrs):
        return rldpc.ldpc_bp_decode(-llrs, params, "MSA", 15)[0][:K].reshape(-1, order="F")

    np.random.seed(seed)
    model = rl.LinkModel(modulate, rch.SISOFlatChannel(None, fading), receive, modem.num_bits_symbol, modem.constellation,
                         modem.Es, decoder, Fraction(1, 2))
    b, bes, _, _ = model.link_performance_full_metrics([snr], BLOCKS, 10 ** 9, K, Fraction(1, 2), stop_on_surpass_error=False)
    print(M, channel, snr, b[0], flush=True)
    return np.asarray(bes[0], dtype=np.int64).reshape(-1)


def main():
    _, _, _, rldpc = _ref()
    out = {"blocks": np.array(BLOCKS), "k": np.array(K)}
    for d in ("gallager/96.3.963", "gallager/96.33.964", "wimax/1440.720", "wimax/960.720.a"):
        params = rldpc.get_ldpc_code_params(os.path.join(DESIGNS, "..", d + ".txt"), True)
        H = params["parity_check_matrix"].tocoo()
        key = "H_" + d.split("/")[1].replace(".", "_")
        out[key + "_rows"], out[key + "_cols"] = H.row.astype(np.int32), H.col.astype(np.int32)
        out[key + "_shape"] = np.array(H.shape)
    rs = np.random.RandomState(1440)
    for name in ("1440.720", "960.720.a"):
        params = rldpc.get_ldpc_code_params(os.path.join(DESIGNS, name + ".txt"), True)
        k = params["n_vnodes"] - params["n_cnodes"]
        msg = rs.randint(0, 2, (ENCODINGS, k))
        cw = np.stack([rldpc.triang_ldpc_systematic_encode(m, params, False) for m in msg])
        key = "wimax_" + name.replace(".", "_")
        out[key + "_msg"] = msg.astype(np.uint8)
        out[key + "_cw"] = cw.astype(np.uint8)
    jobs = []
    for c, ((M, channel), snrs) in enumerate(sorted(CASES.items())):
        for i, snr in enumerate(snrs):
            jobs.append(((M, channel, snr), 5000 + 10 * c + i))
    with Pool(min(len(jobs), os.cpu_count() or 1)) as pool:
        res = pool.map(point, jobs, chunksize=1)
    for c, ((M, channel), snrs) in enumerate(sorted(CASES.items())):
        key = "qam%d_%s" % (M, channel)
        errs = np.stack(res[3 * c:3 * c + 3])
        out[key + "_snr"] = np.array(snrs)
        out[key + "_block_errors"] = errs                  # bit errors of every 720-bit block
        out[key + "_ber"] = errs.sum(axis=1) / float(K * BLOCKS)
    np.savez_compressed(os.path.join(GOLD, "ldpc_link_ber.npz"), **out)


if __name__ == "__main__":
    main()

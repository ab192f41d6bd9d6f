"""Small invocation of every kernel family (used under compute-sanitizer by scripts/sanitize.sh)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import helpers
from commpy_b200.channelcoding import (RandInterlv, ldpc_bp_decode_batch, map_decode_batch, turbo_decode_batch, viterbi_decode_batch,
                                        viterbi_decode_punctured_batch, puncturing)
from commpy_b200.links import ConvLinkGPU
from commpy_b200.modulation import QAMModem, PSKModem

rs = np.random.RandomState(0)
tr = helpers.k7()
# Viterbi: hard (byte and packed), soft, unquantized, punctured, generic trellis
_, x = helpers.channel_frames(tr, rs, 70, 200, "hard", "cont", flip=0.06)
viterbi_decode_batch(x.astype(np.uint8), tr, None, "hard")
_, x = helpers.channel_frames(tr, rs, 70, 256, "hard", "cont", flip=0.06)
viterbi_decode_batch(np.packbits(x.astype(np.uint8), axis=1), tr, None, "hard", packed=True)
for mode in ("soft", "unquantized"):
    _, x = helpers.channel_frames(tr, rs, 40, 130, mode, "term", ebn0_db=2.0)
    viterbi_decode_batch(x.astype(np.float32), tr, 15, mode)
pv = [1, 1, 1, 0, 0, 1]
_, x = helpers.channel_frames(tr, rs, 40, 300, "soft", "cont", ebn0_db=3.0)
viterbi_decode_punctured_batch(np.stack([puncturing(r, pv) for r in x]).astype(np.float32), tr, pv, x.shape[1])
g = helpers.reference_test_trellises()[2]
_, x = helpers.channel_frames(g, rs, 20, 120 * g.k, "hard", "cont", flip=0.05)
viterbi_decode_batch(x.astype(np.uint8), g, None, "hard")
# BCJR / turbo
rsc = helpers.rsc_k4()
N = 2048
ys, y1, y2 = (torch.randn(6, N, device="cuda") * 0.8 - 1 for _ in range(3))
map_decode_batch(ys, y1, rsc, 0.64, torch.zeros(6, N, device="cuda"))
turbo_decode_batch(ys, y1, y2, rsc, 0.64, 2, RandInterlv(N, 1))
turbo_decode_batch(ys[:, :516].contiguous(), y1[:, :516].contiguous(), y2[:, :516].contiguous(), rsc, 0.64, 2, RandInterlv(516, 2),
                   torch.randn(6, 516, device="cuda"))            # step-major loop, 4-step tail segment, a-priori L_int
ys, y1 = (torch.randn(5, 301, device="cuda") - 1 for _ in range(2))
map_decode_batch(ys, y1, rsc, 0.7, torch.zeros(5, 301, device="cuda"))
# LDPC: bulk-copy check pass (>= 128 frames), small batch, fp64, SPA
import scipy.sparse as sp
gl = np.load(os.path.join(ROOT, "tests", "golden", "ldpc.npz"))
rel, nblk, iters, m, n = gl["l03_meta"]
H = sp.csr_matrix((np.ones(len(gl["l03_indices"]), np.int8), gl["l03_indices"], gl["l03_indptr"]), shape=(int(m), int(n)))
params = {"n_vnodes": int(n), "n_cnodes": int(m), "parity_check_matrix": H.tocsc()}
sigma = 0.8
llr = (2.0 * (1.0 + sigma * rs.randn(160, int(n))) / sigma ** 2)
ldpc_bp_decode_batch(llr.astype(np.float32), params, 6, "fp32")
ldpc_bp_decode_batch(llr[:9].astype(np.float32), params, 6, "fp32")
ldpc_bp_decode_batch(llr[:9].copy(), params, 4, "fp64")
ldpc_bp_decode_batch(llr[:9].astype(np.float32), params, 4, "fp32", decoder_algorithm="SPA")
# demapper (separable, general, hard) and the TX + link chain
y = torch.view_as_complex(torch.randn(5000, 2, device="cuda") * 3)
QAMModem(64).demodulate_batch(y, "soft", 1.5)
PSKModem(8).demodulate_batch(y, "soft", 0.5)
QAMModem(16).demodulate_batch(y, "hard")
link = ConvLinkGPU(tr, QAMModem(16), frame_bits=512, frames_per_batch=64, decoding_type="soft", seed=1)
link.link_performance([9.0], send_max=100000, err_min=10 ** 9)
link = ConvLinkGPU(helpers.k7_wifi_quirk(), QAMModem(256), frame_bits=600, frames_per_batch=64, decoding_type="soft", seed=1, puncture=pv)
link.link_performance([27.0], send_max=100000, err_min=10 ** 9)
# flat fading: CSI demapper (separable, general, hard, h = 0 included), fading TX (word-parallel, bit-serial, punctured)
h = torch.view_as_complex(torch.randn(5000, 2, device="cuda"))
h[::50] = 0
QAMModem(64).demodulate_batch(y, "soft", 1.5, channel_gains=h)
PSKModem(8).demodulate_batch(y, "soft", 0.5, channel_gains=h)
QAMModem(16).demodulate_batch(y, "hard", channel_gains=h)
link = ConvLinkGPU(tr, QAMModem(16), frame_bits=512, frames_per_batch=64, decoding_type="soft", seed=1, fading_param=(0j, 1))
link.link_performance([12.0], send_max=100000, err_min=10 ** 9)
link = ConvLinkGPU(tr, QAMModem(4), frame_bits=200, frames_per_batch=64, decoding_type="hard", seed=1, fading_param=(0j, 1))
link.link_performance([12.0], send_max=30000, err_min=10 ** 9)
link = ConvLinkGPU(helpers.k7_wifi_quirk(), QAMModem(16), frame_bits=600, frames_per_batch=64, decoding_type="soft", seed=1,
                   puncture=pv, fading_param=(0.6 + 0j, 0.64))
link.link_performance([20.0], send_max=100000, err_min=10 ** 9)
# turbo link over fading: fading turbo TX (N not a multiple of 4), combiner (vector path + tail, unaligned scalar path)
from commpy_b200.links import TurboLinkGPU, bpsk_combine
link = TurboLinkGPU(rsc, RandInterlv(301, 3), 301, frames_per_batch=37, iterations=2, seed=1, fading_param=(0j, 1))
link.link_performance([2.0], send_max=30000, err_min=10 ** 9)
bpsk_combine(y[:4999], h[:4999])
bpsk_combine(y[1:], h[:4999])
# LDPC encoder (peeled and dense forms, a batch that is not a multiple of 32) and the LDPC link over AWGN and fading
from commpy_b200 import _lib
from commpy_b200.channelcoding import ldpc_encode_batch
from commpy_b200.links import LdpcLinkGPU
Hs = helpers.dvbs2_like_H(n=720, m=360, n8=144, n3=216)
sparams = {"parity_check_matrix": Hs.tocsc(), "n_vnodes": 720, "n_cnodes": 360}
smsg = rs.randint(0, 2, (45, 360)).astype(np.uint8)
ldpc_encode_batch(smsg, sparams)
_lib.set_option(_lib.OPT_LDPC_ENC_FORCE_DENSE, 1)
ldpc_encode_batch(smsg, sparams)
_lib.set_option(_lib.OPT_LDPC_ENC_FORCE_DENSE, 0)
link = LdpcLinkGPU(sparams, QAMModem(16), 37, n_iters=4, seed=1)
link.link_performance([8.0], send_max=30000, err_min=10 ** 9)
link = LdpcLinkGPU(sparams, QAMModem(4), 37, n_iters=4, seed=1, fading_param=(0j, 1))
link.link_performance([8.0], send_max=30000, err_min=10 ** 9)
# turbo link over a modem: parity kernel on its byte path (N = 301) and 16-byte path (N = 512), both modem TX entry points
from commpy_b200.links import turbo_link_tx_modem, turbo_link_tx_modem_fading
link = TurboLinkGPU(rsc, RandInterlv(301, 3), 301, frames_per_batch=37, iterations=2, seed=1, modem=PSKModem(8))
link.link_performance([4.0], send_max=30000, err_min=10 ** 9)
link = TurboLinkGPU(rsc, RandInterlv(512, 3), 512, frames_per_batch=37, iterations=2, seed=1, fading_param=(0j, 1),
                    modem=QAMModem(16))
link.link_performance([6.0], send_max=30000, err_min=10 ** 9)
turbo_link_tx_modem(rsc, RandInterlv(512, 2), QAMModem(256), 33, 512, 3, 5, 0.5)
turbo_link_tx_modem_fading(rsc, RandInterlv(301, 2), PSKModem(8), 33, 301, 3, 5, 0.5, (0.6 + 0j, 0.64))
torch.cuda.synchronize()
print("sanitize driver ok")

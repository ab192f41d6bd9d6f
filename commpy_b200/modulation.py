"""Modems: constellation construction / mapping on the host, soft and hard demapping on the GPU.

Mirror of commpy/modulation.py:39-262 (Modem, PSKModem, QAMModem).  `demodulate` runs in CUDA
(commpy_b200/csrc/demap.cu) through `cpb_demod_soft` / `cpb_demod_hard`; there is no CPU demapper.
The MIMO tree-search detectors (kbest, best_first_detector, max_log_approx, bit_lvl_repr: :325-646) are host-side mirrors
(callers of the decoders in coded MIMO links); OFDM helpers are outside the decoding path.
"""
import ctypes as C

import numpy as np

from . import _lib
from .utilities import signal_power

__all__ = ["Modem", "PSKModem", "QAMModem", "kbest", "best_first_detector", "max_log_approx", "bit_lvl_repr"]


class _ModemBox:
    def __init__(self, ptr):
        self.ptr = ptr

    def __del__(self):
        try:
            if self.ptr:
                _lib.load().cpb_modem_destroy(self.ptr)
        except Exception:
            pass


class Modem:
    """Custom modem (modulation.py:39-172).

    Attributes as in the reference: `constellation` (settable; length must be a power of two), `Es`, `m`,
    `num_bits_symbol`.  Symbol index k <-> bit pattern of k, MSB first.  With `reorder_as_gray=True` the given
    points are re-indexed so that `constellation[k] = given[gray^-1(k)]` (:68-77).
    """

    def __init__(self, constellation, reorder_as_gray=True):
        if reorder_as_gray:
            size = len(constellation)
            gray = np.arange(size) ^ (np.arange(size) >> 1)          # binary-reflected Gray sequence
            self.constellation = np.array(constellation)[gray.argsort()]
        else:
            self.constellation = constellation

    @property
    def constellation(self):
        return self._constellation

    @constellation.setter
    def constellation(self, value):
        num_bits_symbol = np.log2(len(value))
        if num_bits_symbol != int(num_bits_symbol):
            raise ValueError("Constellation length must be a power of 2.")
        self._constellation = np.array(value)
        self.Es = signal_power(self.constellation)
        self.m = self._constellation.size
        self.num_bits_symbol = int(num_bits_symbol)
        self._handles = {}

    def modulate(self, input_bits):
        """Map bits (MSB first, `num_bits_symbol` per symbol) to constellation points (modulation.py:79-98)."""
        bits = np.asarray(input_bits).astype(np.int64)
        nb = self.num_bits_symbol
        full = (len(bits) // nb) * nb
        idx = bits[:full].reshape(-1, nb) @ (1 << np.arange(nb - 1, -1, -1))
        if full != len(bits):                                   # a short last group is read as a shorter number
            tail = bits[full:]
            idx = np.append(idx, int(tail @ (1 << np.arange(len(tail) - 1, -1, -1))))
        return self._constellation[idx]

    def _handle(self):
        torch = _lib.require_cuda()
        dev = torch.cuda.current_device()
        box = self._handles.get(dev)
        if box is None:
            pts = np.ascontiguousarray(self._constellation, dtype=np.complex128)
            h = C.c_void_p()
            rc = _lib.load().cpb_modem_create(_lib.ptr(pts.view(np.float64)), int(self.m), C.byref(h))
            _lib.check(rc, "Modem constellation")
            box = _ModemBox(h)
            self._handles[dev] = box
        return box.ptr

    def demodulate_batch(self, input_symbols, demod_type, noise_var=0, channel_gains=None):
        """GPU demapper on a torch CUDA complex64 tensor (or numpy complex array) of any shape.

        Returns a torch CUDA tensor shaped input.shape + (num_bits_symbol,) flattened on the last two axes:
        float32 LLRs ('soft') or uint8 bits ('hard').

        `channel_gains` (a scalar, or an array or tensor broadcastable to the symbols): the flat-fading gain h of each
        symbol, known to the receiver.  The distances become |y - h c|^2, i.e. the reference's
        demodulate(y / h, 'soft', noise_var / |h|^2) symbol by symbol (cpb_demod_soft_csi / cpb_demod_hard_csi); LLRs are
        finite in deep fades and 0 where h = 0.  None: the AWGN demapper."""
        torch = _lib.require_cuda()
        if demod_type not in ("hard", "soft"):
            raise ValueError('demod_type must be "hard" or "soft"')
        if hasattr(input_symbols, "data_ptr"):
            y = input_symbols if input_symbols.is_cuda else input_symbols.cuda()
            if y.dtype != torch.complex64:
                y = y.to(torch.complex64)
            y = y.contiguous()
        else:
            y = torch.from_numpy(np.ascontiguousarray(np.atleast_1d(input_symbols), dtype=np.complex64)).cuda()
        nsym = y.numel()
        nb = self.num_bits_symbol
        yr = torch.view_as_real(y)
        lib = _lib.load()
        h = None if channel_gains is None else _gains_like(channel_gains, y, torch)
        if demod_type == "soft":
            if not noise_var > 0:
                raise ValueError("noise_var must be positive for soft demodulation")
            out = torch.empty((nsym * nb,), dtype=torch.float32, device=y.device)
            if h is None:
                rc = lib.cpb_demod_soft(self._handle(), _lib.ptr(yr), C.c_int64(nsym), C.c_float(noise_var), _lib.ptr(out),
                                        _lib.stream_ptr(torch))
            else:
                rc = lib.cpb_demod_soft_csi(self._handle(), _lib.ptr(yr), _lib.ptr(h), C.c_int64(nsym), C.c_float(noise_var),
                                            _lib.ptr(out), _lib.stream_ptr(torch))
        else:
            out = torch.empty((nsym * nb,), dtype=torch.uint8, device=y.device)
            if h is None:
                rc = lib.cpb_demod_hard(self._handle(), _lib.ptr(yr), C.c_int64(nsym), _lib.ptr(out), _lib.stream_ptr(torch))
            else:
                rc = lib.cpb_demod_hard_csi(self._handle(), _lib.ptr(yr), _lib.ptr(h), C.c_int64(nsym), _lib.ptr(out),
                                            _lib.stream_ptr(torch))
        _lib.check(rc, "demodulate")
        return out.reshape(tuple(y.shape[:-1]) + (y.shape[-1] * nb,)) if y.dim() > 1 else out

    def demodulate_soft_host(self, input_symbols, noise_var):
        """Soft demapper for HOST arrays through the pipelined host entry point (cpb_demod_soft_host: chunked H2D / kernel /
        D2H on the modem handle's streams).  numpy complex array (any shape) -> float32 numpy array of LLRs, MSB first."""
        _lib.require_cuda()
        if not noise_var > 0:
            raise ValueError("noise_var must be positive for soft demodulation")
        y = np.ascontiguousarray(np.atleast_1d(input_symbols), dtype=np.complex64)
        out = np.empty(y.size * self.num_bits_symbol, dtype=np.float32)
        rc = _lib.load().cpb_demod_soft_host(self._handle(), _lib.ptr(y.view(np.float32)), C.c_int64(y.size),
                                             C.c_float(noise_var), _lib.ptr(out))
        _lib.check(rc, "demodulate")
        return out.reshape(tuple(y.shape[:-1]) + (y.shape[-1] * self.num_bits_symbol,)) if y.ndim > 1 else out

    def demodulate(self, input_symbols, demod_type, noise_var=0, channel_gains=None):
        """Drop-in for Modem.demodulate (modulation.py:100-141).

        'hard': nearest constellation point -> its bits (int8).  'soft': exact log-sum-exp LLRs
        log(sum_{bit=1} exp(-|y-c|^2/noise_var) / sum_{bit=0} ...), float64 array, MSB first per symbol.
        Computed in float32 on the GPU (relative error ~1e-4); finite where the reference under/overflows.
        `channel_gains`: per-symbol flat-fading gains h (see `demodulate_batch`); a fading receiver for LinkModel is
        `lambda y, h, c, nv: modem.demodulate(y, 'soft', nv, channel_gains=h)`."""
        if channel_gains is not None:
            y = np.atleast_1d(np.asarray(input_symbols))
            try:
                h = np.broadcast_to(np.asarray(channel_gains), y.shape)
            except ValueError:
                raise ValueError("channel_gains of shape %s does not broadcast to the symbols' shape %s"
                                 % (np.shape(channel_gains), y.shape)) from None
            out = self.demodulate_batch(y.reshape(-1), demod_type, noise_var, h.reshape(-1)).cpu().numpy()
            return out.astype(np.float64) if demod_type == "soft" else out.astype(np.int8)
        if demod_type == "soft":
            return self.demodulate_soft_host(np.atleast_1d(np.asarray(input_symbols)).reshape(-1), noise_var).astype(np.float64)
        out = self.demodulate_batch(np.atleast_1d(np.asarray(input_symbols)).reshape(-1), demod_type, noise_var)
        return out.cpu().numpy().astype(np.int8)


def _gains_like(channel_gains, y, torch):
    """per-symbol gains as a contiguous complex64 tensor of y's shape on y's device"""
    if hasattr(channel_gains, "data_ptr"):
        h = channel_gains.to(device=y.device, dtype=torch.complex64)
    else:
        h = torch.from_numpy(np.ascontiguousarray(channel_gains, dtype=np.complex64)).to(y.device)
    try:
        h = torch.broadcast_to(h, y.shape)
    except RuntimeError:
        raise ValueError("channel_gains of shape %s does not broadcast to the symbols' shape %s"
                         % (tuple(h.shape), tuple(y.shape))) from None
    return torch.view_as_real(h.contiguous())


class PSKModem(Modem):
    """M-PSK: points exp(j*2*pi*i/m), Gray-labelled (modulation.py:175-210)."""

    def __init__(self, m):
        num_bits_symbol = np.log2(m)
        if num_bits_symbol != int(num_bits_symbol):
            raise ValueError("Constellation length must be a power of 2.")
        super().__init__(np.exp(1j * np.arange(0, 2 * np.pi, 2 * np.pi / m)))


class QAMModem(Modem):
    """Square M-QAM on the odd-integer grid, Gray-labelled per axis, no power normalisation
    (modulation.py:213-262): Es = 2(m-1)/3."""

    def __init__(self, m):
        side = np.sqrt(m)
        if side != int(side):
            raise ValueError("m must lead to a square QAM.")
        side = int(side)
        pam = np.arange(-side + 1, side, 2)
        # column-by-column snake through the grid: real part fixed per column, imaginary part up then down
        imag = np.tile(np.hstack((pam, pam[::-1])), side // 2)
        real = pam.repeat(side)
        super().__init__(imag * 1j + real)


# ----------------------------------------------------------------------------------------------------
# MIMO detectors (host side): callers of the decoders in coded MIMO links, SURVEY 8(f) row 4.
# Tree searches over the QR-decomposed channel; they feed LLRs to the GPU decoders (ldpc_bp_decode, ...).
# ----------------------------------------------------------------------------------------------------
def max_log_approx(y, h, noise_var, pts_list, demode):
    """Max-log LLRs from a list of candidate symbol vectors (modulation.py:599-646): for every bit,
    -(min_{bit=0} |y - H x|^2 - min_{bit=1} |y - H x|^2) / (2 noise_var); an empty side counts as +inf."""
    pts_list = np.asarray(pts_list)
    npts = pts_list.shape[1]
    words = np.asarray(demode(pts_list.reshape(-1, order="F"))).reshape(npts, -1)
    dist = np.sum(np.abs(np.asarray(y)[:, None] - np.asarray(h).dot(pts_list)) ** 2, axis=0)
    llr = np.empty(words.shape[1])
    for k in range(words.shape[1]):
        d0 = dist[words[:, k] == 0]
        d1 = dist[words[:, k] == 1]
        llr[k] = (d0.min() if d0.size else np.inf) - (d1.min() if d1.size else np.inf)
    return -llr / (2 * noise_var)


def kbest(y, h, constellation, K, noise_var=0, output_type="hard", demode=None):
    """MIMO K-best (breadth-first) detection on the QR-decomposed channel (modulation.py:325-419): level by level from the
    last transmit antenna, every surviving candidate is extended by every constellation point and the K smallest partial
    distances survive.  'hard' returns the best symbol vector, 'soft' the max-log LLRs over the final survivors."""
    h = np.asarray(h)
    rows, cols = h.shape
    if cols > rows:
        raise ValueError("h has more columns than rows")
    if output_type not in ("hard", "soft"):
        raise ValueError('output_type must be "hard" or "soft"')
    q, r = np.linalg.qr(h)
    yt = q.conj().T.dot(y)
    cst = np.asarray(constellation)
    m = len(cst)
    cand = np.zeros((cols, 1), dtype=complex if np.iscomplexobj(cst) else float)
    resid = np.array(yt, dtype=complex)[:, None]
    dist = np.zeros(1)
    for level in range(cols - 1, -1, -1):
        ncand = cand.shape[1]
        cand = np.tile(cand, (1, m))
        resid = np.tile(resid, (1, m))
        hyp = np.repeat(cst, ncand)                          # point i for all candidates, then point i+1, ...
        cand[level] = hyp
        resid[level] = resid[level] - r[level, level] * hyp
        dist = np.tile(dist, m) + np.abs(resid[level]) ** 2
        keep = np.argsort(dist)[:K]
        cand, resid, dist = cand[:, keep], resid[:, keep], dist[keep]
        resid[:level] = resid[:level] - r[:level, level, None] * hyp[keep]
    if output_type == "hard":
        return cand[:, 0]
    return max_log_approx(y, h, noise_var, cand, demode)


class _TreeNode:
    """A node of the detection tree with lazy access to its next-best sibling: `order` indexes the parent's children by
    increasing partial metric."""
    __slots__ = ("vec", "metric", "_vecs", "_metrics", "_k")

    def __init__(self, vecs, metrics, k=0):
        self._vecs, self._metrics, self._k = vecs, metrics, k
        self.vec = vecs[:, k]
        self.metric = metrics[k]

    def sibling(self):
        return _TreeNode(self._vecs, self._metrics, self._k + 1) if self._k + 1 < len(self._metrics) else None

    def best_child(self, yt, r, cst):
        depth = self.vec.size + 1                              # symbols fixed in a child, counted from the last antenna
        vecs = np.empty((depth, cst.size), dtype=cst.dtype)
        vecs[0] = cst
        vecs[1:] = self.vec[:, None]
        metrics = np.abs(yt[-depth] - r[-depth, -depth:].dot(vecs)) ** 2 + self.metric
        order = np.argsort(metrics)
        return _TreeNode(vecs[:, order], metrics[order])


def best_first_detector(y, h, constellation, stack_size, noise_var, demode, llr_max):
    """MIMO best-first (stack) detection with max-log LLR output (modulation.py:422-565; He, Zhang, Liang, IEEE TVLSI 2019).

    One sorted stack per tree level; every sweep pops the best node of each level, re-inserts its next sibling and pushes its
    best child one level down when they lie inside the current search radius, then folds a reached leaf into the MAP /
    counter-hypothesis metrics; the stacks are cut to `stack_size` after every sweep.  Returns
    (metric_MAP - metric_counter-hypothesis) * (+-1 of the MAP bit) per bit, clipped to +-llr_max."""
    from bisect import bisect_right
    h = np.asarray(h)
    n = h.shape[0]
    cst = np.array(constellation)
    nbits = int(np.log2(cst.size))
    q, r = np.linalg.qr(h)
    yt = q.conj().T.dot(y)
    map_metric, map_bits = np.inf, None
    counter = np.full((n, nbits), np.inf)
    stacks = [[] for _ in range(n)]                            # stacks[i]: nodes with n - i symbols fixed; stacks[0]: leaves

    def push(stack, node):                                     # sorted by partial metric, after equal ones (bisect.insort)
        stack.insert(bisect_right([nd.metric for nd in stack], node.metric), node)

    def signed_bits(vec):
        b = np.asarray(demode(vec)).reshape(-1, nbits).astype(float)
        b[b == 0] = -1
        return b

    root = _TreeNode(np.empty((0, 1), dtype=cst.dtype), np.zeros(1))
    stacks[-1].append(root.best_child(yt, r, cst))
    while any(stacks[1:]):
        for lower in range(n - 1):
            level = lower + 1
            if not stacks[level]:
                continue
            node = stacks[level].pop(0)
            if map_bits is None:
                radius = np.inf                                # no leaf yet: keep everything
            else:
                differs = map_bits[level:] != signed_bits(node.vec)
                sel = counter[level:][differs]
                radius = max(counter[:level].max(), sel.max() if sel.size else np.inf)
            sib = node.sibling()
            if sib is not None and sib.metric <= radius:
                push(stacks[level], sib)
            child = node.best_child(yt, r, cst)
            if child.metric <= radius:
                push(stacks[lower], child)
        if stacks[0]:
            leaf = stacks[0][0]
            if leaf.metric < map_metric:
                np.minimum(counter, map_metric, out=counter)
                map_metric = leaf.metric
                map_bits = signed_bits(leaf.vec)
            else:
                np.minimum(counter, leaf.metric, out=counter)
            np.clip(counter, map_metric - llr_max, map_metric + llr_max, out=counter)
        stacks[0].clear()
        for lower in range(n - 1):
            del stacks[lower + 1][stack_size[lower]:]
    return ((map_metric - counter) * map_bits).reshape(-1)


def bit_lvl_repr(H, w):
    """Channel matrix of the bit-level representation: H (I_n kron w) for an even number of weights (modulation.py:568-596)."""
    if len(w) % 2:
        raise ValueError("Beta (length of w) must be even.")
    H = np.asarray(H)
    return H.dot(np.kron(np.eye(H.shape[1]), w))

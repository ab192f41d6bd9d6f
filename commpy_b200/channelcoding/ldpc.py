"""LDPC codes: design-file loader (host) and min-sum belief propagation on the GPU.

Mirror of commpy/channelcoding/ldpc.py.  `ldpc_bp_decode(..., 'MSA', ...)` runs in CUDA
(commpy_b200/csrc/ldpc.cu) through `cpb_ldpc_minsum`; there is no CPU decode path.
"""
import ctypes as C

import numpy as np
import scipy.sparse as sp

from .. import _lib

__all__ = ["build_matrix", "get_ldpc_code_params", "ldpc_bp_decode", "ldpc_bp_decode_batch", "write_ldpc_params",
           "triang_ldpc_systematic_encode", "ldpc_encode_batch"]

_llr_max = 500


def build_matrix(ldpc_code_params):
    """Add 'parity_check_matrix' (CSC int8) and 'generator_matrix' (CSR) to the dict (ldpc.py:13-48).

    The generator is valid for triangular systematic codes only, like the reference's."""
    import scipy.sparse.linalg as splg
    n_c = ldpc_code_params["n_cnodes"]
    if ldpc_code_params.get("parity_check_matrix") is not None and "cnode_adj_list" not in ldpc_code_params:
        H = sp.csc_matrix(ldpc_code_params["parity_check_matrix"])     # dict built from a matrix: only the generator is missing
        ldpc_code_params["generator_matrix"] = splg.inv(H[:, -n_c:]).dot(H[:, :-n_c]).tocsr()
        return
    deg = np.asarray(ldpc_code_params["cnode_deg_list"])
    adj = np.asarray(ldpc_code_params["cnode_adj_list"]).reshape((n_c, ldpc_code_params["max_cnode_deg"]))
    rows = np.repeat(np.arange(n_c), deg)
    cols = np.concatenate([adj[i, :deg[i]] for i in range(n_c)])
    H = sp.csc_matrix((np.ones(len(rows), np.int8), (rows, cols)), shape=(n_c, ldpc_code_params["n_vnodes"]))
    H.data[:] = 1
    ldpc_code_params["parity_check_matrix"] = H
    ldpc_code_params["generator_matrix"] = splg.inv(H[:, -n_c:]).dot(H[:, :-n_c]).tocsr()


def get_ldpc_code_params(ldpc_design_filename, compute_matrix=False):
    """Parse an LDPC design file (ldpc.py:51-141; format documented there) into the reference's dict."""
    with open(ldpc_design_filename) as fh:
        n_v, n_c = (int(x) for x in fh.readline().split(" "))
        max_v, max_c = (int(x) for x in fh.readline().split(" "))
        vdeg = np.array([int(x) for x in fh.readline().split(" ")[:-1]], np.int32)
        cdeg = np.array([int(x) for x in fh.readline().split(" ")[:-1]], np.int32)
        vadj = -np.ones([n_v, max_v], int)
        cadj = -np.ones([n_c, max_c], int)
        for v in range(n_v):
            vadj[v, :vdeg[v]] = [int(x) - 1 for x in fh.readline().split("\t")]
        for c in range(n_c):
            cadj[c, :cdeg[c]] = [int(x) - 1 for x in fh.readline().split("\t")]
    c_v_map = -np.ones([n_c, max_c], int)
    v_c_map = -np.ones([n_v, max_v], int)
    for c in range(n_c):
        for i, v in enumerate(cadj[c, :cdeg[c]]):
            c_v_map[c, i] = np.where(vadj[v, :] == c)[0][0]
    for v in range(n_v):
        for i, c in enumerate(vadj[v, :vdeg[v]]):
            v_c_map[v, i] = np.where(cadj[c, :] == v)[0][0]
    params = {
        "n_vnodes": n_v, "n_cnodes": n_c, "max_cnode_deg": max_c, "max_vnode_deg": max_v,
        "cnode_adj_list": cadj.flatten().astype(np.int32), "cnode_vnode_map": c_v_map.flatten().astype(np.int32),
        "vnode_adj_list": vadj.flatten().astype(np.int32), "vnode_cnode_map": v_c_map.flatten().astype(np.int32),
        "cnode_deg_list": cdeg, "vnode_deg_list": vdeg,
    }
    if compute_matrix:
        build_matrix(params)
    return params


class _LdpcBox:
    def __init__(self, ptr):
        self.ptr = ptr

    def __del__(self):
        try:
            if self.ptr:
                _lib.load().cpb_ldpc_destroy(self.ptr)
        except Exception:
            pass


def _ldpc_handle(ldpc_code_params):
    torch = _lib.require_cuda()
    if ldpc_code_params.get("parity_check_matrix") is None:
        build_matrix(ldpc_code_params)                       # ldpc.py:189-190
    Hm = ldpc_code_params["parity_check_matrix"]
    dev = torch.cuda.current_device()
    cache = ldpc_code_params.get("_cpb_handles")
    if cache is None or cache.get("id") != id(Hm):
        cache = {"id": id(Hm)}
        ldpc_code_params["_cpb_handles"] = cache
    if dev not in cache:
        H = sp.csr_matrix(Hm)
        H.sort_indices()
        row_ptr = np.ascontiguousarray(H.indptr, dtype=np.int32)
        col_idx = np.ascontiguousarray(H.indices, dtype=np.int32)
        h = C.c_void_p()
        rc = _lib.load().cpb_ldpc_create(_lib.ptr(row_ptr), _lib.ptr(col_idx), int(H.shape[0]), int(H.shape[1]),
                                         C.byref(h))
        _lib.check(rc, "ldpc parity-check matrix")
        cache[dev] = (_LdpcBox(h), H.shape[1])
    return cache[dev][0].ptr, cache[dev][1]


def _code_dims(ldpc_code_params):
    """(n, m) of a code dict, from its parity-check matrix when it has one, else from its design-file fields"""
    H = ldpc_code_params.get("parity_check_matrix")
    if H is not None:
        return int(H.shape[1]), int(H.shape[0])
    return int(ldpc_code_params["n_vnodes"]), int(ldpc_code_params["n_cnodes"])


def ldpc_encode_batch(msg, ldpc_code_params):
    """Systematic LDPC encoding on the GPU (cpb_ldpc_encode) of a (batch, k) array of message bits, k = n - m.

    msg : torch tensor (CUDA or host) or numpy array of 0/1 values.  Returns the (batch, n) uint8 code words
    [message | parity] with H c = 0 over GF(2), as a torch CUDA tensor.  The parity is p = H_p^-1 H_s msg with
    H = [H_s | H_p], H_p the last m columns, computed by peeling when H_p allows it and through the dense GF(2) inverse
    otherwise (DESIGN.md section 4.7).  Where H_p is invertible over GF(2) the parity of a message is unique, so this is
    what triang_ldpc_systematic_encode returns whenever the reference's encoding is a code word.
    Raises ValueError for a wrong shape, values other than 0/1 or an H_p that is singular over GF(2), and
    NotImplementedError for a code whose H_p does not peel and whose dense inverse (k * m bits) exceeds 2^26 bits.
    A dict given only as a parity_check_matrix is used as it is: no generator matrix is computed."""
    torch = _lib.require_cuda()
    handle, n = _ldpc_handle(ldpc_code_params)
    k = n - _code_dims(ldpc_code_params)[1]
    x = msg if hasattr(msg, "data_ptr") else torch.from_numpy(np.ascontiguousarray(msg))
    if x.dim() != 2 or x.shape[1] != k:
        raise ValueError("msg must be (batch, k) = (batch, %d), got %s" % (k, tuple(x.shape)))
    x = x.cuda()
    if x.numel() and bool(((x != 0) & (x != 1)).any()):
        raise ValueError("msg must hold 0/1 values")
    x = x.to(torch.uint8).contiguous()
    cw = torch.empty((x.shape[0], n), dtype=torch.uint8, device=x.device)
    rc = _lib.load().cpb_ldpc_encode(handle, _lib.ptr(x), C.c_int64(x.shape[0]), _lib.ptr(cw), _lib.stream_ptr(torch))
    _lib.check(rc, "ldpc_encode (H_p = H[:, k:] must be invertible over GF(2))")
    return cw


def ldpc_bp_decode_batch(llr, ldpc_code_params, n_iters, precision="fp32", return_llrs=True, return_iters=False,
                         decoder_algorithm="MSA"):
    """Min-sum ('MSA') or sum-product ('SPA') BP on a (batch, n_vnodes) array of LLRs (reference sign convention:
    bit = signbit(llr)).

    llr : torch CUDA tensor (float32 for 'fp32', float64 for 'fp64' -- clipped IN PLACE to +-500) or numpy array.
    Returns dec (batch, n) uint8 [, out_llrs (batch, n)] [, iterations (batch,) int32] as torch CUDA tensors.
    """
    torch = _lib.require_cuda()
    handle, n = _ldpc_handle(ldpc_code_params)
    tdt = torch.float64 if precision == "fp64" else torch.float32
    if hasattr(llr, "data_ptr"):
        x = llr if llr.is_cuda else llr.cuda()
        if x.dtype != tdt or not x.is_contiguous():
            x = x.to(tdt).contiguous()
    else:
        x = torch.from_numpy(np.ascontiguousarray(llr, dtype=np.float64 if precision == "fp64" else np.float32)).cuda()
    if x.dim() != 2 or x.shape[1] != n:
        raise ValueError("llr must be (batch, n_vnodes)")
    batch = x.shape[0]
    dec = torch.empty((batch, n), dtype=torch.uint8, device=x.device)
    out = torch.empty_like(x) if return_llrs else None
    iters = torch.empty((batch,), dtype=torch.int32, device=x.device) if return_iters else None
    if decoder_algorithm not in ("MSA", "SPA"):
        raise NameError('Please input a valid decoder_algorithm string (meanning "SPA" or "MSA").')
    fn = _lib.load().cpb_ldpc_minsum if decoder_algorithm == "MSA" else _lib.load().cpb_ldpc_sumproduct
    rc = fn(handle, _lib.ptr(x), _lib.LDPC_FP64 if precision == "fp64" else _lib.LDPC_FP32,
                                     C.c_int64(batch), int(n_iters), _lib.ptr(dec), _lib.ptr(out), _lib.ptr(iters),
                                     C.c_void_p(0), C.c_size_t(0), _lib.stream_ptr(torch))
    _lib.check(rc, "ldpc_bp_decode")
    res = [dec]
    if return_llrs:
        res.append(out)
    if return_iters:
        res.append(iters)
    return res[0] if len(res) == 1 else tuple(res)


def ldpc_bp_decode_batch_host(llr, ldpc_code_params, n_iters, precision="fp32", return_llrs=True, return_iters=False,
                              decoder_algorithm="MSA", out=None):
    """The same for a HOST array through the pipelined host entry point (cpb_ldpc_decode_host): `llr` is a C-contiguous
    numpy (batch, n) array of the precision's dtype and is clipped IN PLACE to +-500 like the reference (ldpc.py:186).
    Returns numpy arrays: dec (batch, n) uint8 [, out_llrs] [, iterations int32]; `out` (e.g. a pinned buffer) receives dec."""
    _lib.require_cuda()
    if decoder_algorithm not in ("MSA", "SPA"):
        raise NameError('Please input a valid decoder_algorithm string (meanning "SPA" or "MSA").')
    handle, n = _ldpc_handle(ldpc_code_params)
    dt = np.float64 if precision == "fp64" else np.float32
    x = llr if (isinstance(llr, np.ndarray) and llr.dtype == dt and llr.flags["C_CONTIGUOUS"]) else np.ascontiguousarray(llr, dtype=dt)
    if x.ndim != 2 or x.shape[1] != n:
        raise ValueError("llr must be (batch, n_vnodes)")
    batch = x.shape[0]
    from .turbo import _host_out
    dec = _host_out(out, (batch, n), np.uint8, "out")
    out = np.empty((batch, n), dtype=dt) if return_llrs else None
    iters = np.empty((batch,), dtype=np.int32) if return_iters else None
    rc = _lib.load().cpb_ldpc_decode_host(handle, 0 if decoder_algorithm == "MSA" else 1, _lib.ptr(x),
                                          _lib.LDPC_FP64 if precision == "fp64" else _lib.LDPC_FP32, C.c_int64(batch),
                                          int(n_iters), _lib.ptr(dec), _lib.ptr(out), _lib.ptr(iters))
    _lib.check(rc, "ldpc_bp_decode")
    res = [dec]
    if return_llrs:
        res.append(out)
    if return_iters:
        res.append(iters)
    return res[0] if len(res) == 1 else tuple(res)


def ldpc_bp_decode(llr_vec, ldpc_code_params, decoder_algorithm, n_iters, precision="fp64"):
    """Drop-in for commpy.channelcoding.ldpc_bp_decode (ldpc.py:144-254), 'MSA' and 'SPA' algorithms.

    `llr_vec` (1-D, one or several blocks back to back) is clipped in place to +-500 like the reference
    (:186).  With the default precision='fp64' the GPU reproduces the float64 reference bit for bit
    (decisions AND out_llrs); precision='fp32' is the throughput mode.  Returns (dec_word int8, out_llrs) with
    one block per column, squeezed (:251-254).  'SPA' (sum-product, :209-227) agrees with the reference within the
    conditioning of its check node (messages near the +-500 saturation knee may round either way; DESIGN.md section 4.4),
    'MSA' exactly; any other name raises NameError as the reference does (:239-240).
    """
    if decoder_algorithm not in ("MSA", "SPA"):
        raise NameError('Please input a valid decoder_algorithm string (meanning "SPA" or "MSA").')
    llr_vec = np.asarray(llr_vec) if not isinstance(llr_vec, np.ndarray) else llr_vec
    if np.issubdtype(llr_vec.dtype, np.floating):
        llr_vec.clip(-_llr_max, _llr_max, llr_vec)            # in place, ldpc.py:186
    _, n = _ldpc_handle(ldpc_code_params)
    n_blocks = llr_vec.size // n
    dec, out = ldpc_bp_decode_batch_host(llr_vec.reshape(n_blocks, n), ldpc_code_params, n_iters, precision,
                                         decoder_algorithm=decoder_algorithm)
    dec_word = dec.reshape(-1).reshape(-1, n_blocks, order="F").squeeze().astype(np.int8)
    out_llrs = out.astype(np.float64).reshape(-1).reshape(-1, n_blocks, order="F").squeeze()
    return dec_word, out_llrs


def write_ldpc_params(parity_check_matrix, file_path):
    """Write a dense 0/1 parity-check matrix as a design file (ldpc.py:257-299)."""
    H = np.asarray(parity_check_matrix)
    with open(file_path, "x") as fh:
        fh.write("{} {}\n".format(H.shape[1], H.shape[0]))
        fh.write("{} {}\n".format(H.sum(0).max(), H.sum(1).max()))
        fh.write("".join("{} ".format(d) for d in H.sum(0)) + "\n")
        fh.write("".join("{} ".format(d) for d in H.sum(1)) + "\n")
        for col in H.T:
            fh.write("\t".join(str(i + 1) for i in col.nonzero()[0]) + "\n")
        for row in H:
            fh.write("\t".join(str(i + 1) for i in row.nonzero()[0]) + "\n")
        fh.write("\n")


def triang_ldpc_systematic_encode(message_bits, ldpc_code_params, pad=True):
    """Systematic encoding with the generator of a (near-)triangular code (ldpc.py:302-354), host side."""
    if ldpc_code_params.get("generator_matrix") is None or ldpc_code_params.get("parity_check_matrix") is None:
        build_matrix(ldpc_code_params)
    message_bits = np.asarray(message_bits)
    block_length = ldpc_code_params["generator_matrix"].shape[1]
    modulo = len(message_bits) % block_length
    if modulo:
        if not pad:
            raise ValueError("Padding is disable but message length is not a multiple of block length.")
        message_bits = np.concatenate((message_bits, np.zeros(block_length - modulo, message_bits.dtype)))
    message_bits = message_bits.reshape(block_length, -1, order="F")
    parity_part = ldpc_code_params["generator_matrix"].dot(message_bits) % 2
    return np.vstack((message_bits, parity_part)).squeeze().astype(np.int8)

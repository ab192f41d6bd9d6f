"""NumPy GF(2) model of the systematic LDPC encoder plan (commpy_b200/csrc/ldpclink.cu, DESIGN.md section 4.7).

Code word c = [msg (k bits) | parity (m bits)], H = [H_s | H_p] with H_p the last m columns, parity p = H_p^-1 H_s msg.
* peeled form: rows whose parity part has exactly one unsolved bit are queued in ascending row order and taken first in,
  first out; taking row r solves that bit (its pivot).  The plan is the list of (row, pivot) steps; complete when m steps.
* dense form: P = H_p^-1 H_s by Gauss-Jordan elimination over GF(2) (lowest-index pivot row per column).
plan() chooses between them exactly as the library does."""
from collections import deque

import numpy as np

DENSE_MAX_BITS = 1 << 26
PEELED, DENSE = 0, 1


def _csr(H):
    import scipy.sparse as sp
    H = sp.csr_matrix(H)
    H.sort_indices()
    return H


def peel(H):
    """(order, pivot) int arrays of the peeled form, or None when H_p does not peel completely"""
    H = _csr(H)
    m, n = H.shape
    k = n - m
    rows = [H.indices[H.indptr[i]:H.indptr[i + 1]] for i in range(m)]
    prow = [r[r >= k] - k for r in rows]
    cnt = np.array([len(p) for p in prow])
    col_rows = [[] for _ in range(m)]
    for i in range(m):
        for j in prow[i]:
            col_rows[j].append(i)
    solved = np.zeros(m, bool)
    used = np.zeros(m, bool)
    q = deque(i for i in range(m) if cnt[i] == 1)
    order, pivot = [], []
    while q:
        i = q.popleft()
        if used[i] or cnt[i] != 1:
            continue
        j = [c for c in prow[i] if not solved[c]][-1]
        used[i] = solved[j] = True
        order.append(i)
        pivot.append(j)
        for r in col_rows[j]:
            cnt[r] -= 1
            if cnt[r] == 1 and not used[r]:
                q.append(r)
    if len(order) != m:
        return None
    return np.array(order), np.array(pivot)


def gf2_rank(A):
    A = (np.asarray(A) % 2).astype(np.uint8).copy()
    r = 0
    for c in range(A.shape[1]):
        nz = np.nonzero(A[r:, c])[0]
        if len(nz) == 0:
            continue
        p = r + nz[0]
        A[[r, p]] = A[[p, r]]
        others = np.nonzero(A[:, c])[0]
        others = others[others != r]
        A[others] ^= A[r]
        r += 1
        if r == A.shape[0]:
            break
    return r


def dense_P(H):
    """P = H_p^-1 H_s over GF(2) as an (m, k) uint8 array, or None when H_p is singular"""
    Hd = np.asarray(_csr(H).todense(), dtype=np.uint8) % 2
    m, n = Hd.shape
    k = n - m
    A = np.concatenate([Hd[:, k:], Hd[:, :k]], axis=1)
    for c in range(m):
        nz = np.nonzero(A[c:, c])[0]
        if len(nz) == 0:
            return None
        p = c + nz[0]
        A[[c, p]] = A[[p, c]]
        others = np.nonzero(A[:, c])[0]
        others = others[others != c]
        A[others] ^= A[c]
    return A[:, m:].copy()


def plan(H, force_dense=False):
    """(form, order, pivot, P) as cpb_ldpc_encoder_plan describes it; raises ValueError for a singular H_p and
    NotImplementedError for a code that neither peels nor fits the dense bound"""
    m, n = H.shape
    k = n - m
    fits = k * m <= DENSE_MAX_BITS
    if not (force_dense and fits):
        pe = peel(H)
        if pe is not None:
            return PEELED, pe[0], pe[1], None
    if not fits:
        raise NotImplementedError("H_p does not peel and k m exceeds the dense bound")
    P = dense_P(H)
    if P is None:
        raise ValueError("H_p is singular over GF(2)")
    return DENSE, np.arange(m), np.arange(m), P


def encode(H, msg, force_dense=False):
    """(batch, n) uint8 code words of the (batch, k) messages by the form plan() picks"""
    H = _csr(H)
    m, n = H.shape
    k = n - m
    msg = np.asarray(msg, dtype=np.uint8) % 2
    form, order, pivot, P = plan(H, force_dense)
    if form == DENSE:
        par = (msg.astype(np.int64) @ P.T.astype(np.int64)) % 2
    else:
        Hs = H[:, :k]
        s = np.asarray((Hs @ msg.T.astype(np.int64))).T % 2              # (batch, m) syndrome of the message part
        par = np.zeros((msg.shape[0], m), dtype=np.int64)
        for i, j in zip(order, pivot):
            cols = H.indices[H.indptr[i]:H.indptr[i + 1]]
            others = cols[(cols >= k) & (cols != k + j)] - k
            par[:, j] = (s[:, i] + par[:, others].sum(axis=1)) % 2
    return np.concatenate([msg, par.astype(np.uint8)], axis=1)


def library_plan(H, force_dense=False):
    """cpb_ldpc_encoder_plan of the built library (host only, no device): (form, order, pivot, P as (m, k) uint8)"""
    import ctypes as C
    from commpy_b200 import _lib
    H = _csr(H)
    m, n = H.shape
    k = n - m
    rp = np.ascontiguousarray(H.indptr, dtype=np.int32)
    ci = np.ascontiguousarray(H.indices, dtype=np.int32)
    form = C.c_int(-1)
    order = np.zeros(m, np.int32)
    pivot = np.zeros(m, np.int32)
    kw = (k + 31) // 32
    Pw = np.zeros((m, kw), np.uint32)
    rc = _lib.load().cpb_ldpc_encoder_plan(_lib.ptr(rp), _lib.ptr(ci), m, n, int(force_dense), C.byref(form), _lib.ptr(order),
                                           _lib.ptr(pivot), _lib.ptr(Pw))
    _lib.check(rc, "ldpc_encoder_plan")
    P = None
    if form.value == DENSE:
        P = ((Pw[:, np.arange(k) // 32] >> (np.arange(k) % 32).astype(np.uint32)) & 1).astype(np.uint8)
    return form.value, order, pivot, P

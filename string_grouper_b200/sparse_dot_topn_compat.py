"""CUDA stand-ins for the two callables the reference imports from `sparse_dot_topn`
(string_grouper/string_grouper.py:12), with the keyword usage of its call sites (:725-732, :737-743, :746):

    from string_grouper_b200.sparse_dot_topn_compat import sp_matmul_topn, zip_sp_matmul_topn

A maintainer who only wants the product on the GPU changes that one import line; `_build_matches` keeps its own
block loop (`define_chunks`, `Bi.T`, zip, vstack) and every block product / merge runs in libsg_b200.so.  scipy CSR
in, scipy CSR out (fresh numpy arrays), errors as Python exceptions; there is no CPU fallback.

Semantics (SURVEY.md Appendix A.3 / A.4): per row of A the `top_n` largest entries of A·B strictly above
`threshold`; `sort=True` orders a row by descending value (ties: ascending column), `sort=False` leaves the order
unspecified upstream — the same value-descending rows are returned.  Among EQUAL values at the top-n cut the larger
column is kept (what the upstream first-touch / reverse-block traversals yield for identical rows).
`threshold=None` means "no threshold": supported for non-negative operands, where it equals "strictly positive".
Any float32 / float64 matrix is accepted: it is made canonical first (duplicate entries summed, indices sorted, stored
zeros dropped, as scipy's own product sees it), and the result is that of the exact product.  Refused up front:
NaN / infinite values and nonzero magnitudes outside [2^-50, 2^50] (ValueError); operands with negative values with
`threshold=None` or a negative one (NotImplementedError) or below CAND_MARGIN * max(1, product of the largest row
norms) (ValueError), where a positive score could cancel in the approximate candidate stage.
"""
import ctypes

import numpy as np
from scipy.sparse import csr_matrix, issparse

from . import _device, _lib


def _check_pair(A, B):
    if not (issparse(A) and issparse(B)):
        raise TypeError("A and B must be scipy sparse matrices")
    if A.shape[1] != B.shape[0]:
        raise ValueError("shape mismatch: A is %r, B is %r" % (A.shape, B.shape))
    if A.dtype != B.dtype:
        raise TypeError("A and B must have the same dtype")
    if A.dtype not in (np.float32, np.float64):
        raise TypeError("the device path supports float32 and float64 matrices, got %s" % A.dtype)


def _to_csr(M, out_dtype, idx_dtype):
    """DeviceMatches -> scipy CSR in storage order (rows value-descending), fresh arrays."""
    r, c, s = M.host_triples()
    n_rows = M.shape[0]
    indptr = np.zeros(n_rows + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=n_rows), out=indptr[1:])
    if idx_dtype is None:
        idx_dtype = np.int32 if max(M.shape) < 2**31 and len(r) < 2**31 else np.int64
    return csr_matrix((s.astype(out_dtype), c.astype(idx_dtype), indptr.astype(idx_dtype)), shape=M.shape)


def sp_matmul_topn(A, B, top_n, threshold=None, sort=False, density=None, n_threads=None, idx_dtype=None):
    """C = A·B keeping per row of A the `top_n` largest entries strictly above `threshold`.

    `B` is (features x right rows) — the reference passes the transpose `Bi.T` of a CSR block (:727, :738).
    `density` and `n_threads` are accepted for signature compatibility and ignored (the product runs on the GPU)."""
    _check_pair(A, B)
    _device.require_cuda()
    A = A.tocsr()
    Bt = B.T.tocsr()                  # right rows x features: the layout the reference started from
    top_n = int(min(int(top_n), B.shape[1]))
    if top_n <= 0 or A.shape[0] == 0 or B.shape[1] == 0:
        return csr_matrix((A.shape[0], B.shape[1]), dtype=A.dtype)
    if threshold is None or threshold < 0:
        # candidates are the pairs with a positive partial score: complete only when no product can be negative
        if (A.nnz and A.data.min() < 0) or (Bt.nnz and Bt.data.min() < 0):
            raise NotImplementedError("threshold=None / a negative threshold with negative stored values is not "
                                      "supported by the device path")
        threshold = -np.inf if threshold is None else threshold
    Ad = _device.DeviceCSR.from_scipy(A)
    Bd = _device.DeviceCSR.from_scipy(Bt)
    M = _device.cossim_topn(Ad, Bd, top_n, float(threshold))
    return _to_csr(M, A.dtype, idx_dtype)


def zip_sp_matmul_topn(top_n, C_mats):
    """Per-row top-n merge of the results of column blocks (K3, sg_topn_merge): block b's columns are offset by the
    widths of the blocks before it; exact zeros / negatives are dropped like upstream's heap does."""
    C_mats = [c.tocsr() for c in C_mats]
    if not C_mats:
        raise ValueError("C_mats is empty")
    n_rows = C_mats[0].shape[0]
    if any(c.shape[0] != n_rows for c in C_mats):
        raise ValueError("all C_mats must have the same number of rows")
    dtype = C_mats[0].dtype
    if dtype not in (np.float32, np.float64):
        raise TypeError("the device path supports float32 and float64 matrices, got %s" % dtype)
    t = _device.require_cuda()
    L = _lib.load()
    widths = np.array([c.shape[1] for c in C_mats], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(widths)[:-1]])
    shape = (n_rows, int(widths.sum()))
    if shape[1] >= 2**31:
        raise OverflowError("merged matrix has %d columns; int32 column ids overflow" % shape[1])
    rows = np.concatenate([np.repeat(np.arange(n_rows, dtype=np.int32), np.diff(c.indptr)) for c in C_mats])
    cols = np.concatenate([(c.indices.astype(np.int64) + o).astype(np.int32) for c, o in zip(C_mats, offs)])
    vals = np.concatenate([c.data.astype(np.float64) for c in C_mats])
    n = len(rows)
    top_n = int(top_n)
    if n == 0 or top_n <= 0:
        return csr_matrix(shape, dtype=dtype)
    dev = t.device("cuda", t.cuda.current_device())
    d_row, d_col, d_val = (t.from_numpy(x).to(dev) for x in (rows, cols, vals))
    out_indptr = t.empty(n_rows + 1, dtype=t.int64, device=dev)
    out_row = t.empty(n, dtype=t.int32, device=dev)
    out_col = t.empty(n, dtype=t.int32, device=dev)
    out_val = t.empty(n, dtype=t.float64, device=dev)
    tail = t.zeros(2, dtype=t.int64, device=dev)
    ws_bytes = int(L.sg_topn_merge_workspace_bytes(n, n_rows))
    ws = t.empty(max(ws_bytes, 1), dtype=t.uint8, device=dev)
    dt = _lib.SG_DTYPE_F32 if dtype == np.float32 else _lib.SG_DTYPE_F64
    p = lambda x: ctypes.c_void_p(x.data_ptr())     # noqa: E731
    _lib.check(L.sg_topn_merge(n, p(d_row), p(d_col), p(d_val), n_rows, top_n, dt, p(out_indptr), p(out_row),
                               p(out_col), p(out_val), ctypes.c_void_p(tail.data_ptr()),
                               ctypes.c_void_p(tail.data_ptr() + 8), p(ws), ws_bytes,
                               ctypes.c_void_p(t.cuda.current_stream().cuda_stream)))
    _device.LAUNCH_COUNTS["select"] += 7
    nnz = int(tail[0].item())
    M = _device.DeviceMatches(shape, out_row, out_col, out_val, nnz, 0)
    return _to_csr(M, dtype, None)

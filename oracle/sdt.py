"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

Python face of the C oracle (`oracle/sdt_oracle.c`): the two callables the
reference imports from the absent third-party package `sparse_dot_topn`
(string_grouper/string_grouper.py:12), with the keyword
signatures the reference uses at :725-732, :737-743 and :746.

`oracle/standin/sparse_dot_topn/` re-exports these under the upstream module
name so that the UNMODIFIED reference can be imported by the golden-vector
generator and by the reference-suite pin test.
"""
import ctypes
import os
import subprocess

import numpy as np
from scipy.sparse import csr_matrix, issparse

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build():
    """Compile the C restatement (gcc + OpenMP); idempotent."""
    so = os.path.join(_HERE, "libsg_oracle.so")
    src = os.path.join(_HERE, "sdt_oracle.c")
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def _lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        i64, p = ctypes.c_int64, ctypes.c_void_p
        for name in ("sgo_sp_matmul_topn_f64", "sgo_sp_matmul_topn_f32"):
            f = getattr(L, name)
            f.restype = i64
            f.argtypes = [i64, i64, i64, ctypes.c_double, ctypes.c_int, ctypes.c_int,
                          p, p, p, p, p, p, p, p, p]
        L.sgo_zip_topn_f64.restype = i64
        L.sgo_zip_topn_f64.argtypes = [i64, i64, i64, p, p, p, p, ctypes.c_int, p, p, p]
        L.sgo_max_threads.restype = ctypes.c_int
        _LIB = L
    return _LIB


def max_threads():
    return int(_lib().sgo_max_threads())


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _pack_rows(nrows, top_n, row_cnt, out_idx, out_val, shape, dtype):
    indptr = np.zeros(nrows + 1, dtype=np.int64)
    np.cumsum(row_cnt, out=indptr[1:])
    keep = (np.arange(top_n, dtype=np.int64)[None, :] < row_cnt[:, None]).ravel()
    idx = out_idx[keep]
    val = out_val[keep].astype(dtype, copy=False)
    idx_dtype = np.int32 if max(shape) < 2**31 and indptr[-1] < 2**31 else np.int64
    return csr_matrix((val, idx.astype(idx_dtype), indptr.astype(idx_dtype)), shape=shape)


def sp_matmul_topn(A, B, top_n, threshold=None, sort=False, density=None, n_threads=None,
                   idx_dtype=None):
    """C = A·B keeping, per row of A, the `top_n` largest entries strictly above
    `threshold` (SURVEY.md Appendix A.3).  `B` is (features × right rows); the
    reference passes the CSC transpose `Bi.T` (string_grouper.py:727, :738)."""
    if not (issparse(A) and issparse(B)):
        raise TypeError("A and B must be scipy sparse matrices")
    if A.shape[1] != B.shape[0]:
        raise ValueError("shape mismatch: A is %r, B is %r" % (A.shape, B.shape))
    A = A.tocsr()
    B = B.tocsr()
    if A.dtype != B.dtype:
        raise TypeError("A and B must have the same dtype")
    if A.dtype == np.float32:
        fn, ct = _lib().sgo_sp_matmul_topn_f32, np.float32
    elif A.dtype == np.float64:
        fn, ct = _lib().sgo_sp_matmul_topn_f64, np.float64
    else:
        raise TypeError("only float32 / float64 are supported by this oracle")
    nrows, ncols = A.shape[0], B.shape[1]
    top_n = int(min(int(top_n), ncols))
    if threshold is None:
        threshold = float(np.finfo(ct).min)
    nt = 1 if (n_threads is None or n_threads <= 1) else int(n_threads)
    a_ip = np.ascontiguousarray(A.indptr, dtype=np.int64)
    a_ix = np.ascontiguousarray(A.indices, dtype=np.int64)
    a_v = np.ascontiguousarray(A.data, dtype=ct)
    b_ip = np.ascontiguousarray(B.indptr, dtype=np.int64)
    b_ix = np.ascontiguousarray(B.indices, dtype=np.int64)
    b_v = np.ascontiguousarray(B.data, dtype=ct)
    tn = max(top_n, 1)
    row_cnt = np.zeros(nrows, dtype=np.int64)
    out_idx = np.empty(nrows * tn, dtype=np.int64)
    out_val = np.empty(nrows * tn, dtype=np.float64)
    rc = fn(nrows, ncols, top_n, float(threshold), int(bool(sort)), nt,
            _ptr(a_ip), _ptr(a_ix), _ptr(a_v), _ptr(b_ip), _ptr(b_ix), _ptr(b_v),
            _ptr(row_cnt), _ptr(out_idx), _ptr(out_val))
    if rc < 0:
        raise MemoryError("oracle sp_matmul_topn: allocation failed")
    return _pack_rows(nrows, tn, row_cnt, out_idx, out_val, (nrows, ncols), ct)


def zip_sp_matmul_topn(top_n, C_mats):
    """Per-row top-n merge of column-block results (SURVEY.md Appendix A.4)."""
    C_mats = [c.tocsr() for c in C_mats]
    if not C_mats:
        raise ValueError("C_mats is empty")
    nrows = C_mats[0].shape[0]
    if any(c.shape[0] != nrows for c in C_mats):
        raise ValueError("all C_mats must have the same number of rows")
    dtype = C_mats[0].dtype
    widths = np.array([c.shape[1] for c in C_mats], dtype=np.int64)
    offs = np.zeros(len(C_mats), dtype=np.int64)
    offs[1:] = np.cumsum(widths)[:-1]
    ips = [np.ascontiguousarray(c.indptr, dtype=np.int64) for c in C_mats]
    ixs = [np.ascontiguousarray(c.indices, dtype=np.int64) for c in C_mats]
    vs = [np.ascontiguousarray(c.data, dtype=np.float64) for c in C_mats]
    P = ctypes.c_void_p * len(C_mats)
    top_n = int(top_n)
    tn = max(top_n, 1)
    row_cnt = np.zeros(nrows, dtype=np.int64)
    out_idx = np.empty(nrows * tn, dtype=np.int64)
    out_val = np.empty(nrows * tn, dtype=np.float64)
    rc = _lib().sgo_zip_topn_f64(
        nrows, top_n, len(C_mats),
        P(*[a.ctypes.data for a in ips]), P(*[a.ctypes.data for a in ixs]),
        P(*[a.ctypes.data for a in vs]), _ptr(offs), int(dtype == np.float32),
        _ptr(row_cnt), _ptr(out_idx), _ptr(out_val))
    if rc < 0:
        raise MemoryError("oracle zip_sp_matmul_topn: allocation failed")
    return _pack_rows(nrows, tn, row_cnt, out_idx, out_val, (nrows, int(widths.sum())), dtype)

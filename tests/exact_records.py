"""match_records as a specification: CPU references the CUDA results must equal bit for bit.

* `field_matrices`: per field, the reference's own vectoriser on that column (oracle.pipeline.tf_idf_matrices),
  missing values read as "".
* `stack`: every field's values times sqrt(w_k / sum w) (float64; rounded to float32 for float32 matrices), one
  rounding in the matrix dtype, the fields side by side in field order.
* `exact_record_list`: the exact top-n product of the stacked matrices (tests/exact_topn.py) and, for a self-match,
  the reference's fix-diagonal / symmetrise, as tests/exact_pipeline.exact_match_list does for one column.
* `pair_scores`: field k's score of listed pairs, the products of the common features added left to right in
  ascending feature order in the matrix dtype — scipy's A_k @ B_k.T, as tests/test_exact_topn.py pins it.

numpy / scipy / scikit-learn only: no GPU.
"""
import numpy as np
import pandas as pd
from scipy.sparse import csr_matrix, hstack

from exact_topn import exact_topn, to_csr


def filled(col):
    return ["" if (x is None or (not isinstance(x, str) and pd.isna(x))) else x for x in col]


def scales(weights, dtype):
    w = np.asarray(list(weights.values()), dtype=np.float64)
    s = np.sqrt(w / w.sum())
    return s.astype(np.float32) if np.dtype(dtype) == np.float32 else s


def field_matrices(master, duplicates, weights, dtype=np.float64, **tfidf_kw):
    """[(M_k, D_k)] per field (D_k = M_k for a self-match)"""
    from oracle import pipeline as P
    out = []
    for f in weights:
        m = pd.Series(filled(master[f]))
        d = None if duplicates is None else pd.Series(filled(duplicates[f]))
        M, D, _ = P.tf_idf_matrices(m, d, dtype=dtype, **tfidf_kw)
        out.append((csr_matrix(M), csr_matrix(D)))
    return out


def stack(mats, scale):
    """the fields side by side, field k's values times scale[k] in the matrix dtype"""
    parts = []
    for m, s in zip(mats, scale):
        m = csr_matrix(m, copy=True)
        m.data = m.data * m.dtype.type(s)
        parts.append(m)
    return csr_matrix(hstack(parts, format="csr", dtype=parts[0].dtype))


def pair_scores(A, B, rows, cols):
    """float64 score of every pair (rows[i], cols[i]) of A @ B.T, summed left to right in the matrix dtype"""
    A, B = csr_matrix(A), csr_matrix(B)
    P = csr_matrix(A[np.asarray(rows, np.int64)].multiply(B[np.asarray(cols, np.int64)]), dtype=A.dtype)
    P.sort_indices()
    n = np.diff(P.indptr)
    acc = np.zeros(P.shape[0], dtype=A.dtype)
    for j in range(int(n.max()) if len(n) else 0):
        live = np.flatnonzero(n > j)
        acc[live] = acc[live] + P.data[P.indptr[live] + j]
    return acc.astype(np.float64)


def exact_record_list(master, duplicates=None, *, weights, dtype=np.float64, max_n_matches=20, min_similarity=0.8,
                      **tfidf_kw):
    """(matches_list frame with similarity_<f> columns, true_max_n_matches, (fields, stacked M, stacked D))"""
    from oracle import pipeline as P
    fields = field_matrices(master, duplicates, weights, dtype, **tfidf_kw)
    sc = scales(weights, dtype)
    M = stack([m for m, _ in fields], sc)
    D = M if duplicates is None else stack([d for _, d in fields], sc)
    top_n = min(int(max_n_matches), D.shape[0])
    r, c, s, max_row = exact_topn(M, D, top_n, min_similarity)
    C = to_csr((r, c, s), (M.shape[0], D.shape[0]))
    if duplicates is None:
        C = P.fix_diagonal_and_symmetrize(C)
    ml = P.matches_list(C)
    if duplicates is not None and np.dtype(dtype) == np.float32:
        # the reference's vstack(..., dtype=np.float64) (string_grouper.py:750) re-orders a float32 product's rows by
        # column, as match_strings does
        ml = ml.sort_values(["master_side", "dupe_side"], kind="stable").reset_index(drop=True)
    for f, (A, B) in zip(weights, fields):
        ml["similarity_%s" % f] = pair_scores(A, B, ml.master_side.to_numpy(), ml.dupe_side.to_numpy())
    return ml, max_row, (fields, M, D)

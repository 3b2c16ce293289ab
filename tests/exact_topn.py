"""The top-n product as a specification: a CPU reference of K2 / K3 that the CUDA results must equal bit for bit.

`exact_topn(A, B, top_n, threshold)` is what DESIGN.md §2 / §4 promise for `cossim_topn(A, B, top_n, threshold)`:

* scores: S = A @ B.T in the matrix dtype (scipy adds the products of a pair left to right in ascending feature
  order without FMA, which is the order of the re-score kernel; tests/test_exact_topn.py pins this), widened to
  float64;
* only pairs with s > threshold (strictly) count;
* per row the `top_n` best by (score descending, column descending): among equal scores the larger column wins;
* a row is written score-descending, equal scores in ascending column order.

Returns (row, col, score, max_row) like `DeviceMatches.host_triples()` plus `DeviceMatches.max_row` (the largest
number of entries kept in one row).  numpy / scipy only: no GPU, no oracle.
"""
import numpy as np
from scipy.sparse import csr_matrix


def exact_pairs(A, B, threshold, block_rows=1024):
    """(row, col, score) of every pair of A @ B.T strictly above `threshold` (row-major order).

    A: left rows x features, B: right rows x features, both scipy sparse of the same dtype.  The product is formed in
    row blocks and thresholded block by block, so that 10-20 k rows against as many columns fit in memory."""
    A = csr_matrix(A)
    B = csr_matrix(B)
    if A.dtype != B.dtype:
        raise TypeError("A and B must have the same dtype")
    if not A.has_sorted_indices:
        A = A.sorted_indices()  # the accumulation order is the stored order of A's row
    Bt = B.T.tocsr()
    rows, cols, scores = [], [], []
    for lo in range(0, A.shape[0], block_rows):
        S = (A[lo:lo + block_rows] @ Bt).tocoo()
        s = S.data.astype(np.float64)
        keep = s > threshold
        rows.append(S.row[keep].astype(np.int64) + lo)
        cols.append(S.col[keep].astype(np.int64))
        scores.append(s[keep])
    if not rows:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float64)
    r, c, s = np.concatenate(rows), np.concatenate(cols), np.concatenate(scores)
    o = np.lexsort((c, r))
    return r[o], c[o], s[o]


class RankedPairs:
    """Scored pairs sorted once into output order, each with its rank inside its row.

    The rank of a pair (its position by (score descending, column descending) among the pairs of its row) does not
    change when a threshold drops pairs, because every pair that beats it has a score at least as large.  So the
    result for any (top_n, threshold) at or above the threshold the pairs were collected with is a mask:
    score > threshold and rank < top_n, already in output order."""

    def __init__(self, row, col, score):
        row, col, score = (np.asarray(x) for x in (row, col, score))
        row, col, score = row.astype(np.int64), col.astype(np.int64), score.astype(np.float64)
        o = np.lexsort((-col, -score, row))
        row, col, score = row[o], col[o], score[o]
        start = np.flatnonzero(np.r_[True, row[1:] != row[:-1]]) if len(row) else np.zeros(0, np.int64)
        length = np.diff(np.r_[start, len(row)])
        rank = np.arange(len(row)) - np.repeat(start, length)
        # written by score descending, equal scores in ascending column order
        o = np.lexsort((col, -score, row))
        self.row, self.col, self.score, self.rank = row[o], col[o], score[o], rank[o]

    def topn(self, top_n, threshold=-np.inf, rows=None):
        """(row, col, score, max_row); `rows` = (begin, end) keeps only those left rows (a shard)"""
        keep = (self.score > threshold) & (self.rank < top_n)
        if rows is not None:
            keep &= (self.row >= rows[0]) & (self.row < rows[1])
        max_row = int(self.rank[keep].max()) + 1 if keep.any() else 0
        return self.row[keep], self.col[keep], self.score[keep], max_row


def topn_from_pairs(row, col, score, top_n, threshold=-np.inf):
    """The cut and the output order applied to a list of scored pairs (each (row, col) at most once)."""
    return RankedPairs(row, col, score).topn(top_n, threshold)


def exact_topn(A, B, top_n, threshold, block_rows=1024):
    """Reference of `cossim_topn(A, B, top_n, threshold)` over all rows of A; see the module docstring."""
    r, c, s = exact_pairs(A, B, threshold, block_rows)
    return topn_from_pairs(r, c, s, top_n)


def exact_zip(top_n, blocks):
    """Reference of `zip_sp_matmul_topn(top_n, blocks)` (K3): block b's columns are offset by the widths of the
    blocks before it, values that are not strictly positive are dropped, then the same cut and order."""
    rows, cols, vals = [], [], []
    off = 0
    for b in blocks:
        b = csr_matrix(b)
        rows.append(np.repeat(np.arange(b.shape[0], dtype=np.int64), np.diff(b.indptr)))
        cols.append(b.indices.astype(np.int64) + off)
        vals.append(b.data.astype(np.float64))
        off += b.shape[1]
    return topn_from_pairs(np.concatenate(rows), np.concatenate(cols), np.concatenate(vals), top_n, 0.0)


def to_csr(triples, shape):
    """(row, col, score[, max_row]) -> float64 CSR in the given storage order (for K4 references)."""
    r, c, s = triples[:3]
    indptr = np.zeros(shape[0] + 1, dtype=np.int64)
    np.cumsum(np.bincount(r, minlength=shape[0]), out=indptr[1:])
    return csr_matrix((np.asarray(s, np.float64), np.asarray(c), indptr), shape=shape)


def assert_same(got, want, label=""):
    """Whole outputs equal: rows, columns, scores (bit for bit) and, when both carry it, max_row."""
    names = ("row", "col", "score", "max_row")
    for name, g, w in zip(names, got, want):
        if name == "max_row":
            assert int(g) == int(w), "%s: max_row %d != %d" % (label, g, w)
            continue
        g, w = np.asarray(g), np.asarray(w)
        if g.shape == w.shape and np.array_equal(g, w):
            continue
        n = min(len(g), len(w))
        bad = np.flatnonzero(g[:n] != w[:n])
        first = int(bad[0]) if len(bad) else n
        raise AssertionError("%s: %s differs (%d vs %d entries; first difference at %d: got %s, want %s)" % (
            label, name, len(g), len(w), first,
            [(int(got[0][i]), int(got[1][i]), float(got[2][i])) for i in range(first, min(first + 3, len(g)))],
            [(int(want[0][i]), int(want[1][i]), float(want[2][i])) for i in range(first, min(first + 3, len(w)))]))

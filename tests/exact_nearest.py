"""The arg-max product as a specification: what `cossim_nearest(A, B, threshold)` (match_nearest's kernel path,
DESIGN.md §4 "Nearest row") must return bit for bit.  It extends tests/exact_topn.py: the same exact scores, the same
strict threshold, but per row the single pair of largest score with the SMALLEST column among equal scores (the
top-n cut keeps the larger one).

Returns (best int64 [n_left], -1 for a row without a pair above the threshold; score float64 [n_left], 0 there).
"""
import numpy as np

from exact_topn import exact_pairs


def nearest_from_pairs(row, col, score, n_rows):
    """per row: score descending, then column ascending; the first pair"""
    row, col, score = (np.asarray(x) for x in (row, col, score))
    best = np.full(n_rows, -1, dtype=np.int64)
    best_score = np.zeros(n_rows, dtype=np.float64)
    if len(row):
        o = np.lexsort((col, -score, row))
        first = o[np.r_[True, row[o][1:] != row[o][:-1]]]
        best[row[first]] = col[first]
        best_score[row[first]] = score[first]
    return best, best_score


def exact_nearest(A, B, threshold, block_rows=1024):
    """Reference of `cossim_nearest(A, B, threshold)`: threshold <= 0 keeps the pairs the product stores (score > 0
    for the non-negative TF-IDF matrices)."""
    r, c, s = exact_pairs(A, B, threshold, block_rows)
    return nearest_from_pairs(r, c, s, A.shape[0])


def exact_nearest_many(A, B, thresholds, block_rows=128):
    """{threshold: exact_nearest(A, B, threshold)} from one pass over the product (large right matrices: the pairs of
    a block of rows are reduced before the next block is formed)."""
    out = {thr: (np.full(A.shape[0], -1, dtype=np.int64), np.zeros(A.shape[0])) for thr in thresholds}
    for lo in range(0, A.shape[0], block_rows):
        hi = min(lo + block_rows, A.shape[0])
        r, c, s = exact_pairs(A[lo:hi], B, min(thresholds), block_rows)
        for thr in thresholds:
            keep = s > thr
            best, score = nearest_from_pairs(r[keep], c[keep], s[keep], hi - lo)
            out[thr][0][lo:hi], out[thr][1][lo:hi] = best, score
    return out

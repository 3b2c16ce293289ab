"""The pipeline from strings to matches as a specification: CPU references the CUDA results must equal bit for bit.

* `exact_match_list(master, duplicates, ...)`: scikit-learn's TF-IDF matrices (the reference's own vectoriser,
  oracle.pipeline.tf_idf_matrices), the exact top-n product of tests/exact_topn.py, then for a self-match the
  reference's LIL fix-diagonal / symmetrise.  Returns the match list frame and `_true_max_n_matches`.
* `rowwise_dot(M, D)`: `M.multiply(D).sum(axis=1)` (the reference's `dot()`) restated in Python: the products of
  the common features in ascending order, in the matrix dtype, reduced as scipy reduces a row (`np.add.reduceat`):
  p0 + numpy's pairwise sum of p1..pk-1.  tests/test_exact_pipeline_math.py pins this against scipy itself.

numpy / scipy / scikit-learn only: no GPU.
"""
import numpy as np
from scipy.sparse import csr_matrix

from exact_topn import exact_topn, to_csr
from synth_corpus import make_names

PW_BLOCKSIZE = 128      # numpy's pairwise-sum block (numpy/_core/src/umath/loops_utils.h.src)


def pairwise_sum(a):
    """numpy's pairwise sum of the 1-d array `a` in its own dtype: a plain loop below 8 terms; up to PW_BLOCKSIZE
    eight accumulators over the multiple of 8, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest one by
    one; above, n2 = n/2 rounded down to a multiple of 8 and the two halves added."""
    n = len(a)
    zero = a.dtype.type(0)
    if n < 8:
        res = zero
        for x in a:
            res = res + x
        return res
    if n <= PW_BLOCKSIZE:
        r = list(a[:8])
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = r[j] + a[i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for x in a[i:]:
            res = res + x
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


def common_products(M, D, i):
    """Products of row i of M and D over their common features, ascending feature order, in the matrix dtype."""
    a = slice(M.indptr[i], M.indptr[i + 1])
    b = slice(D.indptr[i], D.indptr[i + 1])
    _, ia, ib = np.intersect1d(M.indices[a], D.indices[b], assume_unique=True, return_indices=True)
    return M.data[a][ia] * D.data[b][ib]


def rowwise_dot(M, D):
    """`M.multiply(D).sum(axis=1)` as a 1-d array in the matrix dtype, summed in scipy's order."""
    M, D = csr_matrix(M).sorted_indices(), csr_matrix(D).sorted_indices()
    out = np.zeros(M.shape[0], dtype=M.dtype)
    for i in range(M.shape[0]):
        p = common_products(M, D, i)
        p = p[p != 0]                      # scipy's element-wise product stores no zeros
        if len(p):
            out[i] = p[0] + pairwise_sum(p[1:]) if len(p) > 1 else p[0]
    return out


def distinct_ngram_word(k, rng, n=3, alphabet="abcdefghijklmnopqrstuvwxyz"):
    """k + n - 1 letters whose k n-grams are all different"""
    while True:
        w = list(rng.choice(list(alphabet), n - 1))
        seen = set()
        for _ in range(k):
            stem = "".join(w[len(w) - n + 1:])
            options = [c for c in alphabet if stem + c not in seen]
            if not options:
                break
            c = options[rng.integers(len(options))]
            seen.add(stem + c)
            w.append(c)
        if len(seen) == k:
            return "".join(w)


COMMON_COUNTS = [0, 1, 2, 7, 8, 9, 16, 17, 128, 129, 130, 137, 257, 300, 1000, 3000]


def common_count_pairs(seed=0):
    """(left, right) string lists whose row i shares exactly COMMON_COUNTS[i] trigrams, then 3 000 make_names rows
    (half of them identical on both sides).  The shared part is letters; each side adds digits of its own (0-4 on the
    left, 5-9 on the right), so no other trigram is common."""
    rng = np.random.default_rng(seed)
    left, right = [], []
    for k in COMMON_COUNTS:
        w = distinct_ngram_word(k, rng) if k else ""
        left.append(w + "".join(rng.choice(list("01234"), int(rng.integers(3, 40)))))
        right.append(w + "".join(rng.choice(list("56789"), int(rng.integers(3, 40)))))
    names = make_names(3000, seed=seed + 7)
    other = make_names(3000, seed=seed + 8)
    return left + names, right + names[:1500] + other[1500:]


def exact_match_list(master, duplicates=None, *, ngram_size=3, dtype=np.float64, max_n_matches=20,
                     min_similarity=0.8, **tfidf_kw):
    """(matches_list frame, true_max_n_matches, (M, D, vectoriser)) of StringGrouper(master, duplicates).fit() in
    the reference: sklearn matrices, exact top-n product, and for a self-match diagonal := 1 and the symmetric
    pattern (string_grouper.py:419-427)."""
    from oracle import pipeline as P
    M, D, vec = P.tf_idf_matrices(master, duplicates, ngram_size=ngram_size, dtype=dtype, **tfidf_kw)
    top_n = min(int(max_n_matches), D.shape[0])
    r, c, s, max_row = exact_topn(M, D, top_n, min_similarity)
    C = to_csr((r, c, s), (M.shape[0], D.shape[0]))
    if duplicates is None:
        C = P.fix_diagonal_and_symmetrize(C)
    return P.matches_list(C), max_row, (M, D, vec)

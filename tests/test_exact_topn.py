"""The exact top-n reference (tests/exact_topn.py) pinned on its own, without a GPU: the tie rule and output order on
hand-built matrices (the written specification), agreement with the oracle of sparse_dot_topn, and the claim that its
scores are the ascending-feature sums without FMA that the re-score kernel computes."""
import math

import numpy as np
import pytest
from scipy.sparse import csr_matrix

from exact_topn import assert_same, exact_pairs, exact_topn, exact_zip, topn_from_pairs
from parity import compare_triples, csr_triples, row_cutoffs
from synth_corpus import make_names


def _dyadic(rows, n_features):
    """rows: lists of features, every stored weight 0.5 (four features: norm 1)"""
    indptr = np.cumsum([0] + [len(r) for r in rows])
    idx = np.concatenate([sorted(r) for r in rows]).astype(np.int32)
    return csr_matrix((np.full(len(idx), 0.5), idx, indptr), shape=(len(rows), n_features))


def test_identical_rows_keep_the_largest_columns_written_ascending():
    """6 identical rows, top_n = 3: every row keeps columns 3, 4, 5 (the larger column wins among equal scores),
    written in ascending column order."""
    A = _dyadic([[0, 1, 2, 3]] * 6, 8)
    r, c, s, mx = exact_topn(A, A, 3, 0.5)
    assert np.array_equal(r, np.repeat(np.arange(6), 3))
    assert np.array_equal(c, np.tile([3, 4, 5], 6))
    assert np.all(s == 1.0) and mx == 3


def test_order_threshold_and_short_rows():
    # row 0 against rows 0..4: scores 1, 0.75, 0.5, 0.75, 0.25
    A = _dyadic([[0, 1, 2, 3], [0, 1, 2, 4], [0, 1, 5, 6], [1, 2, 3, 7], [3, 8, 9, 10]], 11)
    r, c, s, mx = exact_topn(A[:1], A, 10, 0.25)
    assert np.array_equal(c, [0, 1, 3, 2]) and np.array_equal(s, [1.0, 0.75, 0.75, 0.5])
    assert np.all(r == 0) and mx == 4
    # strict threshold: a score equal to it is out, the next double below lets it in
    r, c, s, _ = exact_topn(A[:1], A, 10, 0.75)
    assert np.array_equal(c, [0])
    r, c, s, _ = exact_topn(A[:1], A, 10, np.nextafter(0.75, -np.inf))
    assert np.array_equal(c, [0, 1, 3])
    # the cut inside a tie: of the two 0.75, column 3 wins; written score-descending
    r, c, s, mx = exact_topn(A[:1], A, 2, 0.0)
    assert np.array_equal(c, [0, 3]) and mx == 2
    # -inf: every stored product, rows without any pair produce nothing
    B = _dyadic([[20, 21, 22, 23]], 24)
    A24 = csr_matrix((A.data, A.indices, A.indptr), shape=(5, 24))
    r, c, s, mx = exact_topn(A24, B, 5, -np.inf)
    assert len(r) == 0 and mx == 0


def test_zip_reference_offsets_and_drops_non_positive():
    b0 = csr_matrix(np.array([[0.5, 0.0, 0.25], [0.0, 0.0, 0.0]]))
    # row 0: 0.5 at merged column 3, -1.0 at 4; row 1: an explicitly stored zero at 3, 0.5 at 4
    b1 = csr_matrix((np.array([0.5, -1.0, 0.0, 0.5]), np.array([0, 1, 0, 1]), np.array([0, 2, 4])), shape=(2, 2))
    r, c, s, mx = exact_zip(2, [b0, b1])
    assert np.array_equal(r, [0, 0, 1]) and np.array_equal(c, [0, 3, 4])
    assert np.array_equal(s, [0.5, 0.5, 0.5]) and mx == 2
    # ties at the cut: the larger merged column stays
    r, c, s, _ = exact_zip(1, [b0, b1])
    assert np.array_equal(c, [3, 4])


def test_topn_from_pairs_matches_a_per_row_sort():
    rng = np.random.default_rng(0)
    n = 5000
    row = rng.integers(0, 60, n)
    col = rng.permutation(100000)[:n]
    score = np.round(rng.random(n), 2)                 # many exact ties
    for top_n in (1, 3, 50, 1000):
        r, c, s, mx = topn_from_pairs(row, col, score, top_n, 0.3)
        want_r, want_c, want_s = [], [], []
        for i in range(60):
            sel = (row == i) & (score > 0.3)
            pairs = sorted(zip(score[sel], col[sel]), reverse=True)[:top_n]       # (score desc, col desc)
            pairs.sort(key=lambda p: (-p[0], p[1]))                                # written: ties col ascending
            want_r += [i] * len(pairs)
            want_c += [p[1] for p in pairs]
            want_s += [p[0] for p in pairs]
        assert np.array_equal(r, want_r) and np.array_equal(c, want_c) and np.array_equal(s, want_s)
        assert mx == max(min(((row == i) & (score > 0.3)).sum(), top_n) for i in range(60))


@pytest.fixture(scope="module")
def corpus():
    from oracle import pipeline as P
    names = make_names(3000, seed=7) + ["ACME HOLDINGS LLC"] * 30
    out = {}
    for dtype in (np.float64, np.float32):
        m, _, _ = P.tf_idf_matrices(names, dtype=dtype)
        out[dtype] = m.tocsr()
    return out


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("top_n,thr", [(20, 0.8), (5, 0.5), (50, 0.3)])
def test_equals_oracle_modulo_boundary_ties(corpus, dtype, top_n, thr):
    """Same pairs as the restatement of sparse_dot_topn except ties at the cut, and bit-equal scores on every pair
    both return: the oracle adds the products in the same order."""
    from oracle import sdt
    m = corpus[dtype]
    ref = sdt.sp_matmul_topn(m, m.T, top_n=top_n, threshold=thr, sort=True, n_threads=2)
    r, c, s, mx = exact_topn(m, m, top_n, thr)
    n = m.shape[0]
    cut = row_cutoffs(ref.indptr, ref.data.astype(np.float64), top_n, n)
    st = compare_triples(csr_triples(ref), (r, c, s), n, thr, tol=1e-5, cutoff_row=cut, label="exact vs oracle")
    assert st["max_abs_err"] == 0.0 and st["common"] > n
    assert mx == int(np.diff(ref.indptr).max())


def _sequential(a_idx, a_val, b_idx, b_val, dtype):
    """left-to-right sum over the common features in ascending order, every product and sum rounded in `dtype`"""
    common, ia, ib = np.intersect1d(a_idx, b_idx, assume_unique=True, return_indices=True)
    acc = dtype(0)
    for i, j in zip(ia, ib):
        acc = dtype(acc + dtype(a_val[i] * b_val[j]))
    return acc, [float(a_val[i]) * float(b_val[j]) for i, j in zip(ia, ib)]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_scores_are_the_ascending_sum_without_fma(corpus, dtype):
    """exact_pairs' scores equal an explicit sequential sum in ascending feature order (no FMA, every operation
    rounded in the matrix dtype) on a sample of pairs, bit for bit; against math.fsum of the exact products each
    error stays within (number of terms) x eps, i.e. the reference is the true dot product up to that rounding."""
    m = corpus[dtype]
    rows = np.arange(0, m.shape[0], 37)
    r, c, s = exact_pairs(m[rows], m, 0.0)
    assert len(r) > 2000
    eps = np.finfo(dtype).eps
    pick = np.random.default_rng(1).choice(len(r), size=min(len(r), 4000), replace=False)
    for k in pick:
        a, b = m[rows[r[k]]], m[c[k]]
        seq, products = _sequential(a.indices, a.data, b.indices, b.data, dtype)
        assert float(seq) == s[k], (k, float(seq), s[k])
        true = math.fsum(products)                # float32 products are exact in float64
        assert abs(s[k] - true) <= len(products) * eps * max(true, 1.0), (k, s[k], true)


def test_row_blocks_do_not_change_the_result(corpus):
    m = corpus[np.float64]
    a = exact_topn(m, m, 20, 0.5, block_rows=4096)
    b = exact_topn(m, m, 20, 0.5, block_rows=97)
    assert_same(a, b, "row blocks")

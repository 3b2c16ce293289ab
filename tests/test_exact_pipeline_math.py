"""not-gpu: the two host statements the exact pipeline tests rest on, pinned against scikit-learn / scipy themselves.

* `_device.sklearn_idf` (the idf K1 uploads) is bit-equal to `TfidfTransformer().fit(X).idf_`;
* `exact_pipeline.rowwise_dot` (the order `sg_rowwise_dot` sums in) is bit-equal to `M.multiply(D).sum(axis=1)`.

If numpy changes its `log` dispatch or its reduction order, these fail first, without a GPU.
"""
import os
import re

import numpy as np
import pytest
from scipy.sparse import csr_matrix

from exact_pipeline import COMMON_COUNTS, common_count_pairs, common_products, pairwise_sum, rowwise_dot
from string_grouper_b200._device import sklearn_idf

DTYPES = [np.float32, np.float64]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sklearn_idf_of(df, n, dtype, monkeypatch):
    """TfidfTransformer.fit's idf_ for document frequencies `df` over `n` documents.  The frequencies are handed to
    fit through its own `_document_frequency` hook, so that n = 663 000 needs no matrix with sum(df) entries; fit
    itself runs unchanged."""
    from sklearn.feature_extraction import text
    from sklearn.feature_extraction.text import TfidfTransformer
    monkeypatch.setattr(text, "_document_frequency", lambda X: np.asarray(df, dtype=np.int64))
    X = csr_matrix((n, len(df)), dtype=dtype)
    return TfidfTransformer().fit(X).idf_


@pytest.mark.parametrize("dtype", DTYPES)
def test_sklearn_idf_on_a_real_matrix(dtype):
    from sklearn.feature_extraction.text import TfidfTransformer
    rng = np.random.default_rng(0)
    X = csr_matrix((rng.random((500, 37)) < rng.random(37)).astype(dtype))
    X[:, 5] = 1.0                                      # a feature in every document: idf exactly 1
    X = csr_matrix(X)
    want = TfidfTransformer().fit(X).idf_
    df = np.bincount(X.indices, minlength=X.shape[1])
    got = sklearn_idf(df, X.shape[0], dtype)
    assert got.dtype == want.dtype == dtype
    assert np.array_equal(got, want) and got[5] == 1.0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n", [1, 2, 7, 1000, 20_000, 663_000])
def test_sklearn_idf_bit_equal_every_length_and_df(dtype, n, monkeypatch):
    """vocabulary lengths 1..40 (the SIMD tails of numpy's log) and 10^5, df from 1 to n"""
    rng = np.random.default_rng(n)
    for V in list(range(1, 41)) + [100_000]:
        df = rng.integers(1, n + 1, V)
        df[0] = n
        if V > 1:
            df[-1] = 1
        want = _sklearn_idf_of(df, n, dtype, monkeypatch)
        got = sklearn_idf(df, n, dtype)
        assert got.dtype == want.dtype == dtype
        assert np.array_equal(got, want), (V, np.flatnonzero(got != want)[:5])


@pytest.mark.parametrize("dtype", DTYPES)
def test_sklearn_idf_every_df_value_of_the_663k_corpus(dtype, monkeypatch):
    n = 663_000
    df = np.arange(1, n + 1)
    assert np.array_equal(sklearn_idf(df, n, dtype), _sklearn_idf_of(df, n, dtype, monkeypatch))


def test_product_package_does_not_import_sklearn():
    pkg = os.path.join(ROOT, "string_grouper_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert not re.search(r"^\s*(import|from)\s+sklearn", src, flags=re.M), fn


def test_pairwise_sum_is_numpy_sum():
    """numpy's own contiguous sum takes the same pairwise path (np.add.reduce)"""
    rng = np.random.default_rng(1)
    for dtype in DTYPES:
        for n in list(range(0, 40)) + [127, 128, 129, 135, 136, 255, 256, 257, 300, 1000, 5000]:
            a = (rng.random(n) * 10.0 ** rng.integers(-6, 1, n)).astype(dtype)
            assert pairwise_sum(a) == np.add.reduce(a), (dtype, n)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rowwise_dot_order_is_scipy(dtype):
    from oracle import pipeline as P
    left, right = common_count_pairs()
    M, D, _ = P.tf_idf_matrices(left, right, dtype=dtype)
    want = np.asarray(M.multiply(D).sum(axis=1)).squeeze(axis=1)
    got = rowwise_dot(M, D)
    counts = [len(np.intersect1d(M[i].indices, D[i].indices)) for i in range(len(COMMON_COUNTS))]
    assert counts == COMMON_COUNTS
    assert want.dtype == got.dtype == dtype
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:10]
    # the order matters: a sequential sum differs from scipy on some rows of this corpus
    prods = [common_products(M, D, i) for i in range(M.shape[0])]
    seq = np.array([np.cumsum(p)[-1] if len(p) else 0 for p in prods], dtype=dtype)
    assert (seq != want).sum() > 10

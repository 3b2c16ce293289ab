"""-m gpu: the triangle of a self-match.  cossim_topn(A, A) over all rows computes each unordered pair once and mirrors
the kept pairs; two distinct DeviceCSR objects of the same matrix take the full product.  Both must give the same
output bit for bit (rows, columns, scores, order, max_row), while the triangle reports about half the candidates."""
import numpy as np
import pytest

from synth_corpus import make_names

pytestmark = pytest.mark.gpu


def _D():
    from string_grouper_b200 import _device as D
    return D


def _matrix(n, seed):
    from oracle import pipeline as P
    m, _, _ = P.tf_idf_matrices(make_names(n, seed=seed))
    return m


def _both(D, m, thr, **kw):
    """(triangle output, full output, triangle stats, full stats)"""
    A = D.DeviceCSR.from_scipy(m)
    A_copy = D.DeviceCSR.from_scipy(m)
    st_tri, st_full = {}, {}
    tri = D.cossim_topn(A, A, 20, thr, stats=st_tri, **kw)
    full = D.cossim_topn(A, A_copy, 20, thr, stats=st_full, **kw)
    return tri, full, st_tri, st_full


def _assert_same(tri, full, st_tri, st_full, what, n_diag=0):
    """n_diag: pairs (i, i) both products report once; the triangle halves the others"""
    got, want = tri.host_triples(), full.host_triples()
    for name, g, w in zip(("rows", "cols", "scores"), got, want):
        assert np.array_equal(g, w), "%s: %s differ" % (what, name)
    assert tri.nnz == full.nnz and tri.max_row == full.max_row, what
    assert st_tri["triangle"] is True and st_full["triangle"] is False, what
    n_tri, n_full = st_tri["n_candidates"] - n_diag, st_full["n_candidates"] - n_diag
    assert n_tri <= 0.6 * n_full, (what, st_tri["n_candidates"], st_full["n_candidates"], n_diag)


@pytest.fixture(scope="module")
def small():
    return _matrix(12000, seed=41)


@pytest.mark.parametrize("kernel,acc", [("row", "u16"), ("row", "f32"), ("tiles", "u16")])
@pytest.mark.parametrize("thr", [0.5, 0.8, 0.95])
def test_triangle_equals_full_product(small, kernel, acc, thr):
    D = _D()
    tri, full, st_tri, st_full = _both(D, small, thr, kernel=kernel, acc=acc)
    for st in (st_tri, st_full):
        assert st["kernel"] == kernel and st["acc"] == acc and st["n_row_chunks"] == 1
    assert tri.nnz > small.shape[0]
    # at 0.95 most candidates are the diagonal pairs, which the triangle keeps: compare the others
    n_diag = np.count_nonzero(np.diff(small.indptr)) if thr > 0.9 else 0
    _assert_same(tri, full, st_tri, st_full, "%s %s thr=%r" % (kernel, acc, thr), n_diag)


@pytest.mark.parametrize("kernel", ["row", "tiles"])
def test_triangle_row_chunks_and_sizing_sample(monkeypatch, kernel):
    """no optimistic launch: the sizing pass runs on a strided sample of the processing order, then the rows go in
    slices of it (row chunks); both pass diag_rank slices and strides of the same order"""
    D = _D()
    m = _matrix(70000, seed=43)
    monkeypatch.setattr(D, "OPTIMISTIC_PAIRS", 0)
    monkeypatch.setattr(D, "CAND_CHUNK", 1 << 16)
    tri, full, st_tri, st_full = _both(D, m, 0.8, kernel=kernel)
    for st in (st_tri, st_full):
        assert st["kernel"] == kernel and st["n_row_chunks"] > 1 and st["n_candidates_estimate"] is not None
    _assert_same(tri, full, st_tri, st_full, "%s chunks" % kernel)


def test_triangle_only_for_the_whole_self_match(small):
    """a row range of A against A (one shard) keeps the full product"""
    D = _D()
    A = D.DeviceCSR.from_scipy(small)
    st = {}
    D.cossim_topn(A, A, 20, 0.8, row_begin=0, row_end=small.shape[0] - 1, stats=st)
    assert st["triangle"] is False

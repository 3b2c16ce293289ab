"""-m gpu: the dedup path of a self-match (cossim_topn's `dedup`, DESIGN.md §4 "Identical rows") is bit-identical to
the plain product: rows, columns, scores, order, nnz and max_row with np.array_equal, on every kernel, accumulator,
dtype, threshold, top_n and selection path, plus the exact reference (tests/exact_topn.py) where it is cheap."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix

from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn
from synth_corpus import make_names

pytestmark = pytest.mark.gpu


def _D():
    from string_grouper_b200 import _device as D
    return D


def _P():
    from oracle import pipeline as P
    return P


def _out(M):
    n = M.shape[0]
    return M.host_triples() + (np.asarray([M.nnz, M.max_row]), M.d_indptr[:n + 1].cpu().numpy())


def _both(A, top_n, thr, **kw):
    """cossim_topn with dedup=True and dedup=False: asserts both paths ran and every output is equal; returns the
    dedup result's (row, col, score, max_row) and stats"""
    D = _D()
    st1, st0 = {}, {}
    a = D.cossim_topn(A, A, top_n, thr, stats=st1, dedup=True, **kw)
    b = D.cossim_topn(A, A, top_n, thr, stats=st0, dedup=False, **kw)
    assert st1["dedup"] is True and st0["dedup"] is False
    assert st1["select"] == "rows" and st1["triangle"] is True
    for name, x, y in zip(("row", "col", "score", "nnz/max_row", "indptr"), _out(a), _out(b)):
        assert np.array_equal(x, y), "%s differs (top_n=%d thr=%r %r)" % (name, top_n, thr, kw)
    return a.host_triples() + (a.max_row,), st1


def _dup_names(n, seed):
    """make_names plus repeats that the analyzer folds into bit-identical rows (case, [,-./], whitespace)"""
    rng = np.random.default_rng(seed)
    names = make_names(n, seed=seed)
    pick = rng.choice(n, n // 4, replace=True)
    names += [names[i].upper() if i % 3 == 0 else names[i] + ("." if i % 3 == 1 else " ,") for i in pick]
    return [names[i] for i in rng.permutation(len(names))]


@pytest.fixture(scope="module")
def corpora():
    """dtype -> device matrix of 25 000 names with about a fifth repeated"""
    D, P = _D(), _P()
    out = {}
    for dtype in (np.float64, np.float32):
        m, _, _ = P.tf_idf_matrices(_dup_names(20000, 41), dtype=dtype)
        out[dtype] = D.DeviceCSR.from_scipy(m)
    return out


def test_groups_are_bit_identical_rows(corpora):
    """uid / members / representatives against a host grouping of the rows by their bytes"""
    D = _D()
    for A in corpora.values():
        g = D.row_groups(A)
        host = A.to_scipy()
        n, m = A.shape[0], g["m"]
        keys = [host.indices[host.indptr[r]:host.indptr[r + 1]].tobytes() +
                host.data[host.indptr[r]:host.indptr[r + 1]].tobytes() for r in range(n)]
        first = {}
        want = np.array([first.setdefault(k, len(first)) for k in keys])
        uid = g["uid"][:n].cpu().numpy()
        mem_ptr = g["mem_ptr"][:m + 1].cpu().numpy()
        mem_rows = g["mem_rows"][:n].cpu().numpy()
        rep = g["rep"][:m].cpu().numpy()
        assert m == len(first) and m < 0.9 * n
        assert np.array_equal(uid, want)                     # groups numbered by their first member
        assert np.array_equal(rep, mem_rows[mem_ptr[:-1]]) and np.all(np.diff(rep) > 0)
        for u in range(m):
            mem = mem_rows[mem_ptr[u]:mem_ptr[u + 1]]
            assert np.all(np.diff(mem) > 0) and np.all(uid[mem] == u)
        U = D.unique_rows(A).to_scipy()
        h = host[rep]
        assert np.array_equal(U.indptr, h.indptr) and np.array_equal(U.indices, h.indices)
        assert np.array_equal(U.data.view(np.uint8), h.data.view(np.uint8))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("kernel,acc", [("row", "u16"), ("row", "f32"), ("tiles", "u16")])
def test_thresholds_and_top_n(corpora, dtype, kernel, acc):
    A = corpora[dtype]
    for thr in (0.5, 0.8, 0.95):
        for top_n in (1, 20, 32, 100, 2048):
            _, st = _both(A, top_n, thr, kernel=kernel, acc=acc)
            assert st["kernel"] == kernel and st["acc"] == acc
            assert st["n_unique_rows"] < A.shape[0]


def test_exact_reference(corpora):
    A = corpora[np.float64]
    host = A.to_scipy()
    for top_n, thr in ((20, 0.8), (2048, 0.5)):
        got, _ = _both(A, top_n, thr)
        assert_same(got, exact_topn(host, host, top_n, thr), "dedup top_n=%d thr=%r" % (top_n, thr))


def test_thresholds_on_pair_scores():
    """thresholds equal to pair scores (the pair must be out) and the next double below (the pair must be in), on the
    corpus of the exact K2 tests (repeated long and short rows, single-feature rows, uniform-weight twins)"""
    from test_gpu_k2_exact import FLOOR, TOP_N, _matrix, _pick_scores, _thresholds
    D = _D()
    for dtype in (np.float64, np.float32):
        A = D.DeviceCSR.from_scipy(_matrix(dtype))
        host = A.to_scipy()
        table = RankedPairs(*exact_pairs(host, host, FLOOR))
        for thr in _thresholds(_pick_scores(host, table)):
            for kernel in ("row", "tiles"):
                got, _ = _both(A, TOP_N, thr, kernel=kernel)
                assert_same(got, table.topn(TOP_N, thr), "dedup %s thr=%r" % (kernel, thr))


def test_row_chunks(corpora, monkeypatch):
    D = _D()
    monkeypatch.setattr(D, "CAND_CHUNK", 1 << 14)
    for kernel in ("row", "tiles"):
        _, st = _both(corpora[np.float64], 20, 0.8, kernel=kernel)
        assert st["n_row_chunks"] > 1


def test_clusters_of_identical_rows():
    """the right side of the selection-path corpus of tests/test_gpu_k2_exact.py as a self-match (smaller): groups of
    up to
    2 049 identical rows with near-duplicates interleaved, so ties at the cut span groups; every selection kernel
    (rows of up to 4 097 survivors)"""
    SIZES = (1, 31, 33, 513, 4097)
    rng = np.random.default_rng(7)
    letters = np.array(list("ABCDEFGHIJKLMNOPQRSTUVWXYZ"))
    right = []
    for m in SIZES:
        base = "".join(rng.choice(letters, 30))
        variants = [base[:k] + "Z" + base[k + 1:] for k in (5, 15, 25)]
        n_id = (m + 1) // 2
        right += [base] * n_id + [variants[i % 3] for i in range(m - n_id)]
    right = [right[i] for i in rng.permutation(len(right))]
    host, _, _ = _P().tf_idf_matrices(right)
    B = _D().DeviceCSR.from_scipy(host)
    host = B.to_scipy()
    table = RankedPairs(*exact_pairs(host, host, 0.5))
    for top_n in (1, 20, 31, 32, 33, 100, 512, 513, 2048):
        got, st = _both(B, top_n, 0.5)
        assert st["n_unique_rows"] < 40
        assert_same(got, table.topn(top_n, 0.5), "clusters top_n=%d" % top_n)


def test_dyadic_ties_across_groups():
    """dyadic weights: every score a multiple of 1/16, groups of different sizes tie exactly at the cut with
    interleaved column ids"""
    D = _D()
    rng = np.random.default_rng(3)
    base = [np.sort(rng.choice(60, 4, replace=False)) for _ in range(40)]
    rows = [base[i % 40] for i in rng.permutation(40 * 9)] + [np.sort(rng.choice(60, 4, replace=False))
                                                               for _ in range(300)]
    rows = [rows[i] for i in rng.permutation(len(rows))]
    m = csr_matrix((np.full(4 * len(rows), 0.5), np.concatenate(rows), np.arange(0, 4 * len(rows) + 1, 4)),
                   shape=(len(rows), 60))
    A = D.DeviceCSR.from_scipy(m)
    table = RankedPairs(*exact_pairs(m, m, 0.2))
    for thr in (0.25, float(np.nextafter(0.25, 0)), 0.5, float(np.nextafter(0.5, 0))):
        for top_n in (1, 5, 20, 32, 100):
            got, _ = _both(A, top_n, thr)
            assert_same(got, table.topn(top_n, thr), "dyadic top_n=%d thr=%r" % (top_n, thr))


def test_no_duplicates_and_all_identical():
    D, P = _D(), _P()
    names = sorted(set(make_names(6000, seed=17)))
    m, _, _ = P.tf_idf_matrices(names)
    A = D.DeviceCSR.from_scipy(m)
    keys = {m.indices[m.indptr[r]:m.indptr[r + 1]].tobytes() + m.data[m.indptr[r]:m.indptr[r + 1]].tobytes()
            for r in range(m.shape[0])}
    _, st = _both(A, 20, 0.8)
    assert st["n_unique_rows"] == len(keys)
    same, _, _ = P.tf_idf_matrices(["acme holdings inc"] * 700)
    A = D.DeviceCSR.from_scipy(same)
    for top_n in (1, 20, 700):
        got, st = _both(A, top_n, 0.8)
        assert st["n_unique_rows"] == 1 and got[3] == top_n
        assert_same(got, exact_topn(same, same, top_n, 0.8), "identical top_n=%d" % top_n)


@pytest.mark.parametrize("mask", [0, 3, (1 << 20) - 1])
def test_hash_collisions_are_verified(corpora, monkeypatch, mask):
    """a narrow hash mask puts different rows under one hash: they must stay apart (and identical rows separated by
    them may split into several groups), and the result is still the plain product"""
    D = _D()
    monkeypatch.setattr(D, "DEDUP_HASH_MASK", mask)
    for dtype in (np.float64, np.float32):
        A = corpora[dtype]
        _, st = _both(A, 20, 0.8)
        _, st2 = _both(A, 100, 0.5, kernel="tiles")
        g = D.row_groups(A)
        uid = g["uid"][:A.shape[0]].cpu().numpy()
        host = A.to_scipy()
        for u in np.unique(uid)[::97]:                      # every member is bit-identical to its representative
            rows = np.flatnonzero(uid == u)
            ref = host[rows[0]]
            for r in rows[1:]:
                x = host[r]
                assert np.array_equal(x.indices, ref.indices) and np.array_equal(x.data.view(np.uint8),
                                                                                 ref.data.view(np.uint8))
    monkeypatch.setattr(D, "DEDUP_HASH_MASK", (1 << 64) - 1)


def test_public_api_equal_to_plain_path(monkeypatch):
    import string_grouper_b200 as api
    D = _D()
    s = pd.Series(_dup_names(8000, 5))
    out = {}
    for min_rows in (0, 1 << 40):
        monkeypatch.setattr(D, "DEDUP_MIN_ROWS", min_rows)
        sg = api.StringGrouper(s).fit()
        assert sg._last_stats["dedup"] is (min_rows == 0)
        out[min_rows] = (api.match_strings(s), api.group_similar_strings(s, min_similarity=0.7),
                         api.match_strings(s, max_n_matches=3))
    for a, b in zip(out[0], out[1 << 40]):
        pd.testing.assert_frame_equal(a.to_frame() if isinstance(a, pd.Series) else a,
                                      b.to_frame() if isinstance(b, pd.Series) else b, check_exact=True)


def test_auto_leaves_other_products_alone(corpora, monkeypatch):
    D = _D()
    A = corpora[np.float64]
    n = A.shape[0]

    def ran(*args, **kw):
        st = {}
        D.cossim_topn(*args, stats=st, **kw)
        return st.get("dedup")

    assert ran(A, A, 20, 0.8) is False                                     # below DEDUP_MIN_ROWS
    monkeypatch.setattr(D, "DEDUP_MIN_ROWS", 0)
    assert ran(A, A, 20, 0.8) is True
    assert ran(A, A, 20, 0.8, row_begin=0, row_end=n // 2) is False          # a row range (shard)
    assert ran(A, A, 20, 0.8, row_begin=n // 2) is False
    B = D.DeviceCSR.from_scipy(A.to_scipy())
    assert ran(A, B, 20, 0.8) is False                                     # two matrices
    assert ran(A, A, 4000, 0.8) is False                                   # top_n above sg_topn_rows_cap() / 2
    assert not ran(A, A, 20, 0.3, floor=True)                              # the top-n floor
    monkeypatch.setattr(D, "SELECT_MODE", "sort")
    assert ran(A, A, 20, 0.8) is False
    monkeypatch.setattr(D, "SELECT_MODE", "rows")
    host = A.to_scipy()
    reps = D.row_groups(A)["rep"][:D.row_groups(A)["m"]].cpu().numpy()
    U = D.DeviceCSR.from_scipy(host[np.r_[reps, reps[:len(reps) // 100]]])      # 1 % repeats
    assert ran(U, U, 20, 0.8) is False                                     # fewer than DEDUP_MIN_SHARE repeats
    assert D.row_groups(U)["m"] == len(reps)


def test_full_size_dedup_is_bit_equal():
    """the 663k benchmark product: auto takes the dedup path, and it equals the plain product"""
    from string_grouper_b200 import StringGrouper
    sg = StringGrouper(pd.Series(make_names(663_000, seed=0))).fit()
    A, _ = sg._get_tf_idf_matrices()
    got, st = _both(A, 20, 0.8)
    assert st["tile_w"] == 128 and st["n_unique_rows"] < 0.8 * A.shape[0]
    st_auto = {}
    _D().cossim_topn(A, A, 20, 0.8, stats=st_auto)
    assert st_auto["dedup"] is True and st_auto["n_expanded"] == st["n_expanded"]

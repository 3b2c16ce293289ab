"""-m gpu: the top-n product without a threshold (min_similarity <= 0: every pair with a positive score counts) through
the top-n floor (DESIGN.md §4): initial floors from exact neighbour scores, pruning against them, and the block-max
bound of rows with more than 32 kept features.  Every case compares the whole output bit for bit (rows, columns,
scores, order, max_row) with the exact reference (tests/exact_topn.py) and asserts from `stats` which path ran."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix

from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

CLUSTER = 320         # identical names: hundreds of pairs tie at the cut
THRESHOLDS = [0.0, -0.25, -np.inf]
LONG = ["international consolidated widget manufacturing holdings of north america incorporated",
        "the first national bank and trust company of greater south western pennsylvania",
        "associated independent wholesale grocers and food distributors cooperative association",
        "amalgamated transcontinental railway equipment leasing and financial services corporation"]


def _D():
    from string_grouper_b200 import _device as D
    return D


def _names(n=6000, seed=11):
    names = make_names(n, seed=seed)
    longs = LONG + [s + " " + t for s in LONG for t in ("ltd", "group", "holdings")]
    return names + ["acme global holdings llc"] * CLUSTER + ["acme global holding llc"] * 40 + longs


@pytest.fixture(scope="module", params=[np.float64, np.float32], ids=["f64", "f32"])
def corpus(request):
    from oracle import pipeline as P
    m, _, _ = P.tf_idf_matrices(_names(), dtype=request.param)
    m = csr_matrix(m).astype(request.param)
    m.sort_indices()
    table = RankedPairs(*exact_pairs(m, m, 0.0))
    return m, _D().DeviceCSR.from_scipy(m), table


def _run(A, B, top_n, thr, floor=True, **kw):
    st = {}
    got = _D().cossim_topn(A, B, top_n, thr, stats=st, floor=floor, **kw)
    assert st["topn_floor"] is bool(floor), st
    if floor:
        assert st["floor_init"] is True and st["acc"] == "f32", st
    return got.host_triples() + (got.max_row,), st


def _exact_blocks(left, right, top_n, thr, block_rows=128):
    """exact_topn row block by row block (rows are independent): the pairs of one block at a time stay in memory"""
    out = [[], [], []]
    max_row = 0
    for lo in range(0, left.shape[0], block_rows):
        r, c, s, mr = exact_topn(left[lo:lo + block_rows], right, top_n, thr, block_rows=block_rows)
        out[0].append(r + lo), out[1].append(c), out[2].append(s)
        max_row = max(max_row, mr)
    return tuple(np.concatenate(x) for x in out) + (max_row,)


@pytest.mark.parametrize("thr", THRESHOLDS)
@pytest.mark.parametrize("top_n", [1, 2, 20, 32])
def test_self_match_exact(corpus, thr, top_n):
    m, A, table = corpus
    got, st = _run(A, A, top_n, thr)
    assert st["n_floor_init_positive"] > 0.5 * m.shape[0], st["n_floor_init_positive"]
    assert st["n_candidates_seed"] > 0 and st["triangle"] is False
    assert_same(got, table.topn(top_n, 0.0), "self-match thr=%r top_n=%d" % (thr, top_n))


def test_floor_init_is_a_lower_bound(corpus):
    m, A, table = corpus
    D = _D()
    n = m.shape[0]
    for top_n in (1, 20, 32):
        nth = np.zeros(n)
        r, _, s, _ = table.topn(top_n, 0.0)
        full = np.bincount(r, minlength=n) == top_n
        last = np.r_[np.flatnonzero(np.diff(r)), len(r) - 1]       # rows are written score-descending
        nth[r[last]] = np.where(full[r[last]], s[last], 0.0)
        for thr in (0.0, -np.inf):
            floor = D.topn_floor_init(A, A, top_n, thr).cpu().numpy().astype(np.float64)
            assert np.all(floor <= nth) and (floor > 0).mean() > 0.5, (top_n, (floor > 0).mean())
        # two matrices: the position is the insertion point of the left row's key among the right rows
        left, right = m[1000:4501], m[2999:]
        nth2 = np.zeros(left.shape[0])
        r2, _, s2, _ = exact_topn(left, right, top_n, 0.0)
        full2 = np.bincount(r2, minlength=left.shape[0]) == top_n
        last2 = np.r_[np.flatnonzero(np.diff(r2)), len(r2) - 1]
        nth2[r2[last2]] = np.where(full2[r2[last2]], s2[last2], 0.0)
        L, R = D.DeviceCSR.from_scipy(left), D.DeviceCSR.from_scipy(right)
        floor2 = D.topn_floor_init(L, R, top_n, 0.0).cpu().numpy().astype(np.float64)
        assert np.all(floor2 <= nth2) and (floor2 > 0).mean() > 0.5, (top_n, (floor2 > 0).mean())
        # a row range: zero outside it
        f3 = D.topn_floor_init(A, A, top_n, 0.0, 1700, 4099).cpu().numpy()
        assert not f3[:1700].any() and not f3[4099:].any() and np.all(f3[1700:4099] <= nth[1700:4099])


def test_two_matrices_odd_widths_and_row_ranges(corpus):
    m, A, table = corpus
    D = _D()
    for lo, hi in ((0, 3001), (2999, m.shape[0])):
        left, right = m[1000:4501], m[lo:hi]
        L, R = D.DeviceCSR.from_scipy(left), D.DeviceCSR.from_scipy(right)
        for thr, top_n in ((0.0, 20), (-np.inf, 1), (-0.25, 32)):
            got, st = _run(L, R, top_n, thr)
            assert st["n_candidates_seed"] == 0
            assert_same(got, exact_topn(left, right, top_n, 0.0), "two matrices [%d, %d) thr=%r" % (lo, hi, thr))
    n = m.shape[0]
    for lo, hi in ((0, 1700), (1700, 4099), (4099, n)):
        got, st = _run(A, A, 20, 0.0, row_begin=lo, row_end=hi)
        assert st["n_candidates_seed"] > 0
        assert_same(got, table.topn(20, 0.0, rows=(lo, hi)), "rows [%d, %d)" % (lo, hi))


def test_row_chunks(corpus, monkeypatch):
    m, A, table = corpus
    D = _D()
    # 64-column fp32 tiles in groups of 64 tiles: several groups, so the launch after the seed has work to chunk
    monkeypatch.setattr(D, "GROUP_BYTES", 1)
    for chunk in (1 << 28, 1000):
        monkeypatch.setattr(D, "CAND_CHUNK", chunk)
        got, st = _run(A, A, 20, 0.0, tile_w=64)
        assert st["tiles_per_group"] < st["n_tiles"] and st["n_candidates_main"] > 0
        assert (st["n_row_chunks"] > 1) == (chunk == 1000)
        assert_same(got, table.topn(20, 0.0), "row chunks of %d candidates" % chunk)


def test_long_rows_are_bounded_and_exact(corpus):
    """rows with more than 32 kept features (the long names) go through the chunked block-max bound"""
    m, A, table = corpus
    long_ids = np.flatnonzero(np.diff(m.indptr) > 32)
    assert len(long_ids) >= len(LONG)
    for top_n in (2, 20):
        got, st = _run(A, A, top_n, 0.0, prune=0.0)            # unpruned: every long row keeps all its features
        assert st["n_rows_long"] == len(long_ids), (st["n_rows_long"], len(long_ids))
        assert_same(got, table.topn(top_n, 0.0), "long rows top_n=%d" % top_n)
        gr = got[0]
        assert np.isin(long_ids, gr).all()


def test_public_api_without_threshold(monkeypatch):
    """match_strings / match_most_similar at min_similarity 0 with the floor forced on equal the usual path"""
    import string_grouper_b200 as api
    from string_grouper_b200 import StringGrouper
    D = _D()
    names = pd.Series(_names(3000, seed=4))
    master = pd.Series(make_names(2500, seed=6) + ["acme global holdings llc"] * 30)
    dupes = pd.Series(make_names(1500, seed=7) + ["acme global holding llc"] * 5)
    res = {}
    for mode in (True, False):
        monkeypatch.setattr(D, "TOPN_FLOOR", mode)
        sg = StringGrouper(names, min_similarity=0, max_n_matches=5).fit()
        assert sg._last_stats["topn_floor"] is mode
        res[mode] = (api.match_strings(names, min_similarity=0, include_zeroes=False, max_n_matches=5),
                     api.match_most_similar(master, dupes, min_similarity=0))
    pd.testing.assert_frame_equal(res[True][0], res[False][0])
    a, b = res[True][1], res[False][1]
    if isinstance(a, pd.DataFrame):
        pd.testing.assert_frame_equal(a, b)
    else:
        pd.testing.assert_series_equal(a, b)


# ---------------------------------------------------------------------------------------------------------------
# full size (the benchmark corpus), like tests/test_gpu_topn_floor.py
# ---------------------------------------------------------------------------------------------------------------
N = 663_000


def test_full_size_self_match_without_threshold_exact_on_sampled_rows():
    """663k self-match at 0.0, top 20: auto takes the path and the run completes; 2 000 sampled rows bit-exact"""
    from string_grouper_b200 import StringGrouper
    D = _D()
    A, _ = StringGrouper(pd.Series(make_names(N, seed=0))).fit()._get_tf_idf_matrices()
    st = {}
    got = D.cossim_topn(A, A, 20, 0.0, stats=st)
    assert st["topn_floor"] is True and st["floor_init"] is True, st
    host = A.to_scipy()
    rows = np.sort(np.random.default_rng(8).choice(N, 2000, replace=False))
    r, c, s, _ = _exact_blocks(host[rows], host, 20, 0.0)
    gr, gc, gs = got.host_triples()
    sel = np.isin(gr, rows)
    assert_same((gr[sel], gc[sel], gs[sel]), (rows[r], c, s), "663k at 0.0, sampled rows")


def test_config4_shape_two_series_without_threshold_exact_on_sampled_rows():
    """400k x 150k two-Series shape at 0.0, top 1 and top 20: sampled rows bit-exact"""
    from string_grouper_b200 import StringGrouper
    D = _D()
    base = make_names(480_000, seed=3)
    master, dupes = pd.Series(base[:400_000]), pd.Series(base[330_000:480_000])
    A, B = StringGrouper(master, duplicates=dupes).fit()._get_tf_idf_matrices()
    left, right = A.to_scipy(), B.to_scipy()
    rows = np.sort(np.random.default_rng(9).choice(left.shape[0], 2000, replace=False))
    for top_n in (1, 20):
        st = {}
        got = D.cossim_topn(A, B, top_n, 0.0, stats=st, floor=True)
        assert st["topn_floor"] is True and st["n_candidates_seed"] == 0
        r, c, s, _ = _exact_blocks(left[rows], right, top_n, 0.0)
        gr, gc, gs = got.host_triples()
        sel = np.isin(gr, rows)
        assert_same((gr[sel], gc[sel], gs[sel]), (rows[r], c, s), "config 4 shape top_n=%d" % top_n)

"""-m gpu: the top-n floor of K2 (DESIGN.md §4, `cossim_topn(..., floor=True)`) against the exact reference
(tests/exact_topn.py).  Every case compares the whole output bit for bit (rows, columns, scores, order, max_row) and
asserts from `stats` that the floor path ran."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix

from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

LOWEST = 0.04         # the reference pairs are collected once above this; every threshold below lies above it
CLUSTER = 320         # identical names: their floor is 1.0 and hundreds of pairs tie at the cut


def _D():
    from string_grouper_b200 import _device as D
    return D


def _names(n=6000, seed=11):
    names = make_names(n, seed=seed)
    return names + ["acme global holdings llc"] * CLUSTER + ["acme global holding llc"] * 40


@pytest.fixture(scope="module", params=[np.float64, np.float32], ids=["f64", "f32"])
def corpus(request):
    from oracle import pipeline as P
    m, _, _ = P.tf_idf_matrices(_names(), dtype=request.param)
    m = csr_matrix(m).astype(request.param)
    m.sort_indices()
    table = RankedPairs(*exact_pairs(m, m, LOWEST))
    return m, _D().DeviceCSR.from_scipy(m), table


def _run(A, B, top_n, thr, floor=True, **kw):
    st = {}
    got = _D().cossim_topn(A, B, top_n, thr, stats=st, floor=floor, **kw)
    assert st["topn_floor"] is bool(floor), st
    return got.host_triples() + (got.max_row,), st


@pytest.mark.parametrize("thr", [0.05, 0.1, 0.3, 0.6])
@pytest.mark.parametrize("top_n", [1, 2, 20, 32])
def test_floor_self_match_exact(corpus, thr, top_n):
    m, A, table = corpus
    got, st = _run(A, A, top_n, thr)
    assert st["n_candidates_seed"] > 0 and st["triangle"] is False
    assert_same(got, table.topn(top_n, thr), "self-match thr=%g top_n=%d" % (thr, top_n))


@pytest.mark.parametrize("acc", ["u16", "f32"])
@pytest.mark.parametrize("prune", [None, 0.0])
def test_floor_accumulators_and_pruning(corpus, acc, prune):
    m, A, table = corpus
    for thr in (0.05, 0.1, 0.3):
        got, st = _run(A, A, 20, thr, acc=acc, prune=prune)
        assert st["acc"] == ("f32" if thr < 0.06 else acc), st["acc"]      # near-zero thresholds take fp32
        assert_same(got, table.topn(20, thr), "acc=%s prune=%s thr=%g" % (acc, prune, thr))


def test_floor_thresholds_on_pair_scores(corpus):
    """thresholds equal to a pair's score (which must then be left out) and the next double below it (kept), among
    them the scores at the top-n cut of rows, where the floor and the threshold meet"""
    m, A, table = corpus
    at_cut = table.score[(table.rank == 19) & (table.score > 0.1)]
    picks = list(np.quantile(at_cut, [0.0, 0.1, 0.5, 0.9]).round(12))
    picks = [at_cut[np.argmin(np.abs(at_cut - q))] for q in picks]
    picks += [table.score[(table.score > 0.05) & (table.score < 0.2)].min()]
    for s in picks:
        for thr in (float(s), float(np.nextafter(s, -np.inf))):
            got, _ = _run(A, A, 20, thr)
            assert_same(got, table.topn(20, thr), "thr=%r" % thr)


def test_floor_on_and_off_agree(corpus):
    m, A, table = corpus
    for thr, top_n in ((0.3, 20), (0.6, 2), (0.1, 1)):
        on, st_on = _run(A, A, top_n, thr, floor=True)
        off, st_off = _run(A, A, top_n, thr, floor=False)
        assert_same(on, off, "on vs off thr=%g" % thr)
        assert st_on["n_survivors"] <= st_off["n_above_threshold"] * 2


def test_floor_row_chunks_and_row_ranges(corpus, monkeypatch):
    m, A, table = corpus
    D = _D()
    # 64-column fp32 tiles in groups of 64 tiles: several groups, so the launch after the seed has work to chunk
    monkeypatch.setattr(D, "GROUP_BYTES", 1)
    for chunk in (1 << 28, 1000):
        monkeypatch.setattr(D, "CAND_CHUNK", chunk)
        for thr in (0.1, 0.3):
            got, st = _run(A, A, 20, thr, acc="f32", tile_w=64)
            assert st["tiles_per_group"] < st["n_tiles"] and st["n_candidates_main"] > 0
            assert (st["n_row_chunks"] > 1) == (chunk == 1000)
            assert_same(got, table.topn(20, thr), "row chunks of %d candidates, thr=%g" % (chunk, thr))
    monkeypatch.undo()
    n = m.shape[0]
    for lo, hi in ((0, 1700), (1700, 4099), (4099, n)):
        got, st = _run(A, A, 20, 0.1, row_begin=lo, row_end=hi)
        assert st["n_candidates_seed"] > 0
        assert_same(got, table.topn(20, 0.1, rows=(lo, hi)), "rows [%d, %d)" % (lo, hi))


def test_floor_two_matrices_odd_widths(corpus):
    m, _, _ = corpus
    D = _D()
    for lo, hi in ((0, 3001), (2999, m.shape[0])):
        left, right = m[1000:4501], m[lo:hi]
        A, B = D.DeviceCSR.from_scipy(left), D.DeviceCSR.from_scipy(right)
        for thr, top_n in ((0.1, 20), (0.3, 1), (0.05, 32)):
            got, st = _run(A, B, top_n, thr)
            assert st["n_candidates_seed"] == 0
            assert_same(got, exact_topn(left, right, top_n, thr), "two matrices [%d, %d) thr=%g" % (lo, hi, thr))


def test_floor_argument_checks(corpus):
    m, A, _ = corpus
    D = _D()
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 33, 0.1, floor=True)
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 20, 0.1, floor=True, kernel="tiles")
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 20, 0.1, floor="yes")


def test_auto_keeps_small_and_high_threshold_inputs_on_the_usual_path(corpus):
    """auto engages only from 65 536 left rows at thresholds below 0.5: every smaller or higher-threshold input
    (all of the suite's other cases, bench.py at 0.8) stays on the usual path"""
    m, A, _ = corpus
    for thr in (0.05, 0.3, 0.8):
        st = {}
        _D().cossim_topn(A, A, 20, thr, stats=st, floor="auto")
        assert st["topn_floor"] is False


def test_medium_candidate_reduction():
    """100k names at 0.3: the floor cuts the candidates and returns the same triples"""
    from oracle import pipeline as P
    D = _D()
    m, _, _ = P.tf_idf_matrices(make_names(100_000, seed=0))
    A = D.DeviceCSR.from_scipy(m)
    on, st_on = _run(A, A, 20, 0.3, floor=True)
    off, st_off = _run(A, A, 20, 0.3, floor=False)
    assert_same(on, off, "100k at 0.3")
    # the usual path reports the triangle (each pair once): compare per ordered pair.  Measured on one H100: 0.546
    ratio = st_on["n_candidates"] / (2.0 * st_off["n_candidates"])
    print("100k at 0.3: floor %d candidates (seed %d), usual %d (triangle), ratio %.3f" % (
        st_on["n_candidates"], st_on["n_candidates_seed"], st_off["n_candidates"], ratio))
    assert ratio < 0.7


def test_public_api_with_the_floor(monkeypatch):
    """match_strings at 0.1 and match_most_similar at 0.3 with the floor forced equal the usual path (itself held
    exact by tests/test_gpu_k2_exact.py), and the product under them equals the exact reference"""
    import string_grouper_b200 as api
    from string_grouper_b200 import StringGrouper
    D = _D()
    names = pd.Series(_names(3000, seed=4))
    master = pd.Series(make_names(2500, seed=6) + ["acme global holdings llc"] * 30)
    dupes = pd.Series(make_names(1500, seed=7) + ["acme global holding llc"] * 5)
    res = {}
    for mode in (True, False):
        monkeypatch.setattr(D, "TOPN_FLOOR", mode)
        sg = StringGrouper(names, min_similarity=0.1).fit()
        assert sg._last_stats["topn_floor"] is mode
        res[mode] = (api.match_strings(names, min_similarity=0.1),
                     api.match_most_similar(master, dupes, min_similarity=0.3))
        A, _ = sg._get_tf_idf_matrices()
        host = A.to_scipy()
        got = D.cossim_topn(A, A, 20, 0.1, floor=mode)
        assert_same(got.host_triples() + (got.max_row,), exact_topn(host, host, 20, 0.1), "API matrix")
    pd.testing.assert_frame_equal(res[True][0], res[False][0])
    a, b = res[True][1], res[False][1]
    if isinstance(a, pd.DataFrame):
        pd.testing.assert_frame_equal(a, b)
    else:
        pd.testing.assert_series_equal(a, b)


# ---------------------------------------------------------------------------------------------------------------
# full size (the benchmark corpus), like tests/test_gpu_fullsize.py
# ---------------------------------------------------------------------------------------------------------------
N = 663_000


def test_full_size_low_threshold_auto_floor_exact_on_sampled_rows():
    """663k self-match at 0.1, top 20: auto takes the floor and the run completes; 2 000 sampled rows bit-exact"""
    from string_grouper_b200 import StringGrouper
    D = _D()
    A, _ = StringGrouper(pd.Series(make_names(N, seed=0))).fit()._get_tf_idf_matrices()
    st = {}
    got = D.cossim_topn(A, A, 20, 0.1, stats=st)
    assert st["topn_floor"] is True, st
    host = A.to_scipy()
    rows = np.sort(np.random.default_rng(8).choice(N, 2000, replace=False))
    r, c, s, _ = exact_topn(host[rows], host, 20, 0.1, block_rows=128)
    gr, gc, gs = got.host_triples()
    sel = np.isin(gr, rows)
    assert_same((gr[sel], gc[sel], gs[sel]), (rows[r], c, s), "663k at 0.1, sampled rows")
    st8 = {}
    D.cossim_topn(A, A, 20, 0.8, stats=st8)
    assert st8["topn_floor"] is False                     # the benchmark setting stays on the usual path


def test_config4_shape_two_series_floor_exact_on_sampled_rows():
    """400k x 150k two-Series shape at 0.3 (as in match_most_similar, top 1 and top 20): sampled rows bit-exact"""
    from string_grouper_b200 import StringGrouper
    D = _D()
    base = make_names(480_000, seed=3)
    master, dupes = pd.Series(base[:400_000]), pd.Series(base[330_000:480_000])
    A, B = StringGrouper(master, duplicates=dupes).fit()._get_tf_idf_matrices()
    left, right = A.to_scipy(), B.to_scipy()
    rows = np.sort(np.random.default_rng(9).choice(left.shape[0], 2000, replace=False))
    for top_n in (1, 20):
        st = {}
        got = D.cossim_topn(A, B, top_n, 0.3, stats=st, floor=True)
        assert st["topn_floor"] is True and st["n_candidates_seed"] == 0
        r, c, s, _ = exact_topn(left[rows], right, top_n, 0.3, block_rows=128)
        gr, gc, gs = got.host_triples()
        sel = np.isin(gr, rows)
        assert_same((gr[sel], gc[sel], gs[sel]), (rows[r], c, s), "config 4 shape top_n=%d" % top_n)

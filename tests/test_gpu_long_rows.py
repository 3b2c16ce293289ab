"""-m gpu: rows of more than 32 kept features in the usual and the position-range candidates kernels.  Their block-max
bound runs over all their kept features, 32 at a time, instead of walking every column tile.  Every case compares the
whole output bit for bit (rows, columns, scores, order, max_row) with the exact reference (tests/exact_topn.py) and
asserts from `stats` that such rows ran and which path they took."""
import numpy as np
import pytest
from scipy.sparse import csr_matrix

from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

FLOOR = 0.3                  # every threshold below lies at or above this
N_LEFT = 3000                # two matrices: the first N_LEFT rows against the rest
WORDS = ["international", "consolidated", "widget", "manufacturing", "holdings", "north", "america", "incorporated",
         "national", "bank", "trust", "company", "greater", "south", "western", "pennsylvania", "associated",
         "independent", "wholesale", "grocers", "food", "distributors", "cooperative", "transcontinental"]


def _D():
    from string_grouper_b200 import _device as D
    return D


def _long_names(rng, n):
    """names of 3 to 12 words: 30 to 110 distinct 3-grams, each with near duplicates"""
    out = []
    for _ in range(n):
        base = " ".join(rng.choice(WORDS, size=int(rng.integers(3, 13)), replace=False))
        out += [base, base + " ltd", base.replace(" ", "  ", 1), "the " + base]
    return out


@pytest.fixture(scope="module", params=[np.float64, np.float32], ids=["f64", "f32"])
def corpus(request):
    from oracle import pipeline as P
    rng = np.random.default_rng(5)
    names = make_names(5000, seed=17) + _long_names(rng, 150)
    names = [names[i] for i in rng.permutation(len(names))]     # long rows spread over the processing order
    m, _, _ = P.tf_idf_matrices(names, dtype=request.param)
    m = csr_matrix(m).astype(request.param)
    m.sort_indices()
    lens = np.diff(m.indptr)
    assert ((lens > 32) & (lens <= 100)).sum() >= 300, np.bincount(np.minimum(lens, 101) // 10)
    return m, _D().DeviceCSR.from_scipy(m), RankedPairs(*exact_pairs(m, m, FLOOR))


def _score_thresholds(table, m):
    """scores of pairs of long rows and the next double below each: the threshold drops the pair, the one below
    keeps it"""
    long_row = np.diff(m.indptr)[table.row] > 32
    s = np.unique(table.score[long_row & (table.rank < 20) & (table.row != table.col) & (table.score < 1.0)])
    picks = s[np.linspace(0, len(s) - 1, 3).astype(int)] if len(s) else []
    return [t for x in picks for t in (float(x), float(np.nextafter(x, -np.inf)))]


def _run(A, B, top_n, thr, expect, **kw):
    st = {}
    got = _D().cossim_topn(A, B, top_n, thr, stats=st, floor=False, **kw)
    for k, v in expect.items():
        assert st.get(k) == v, "path: %s is %r, expected %r" % (k, st.get(k), v)
    assert st["n_rows_long"] > 0, st["n_rows_long"]
    return got.host_triples() + (got.max_row,), st


@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_self_match_triangle(corpus, acc):
    m, A, table = corpus
    for thr in [0.5, 0.8] + _score_thresholds(table, m):
        for prune in (0.0, None):            # unpruned: every long row keeps all its features
            got, st = _run(A, A, 20, thr, {"acc": acc, "kernel": "row", "triangle": True}, acc=acc, prune=prune)
            if prune == 0.0:
                assert st["n_rows_long"] == int((np.diff(m.indptr) > 32).sum())
            assert_same(got, table.topn(20, thr), "self-match %s thr=%r prune=%r" % (acc, thr, prune))


@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_two_matrices_and_row_ranges(corpus, acc):
    m, A, table = corpus
    D = _D()
    left, right = m[:N_LEFT], m[N_LEFT:]
    L, R = D.DeviceCSR.from_scipy(left), D.DeviceCSR.from_scipy(right)
    for thr in (0.5, 0.8):
        got, _ = _run(L, R, 20, thr, {"acc": acc, "triangle": False}, acc=acc, prune=0.0)
        assert_same(got, exact_topn(left, right, 20, thr), "two matrices %s thr=%r" % (acc, thr))
    lo, hi = 1700, 4099
    got, _ = _run(A, A, 20, 0.5, {"acc": acc, "triangle": False}, acc=acc, prune=0.0, row_begin=lo, row_end=hi)
    assert_same(got, table.topn(20, 0.5, rows=(lo, hi)), "rows [%d, %d) %s" % (lo, hi, acc))


@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_range_kernel(corpus, acc):
    """blocked product: the position-range variant of the kernel"""
    import torch
    m, A, table = corpus
    n = m.shape[0]
    ids = np.random.default_rng(9).integers(0, 4, size=n).astype(np.int32)
    d = torch.from_numpy(ids).cuda()
    keep = ids[table.row] == ids[table.col]
    blocked = RankedPairs(table.row[keep], table.col[keep], table.score[keep])
    for thr in (0.5, 0.8):
        got, _ = _run(A, A, 20, thr, {"blocks": True, "acc": acc, "triangle": True}, acc=acc, prune=0.0,
                      block_ids=(d, d))
        assert_same(got, blocked.topn(20, thr), "blocked %s thr=%r" % (acc, thr))


def test_tile_widths_and_groups(corpus, monkeypatch):
    """narrow tiles in several column-tile groups, and wide tiles: long rows bounded in every group"""
    m, A, table = corpus
    D = _D()
    monkeypatch.setattr(D, "GROUP_BYTES", 1)
    for tile_w in (64, 256):
        got, st = _run(A, A, 20, 0.6, {"acc": "f32", "triangle": True}, acc="f32", prune=0.0, tile_w=tile_w)
        assert st["tile_w"] == tile_w and (tile_w > 64 or st["tiles_per_group"] < st["n_tiles"]), st
        assert_same(got, table.topn(20, 0.6), "tile_w=%d" % tile_w)

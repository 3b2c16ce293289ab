"""-m gpu: the candidates kernel's block-max test runs over passes of 128 column tiles, four consecutive tiles per lane.
These cases put the edges of a pass where 64-tile batches had none: the last pass of T = 1, 63, 64, 65 and 127
(mod 128) tiles, which ends inside the padded maxima rows or past them; triangle ranks in every quarter of a pass;
column-tile groups of 64 and 192 tiles, which start or end in the middle of a pass; the range kernel's `hi` inside a
pass; the top-n floor's seed, which starts at the pass holding the row; rows of 33, 64 and 65 kept features.  Each
compares the whole output bit for bit (rows, columns, scores, order, max_row) with the exact reference
(tests/exact_topn.py) and asserts from `stats` which kernel ran."""
import numpy as np
import pytest
from scipy.sparse import csr_matrix

from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

FLOOR = 0.3                  # every threshold below lies at or above this
N_SELF = 32000               # self-match rows: > 192 column tiles of 128 columns after identical rows are merged
N_LEFT = 1500                # two matrices: these rows (after the right rows) against the first n_right rows


def _D():
    from string_grouper_b200 import _device as D
    return D


def _csr(m):
    m = csr_matrix(m).astype(np.float64)
    m.sort_indices()
    return m


@pytest.fixture(scope="module")
def names_matrix():
    from oracle import pipeline as P
    m, _, _ = P.tf_idf_matrices(make_names(66000, seed=23), dtype=np.float64)
    return _csr(m)


@pytest.fixture(scope="module")
def self_match(names_matrix):
    m = names_matrix[:N_SELF]
    return m, _D().DeviceCSR.from_scipy(m), RankedPairs(*exact_pairs(m, m, FLOOR))


def _score_thresholds(table, n=2):
    """scores of pairs in the output and the next double below each: the threshold drops the pair, the one below
    keeps it"""
    keep = (table.rank < 20) & (table.row != table.col) & (table.score < 1.0)
    s = np.unique(table.score[keep])
    picks = s[np.linspace(0, len(s) - 1, n).astype(int)] if len(s) else []
    return [t for x in picks for t in (float(x), float(np.nextafter(x, -np.inf)))]


def _run(A, B, top_n, thr, expect, **kw):
    st = {}
    got = _D().cossim_topn(A, B, top_n, thr, stats=st, **kw)
    assert st["kernel"] == "row", st["kernel"]
    for k, v in expect.items():
        assert st.get(k) == v, "path: %s is %r, expected %r" % (k, st.get(k), v)
    return got.host_triples() + (got.max_row,), st


def _group_bytes(A, tiles_per_group, tile_w=128):
    """GROUP_BYTES that gives `tiles_per_group` tiles per group when A is the right matrix as it stands (no merging of
    identical rows)"""
    T = -(-A.shape[0] // tile_w)
    return int(np.ceil((tiles_per_group + 0.5) * max(4 * A.nnz / T, 1)))


@pytest.mark.parametrize("tile_w,residue", [(128, 1), (128, 63), (128, 64), (128, 65), (128, 127), (256, 1),
                                            (256, 127)])
@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_last_pass_of_the_right_matrix(names_matrix, acc, tile_w, residue):
    """two matrices, T = 128 + residue tiles: the last pass holds 1 to 127 real tiles, and T = 129, 191 and 192
    (padded to 192 tiles) have lanes of the last pass past the padding"""
    D = _D()
    T = 128 + residue
    n_right = tile_w * (T - 1) + 77
    right, left = names_matrix[:n_right], names_matrix[n_right:n_right + N_LEFT]
    L, R = D.DeviceCSR.from_scipy(left), D.DeviceCSR.from_scipy(right)
    table = RankedPairs(*exact_pairs(left, right, FLOOR))
    for thr in [0.5] + _score_thresholds(table):
        got, st = _run(L, R, 20, thr, {"acc": acc, "triangle": False, "tile_w": tile_w, "n_tiles": T},
                       acc=acc, tile_w=tile_w, floor=False)
        assert st["tiles_per_group"] >= T, st["tiles_per_group"]
        assert_same(got, table.topn(20, thr), "T=%d W=%d %s thr=%r" % (T, tile_w, acc, thr))


@pytest.mark.parametrize("tiles_per_group", [None, 64, 192])
@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_triangle_ranks_and_groups(self_match, monkeypatch, acc, tiles_per_group):
    """self-match triangle: the first pass of a row starts at the 128-aligned tile below its rank, so ranks fall in
    every quarter of a pass; groups of 64 tiles start mid-pass, groups of 192 end mid-pass"""
    m, A, table = self_match
    D = _D()
    kw = {}
    if tiles_per_group:        # on A itself, so that the group size is known beforehand
        monkeypatch.setattr(D, "GROUP_BYTES", _group_bytes(A, tiles_per_group))
        kw["dedup"] = False
    for thr in [0.5] + _score_thresholds(table):
        got, st = _run(A, A, 20, thr, {"acc": acc, "triangle": True, "tile_w": 128}, acc=acc, tile_w=128,
                       floor=False, **kw)
        assert st["n_tiles"] > 192, st["n_tiles"]
        if tiles_per_group:
            assert st["tiles_per_group"] == tiles_per_group, st["tiles_per_group"]
        assert_same(got, table.topn(20, thr), "triangle %s groups=%r thr=%r" % (acc, tiles_per_group, thr))


@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_wide_tiles_triangle(self_match, acc):
    m, A, table = self_match
    for thr in (0.5, 0.8):
        got, st = _run(A, A, 20, thr, {"acc": acc, "triangle": True, "tile_w": 256}, acc=acc, tile_w=256,
                       floor=False)
        assert_same(got, table.topn(20, thr), "W=256 %s thr=%r" % (acc, thr))


@pytest.mark.parametrize("tiles_per_group", [None, 64])
@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_range_hi_inside_a_pass(self_match, monkeypatch, acc, tiles_per_group):
    """blocked self-match (the position-range kernel): five blocks of random sizes, so every block's end lies
    somewhere inside a pass"""
    import torch
    m, A, table = self_match
    D = _D()
    n = m.shape[0]
    ids = np.random.default_rng(11).choice(5, size=n, p=[0.07, 0.18, 0.2, 0.25, 0.3]).astype(np.int32)
    d = torch.from_numpy(ids).cuda()
    keep = ids[table.row] == ids[table.col]
    blocked = RankedPairs(table.row[keep], table.col[keep], table.score[keep])
    if tiles_per_group:
        monkeypatch.setattr(D, "GROUP_BYTES", _group_bytes(A, tiles_per_group))
    for thr in [0.5] + _score_thresholds(blocked, 1):
        got, st = _run(A, A, 20, thr, {"blocks": True, "acc": acc, "triangle": True, "tile_w": 128}, acc=acc,
                       tile_w=128, block_ids=(d, d))
        if tiles_per_group:
            assert st["tiles_per_group"] == tiles_per_group, st["tiles_per_group"]
        assert_same(got, blocked.topn(20, thr), "blocked %s groups=%r thr=%r" % (acc, tiles_per_group, thr))


@pytest.mark.parametrize("tiles_per_group", [None, 192])
def test_floor_seed_starts_mid_group(self_match, monkeypatch, tiles_per_group):
    """top-n floor self-match: the seed launch walks each row's own group from the pass that holds the row, wrapping
    round to the group's first pass; groups of 192 tiles end in the middle of their second pass"""
    m, A, table = self_match
    D = _D()
    if tiles_per_group:
        monkeypatch.setattr(D, "GROUP_BYTES", _group_bytes(A, tiles_per_group))
    for thr, top_n in ((0.3, 20), (0.5, 5)):
        got, st = _run(A, A, top_n, thr, {"topn_floor": True, "triangle": False, "tile_w": 128}, tile_w=128,
                       floor=True)
        assert st["n_candidates_seed"] > 0 and st["n_tiles"] > 192, st
        if tiles_per_group:
            assert st["tiles_per_group"] == tiles_per_group, st["tiles_per_group"]
        assert_same(got, table.topn(top_n, thr), "floor top %d groups=%r thr=%r" % (top_n, tiles_per_group, thr))


def _long_rows(seed, n_clusters, lengths, n_features=60000):
    """clusters of four near-duplicate rows of exactly L stored features each (L drawn from `lengths`): the base row's
    features with two of them replaced and every weight jittered, L2-normalised; rows shuffled"""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n_clusters):
        L = int(rng.choice(lengths))
        f = rng.choice(n_features, size=L + 8, replace=False)
        w = rng.uniform(0.2, 1.0, size=L)
        for k in range(4):
            g = f[:L].copy()
            if k:
                g[rng.choice(L, size=2, replace=False)] = f[L + 2 * k:L + 2 * k + 2]
            rows.append((g, w * rng.uniform(0.85, 1.15, size=L)))
    order = rng.permutation(len(rows))
    indptr = np.zeros(len(rows) + 1, np.int64)
    indptr[1:] = np.cumsum([len(rows[i][0]) for i in order])
    ind = np.concatenate([rows[i][0] for i in order])
    val = np.concatenate([rows[i][1] / np.linalg.norm(rows[i][1]) for i in order])
    return _csr(csr_matrix((val, ind, indptr), shape=(len(rows), n_features)))


@pytest.mark.parametrize("tile_w", [128, 256])
@pytest.mark.parametrize("acc", ["u16", "f32"])
def test_rows_of_33_64_65_kept_features(acc, tile_w):
    """unpruned rows of 33, 64 and 65 features: the first 32 from registers, then one chunk of 1, 32 or 33 in two"""
    D = _D()
    m = _long_rows(7, 9000, (33, 64, 65))
    A = D.DeviceCSR.from_scipy(m)
    table = RankedPairs(*exact_pairs(m, m, FLOOR))
    for thr in [0.5] + _score_thresholds(table):
        got, st = _run(A, A, 20, thr, {"acc": acc, "triangle": True, "tile_w": tile_w}, acc=acc, tile_w=tile_w,
                       prune=0.0, floor=False)
        assert st["n_rows_long"] == m.shape[0] and st["n_tiles"] > 128, st
        assert_same(got, table.topn(20, thr), "long rows self-match %s W=%d thr=%r" % (acc, tile_w, thr))
    left, right = m[:3000], m[3000:]
    L, R = D.DeviceCSR.from_scipy(left), D.DeviceCSR.from_scipy(right)
    got, st = _run(L, R, 20, 0.5, {"acc": acc, "triangle": False, "tile_w": tile_w}, acc=acc, tile_w=tile_w,
                   prune=0.0, floor=False)
    assert st["n_rows_long"] == 3000, st["n_rows_long"]
    assert_same(got, exact_topn(left, right, 20, 0.5), "long rows two matrices %s W=%d" % (acc, tile_w))

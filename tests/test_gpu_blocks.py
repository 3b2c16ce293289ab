"""-m gpu: the blocked top-n product (cossim_topn's block_ids, the blocking keys of the public API) against an exact
specification.  Every device case compares rows, columns, scores bit for bit, the output order and max_row with
np.array_equal (tests/exact_topn.assert_same), and asserts from `stats` which path ran."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix

from exact_topn import RankedPairs, assert_same, exact_pairs
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

FLOOR = 0.3                  # every threshold below lies at or above this
N_NAMES = 6000
CLUSTER = 320                # identical names, split across two keys by the "cluster" layout
N_LEFT = 4000                # two matrices: the first N_LEFT rows against the rest
TOP_NS = (1, 20, 33, 512, 2048)


def _D():
    from string_grouper_b200 import _device as D
    return D


def blocked_exact(pairs, ids_a, ids_b):
    """The specification of the blocked product: the exact pairs (tests/exact_topn.exact_pairs) without the pairs of
    different block ids, ranked by the usual top-n rule; .topn(top_n, threshold) gives (row, col, score, max_row)."""
    r, c, s = pairs
    keep = ids_a[r] == ids_b[c]
    return RankedPairs(r[keep], c[keep], s[keep])


def _names():
    names = make_names(N_NAMES, seed=31)
    return names + [names[7]] * CLUSTER


def _layout(kind, n, seed=0):
    """int32 block id per row for the key layouts of the tests"""
    rng = np.random.default_rng(seed)
    if kind == "one":
        return np.zeros(n, np.int32)
    if kind == "own":
        return np.arange(n, dtype=np.int32)
    if kind == "small":                                   # about 40 rows per key: many keys inside one tile
        return rng.integers(0, n // 40, size=n).astype(np.int32)
    if kind == "edges":                                   # keys of 255, 256 and 257 rows: block edges at tile edges
        sizes = np.resize([256, 256, 255, 257, 256, 1, 255, 257], n)
        ids = np.repeat(np.arange(len(sizes)), sizes)[:n]
        return ids[rng.permutation(n)].astype(np.int32)
    if kind == "cluster":                                 # the identical names split across keys 0 and 1
        ids = rng.integers(2, 6, size=n).astype(np.int32)
        cl = np.arange(n - CLUSTER, n)
        ids[cl] = rng.integers(0, 2, size=CLUSTER)
        ids[7] = 0
        return ids
    if kind == "missing":                                 # a fifth of the keys missing: one fresh id each
        from string_grouper_b200.string_grouper import block_ids_of
        keys = pd.Series(rng.choice(["US", "FR", "DE"], size=n), dtype=object)
        keys[rng.random(n) < 0.2] = None
        return block_ids_of(pd.Series(["x"] * n), None, keys)
    raise ValueError(kind)


LAYOUTS = ("one", "own", "small", "edges", "cluster", "missing")


@pytest.fixture(scope="module")
def corpus():
    """dtype -> (host matrix, device matrix, device left block, device right block, self pairs, cross pairs)"""
    from oracle import pipeline as P
    D = _D()
    out = {}
    for dtype in (np.float64, np.float32):
        m, _, _ = P.tf_idf_matrices(_names(), dtype=dtype)
        m = csr_matrix(m).astype(dtype)
        m.sort_indices()
        A = D.DeviceCSR.from_scipy(m)
        L = D.DeviceCSR.from_scipy(m[:N_LEFT])
        R = D.DeviceCSR.from_scipy(m[N_LEFT:])
        host, hl, hr = A.to_scipy(), L.to_scipy(), R.to_scipy()
        out[dtype] = (host, A, L, R, exact_pairs(host, host, FLOOR), exact_pairs(hl, hr, FLOOR))
    return out


def _ids(ids):
    import torch
    return torch.from_numpy(ids).cuda()


def _run(A, B, ids_a, ids_b, top_n, thr, expect, **kw):
    st = {}
    got = _D().cossim_topn(A, B, top_n, thr, stats=st, block_ids=(ids_a, ids_b), **kw)
    for k, v in expect.items():
        assert st.get(k) == v, "path: %s is %r, expected %r" % (k, st.get(k), v)
    return got.host_triples() + (got.max_row,), st


def _score_thresholds(table):
    """pair scores in (FLOOR, 1) and the next double below each: the threshold drops the pair, the one below keeps it"""
    s = np.unique(table.score[(table.rank < 20) & (table.row != table.col) & (table.score < 1.0)])
    picks = s[np.linspace(0, len(s) - 1, 4).astype(int)] if len(s) else []
    return [t for x in picks for t in (float(x), float(np.nextafter(x, -np.inf)))]


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("mode", ["self", "two"])
def test_blocked_product_exact(corpus, dtype, layout, mode):
    host, A, L, R, self_pairs, cross_pairs = corpus[dtype]
    ids = _layout(layout, host.shape[0])
    if mode == "self":
        d = _ids(ids)
        left, right, ia, ib, ha, hb, pairs = A, A, d, d, ids, ids, self_pairs
    else:
        left, right, ia, ib = L, R, _ids(ids[:N_LEFT]), _ids(ids[N_LEFT:])
        ha, hb, pairs = ids[:N_LEFT], ids[N_LEFT:], cross_pairs
    table = blocked_exact(pairs, ha, hb)
    n_used = len(np.unique(ids))
    expect = {"blocks": True, "triangle": mode == "self", "topn_floor": False, "dedup": False, "kernel": "row",
              "n_blocks_used": n_used}
    for thr in [0.3, 0.6, 0.8] + _score_thresholds(table):
        for top_n in (TOP_NS if thr in (0.3, 0.8) else (20,)):
            got, _ = _run(left, right, ia, ib, top_n, thr, expect)
            assert_same(got, table.topn(top_n, thr), "%s %s top %d thr %r" % (layout, mode, top_n, thr))


@pytest.mark.parametrize("acc", ["u16", "f32"])
@pytest.mark.parametrize("refine", [True, False])
@pytest.mark.parametrize("layout", ["small", "cluster"])
def test_blocked_accumulators_and_refine(corpus, monkeypatch, acc, refine, layout):
    D = _D()
    monkeypatch.setattr(D, "REFINE", refine)
    host, A, _, _, pairs, _ = corpus[np.float64]
    ids = _layout(layout, host.shape[0], seed=4)
    d = _ids(ids)
    table = blocked_exact(pairs, ids, ids)
    for thr in (0.6, 0.8):
        got, st = _run(A, A, d, d, 20, thr, {"blocks": True, "acc": acc, "triangle": True}, acc=acc)
        assert ("n_refined" in st) == (refine and acc == "u16")
        assert_same(got, table.topn(20, thr), "%s %s refine=%s" % (layout, acc, refine))


def test_blocked_row_chunks_and_retry(corpus, monkeypatch):
    D = _D()
    host, A, L, R, pairs, cross = corpus[np.float64]
    ids = _layout("cluster", host.shape[0], seed=9)
    d = _ids(ids)
    want = blocked_exact(pairs, ids, ids).topn(20, 0.3)
    monkeypatch.setattr(D, "CAND_CHUNK", 20_000)             # the first launch overflows: chunks from its count
    got, st = _run(A, A, d, d, 20, 0.3, {"blocks": True, "triangle": True})
    assert st["n_row_chunks"] > 1
    assert_same(got, want, "row chunks")
    monkeypatch.setattr(D, "CAND_CHUNK", 1 << 28)
    monkeypatch.setenv("SG_B200_CAND_CAP", "1000")            # too small: the launch is repeated with the count
    before = D.LAUNCH_COUNTS["candidates"]
    got, st = _run(A, A, d, d, 20, 0.3, {"blocks": True})
    assert D.LAUNCH_COUNTS["candidates"] - before >= 2 and st["n_candidates"] > 1000
    assert_same(got, want, "retry")
    got, _ = _run(L, R, _ids(ids[:N_LEFT]), _ids(ids[N_LEFT:]), 20, 0.3, {"blocks": True, "triangle": False})
    assert_same(got, blocked_exact(cross, ids[:N_LEFT], ids[N_LEFT:]).topn(20, 0.3), "retry, two matrices")


def test_blocked_key_spanning_column_tile_groups(monkeypatch):
    """one key of 17 000 rows over three groups of 64 column tiles (8 192 positions each), next to small keys"""
    from oracle import pipeline as P
    D = _D()
    monkeypatch.setattr(D, "GROUP_BYTES", 1)                 # the smallest groups: 64 tiles
    m, _, _ = P.tf_idf_matrices(make_names(24000, seed=12))
    m = csr_matrix(m)
    m.sort_indices()
    A = D.DeviceCSR.from_scipy(m)
    host = A.to_scipy()
    rng = np.random.default_rng(3)
    ids = np.where(rng.random(host.shape[0]) < 0.7, 0, rng.integers(1, 50, size=host.shape[0])).astype(np.int32)
    d = _ids(ids)
    table = blocked_exact(exact_pairs(host, host, 0.6), ids, ids)
    for thr in (0.6, 0.8):
        got, st = _run(A, A, d, d, 20, thr, {"blocks": True, "triangle": True}, tile_w=128)
        assert st["tiles_per_group"] == 64 and -(-st["n_tiles"] // 64) == 3
        assert_same(got, table.topn(20, thr), "groups thr %r" % thr)


def test_unblocked_caches_survive_a_keyed_call(corpus):
    D = _D()
    host, A, _, _, _, _ = corpus[np.float64]
    first = D.cossim_topn(A, A, 20, 0.6).host_triples()
    built = D.LAUNCH_COUNTS["postings"]
    d = _ids(_layout("small", host.shape[0]))
    st = {}
    D.cossim_topn(A, A, 20, 0.6, stats=st, block_ids=(d, d))
    assert st["blocks"] and D.LAUNCH_COUNTS["postings"] > built          # the blocked order has postings of its own
    built = D.LAUNCH_COUNTS["postings"]
    D.cossim_topn(A, A, 20, 0.6, block_ids=(d, d))
    assert D.LAUNCH_COUNTS["postings"] == built                          # ... cached under the id tensor
    st = {}
    again = D.cossim_topn(A, A, 20, 0.6, stats=st).host_triples()
    assert not st["blocks"] and D.LAUNCH_COUNTS["postings"] == built     # the unblocked caches were reused
    for x, y in zip(first, again):
        assert np.array_equal(x, y)


def test_blocked_argument_checks(corpus):
    D = _D()
    host, A, L, R, _, _ = corpus[np.float64]
    d = _ids(np.zeros(host.shape[0], np.int32))
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 20, 0.3, block_ids=(d, d), floor=True)
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 20, 0.8, block_ids=(d, d), kernel="tiles")
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 20, 0.8, block_ids=(d, d), dedup=True)
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 20, 0.8, block_ids=(d[:10], d[:10]))
    with pytest.raises(ValueError):
        D.cossim_topn(A, A, 20, 0.8, block_ids=(d.long(), d.long()))


def test_env_tiles_kernel_falls_back_to_rows(corpus, monkeypatch):
    D = _D()
    monkeypatch.setattr(D, "K2_KERNEL", "tiles")
    host, A, _, _, pairs, _ = corpus[np.float64]
    ids = _layout("edges", host.shape[0])
    d = _ids(ids)
    got, _ = _run(A, A, d, d, 20, 0.8, {"blocks": True, "kernel": "row"})
    assert_same(got, blocked_exact(pairs, ids, ids).topn(20, 0.8), "env tiles")


# ---------------------------------------------------------------------------------------------------------------
# public API: 20k names with seeded keys
# ---------------------------------------------------------------------------------------------------------------
N_API = 20000


@pytest.fixture(scope="module")
def api_data():
    names = pd.Series(make_names(N_API, seed=8))
    rng = np.random.default_rng(8)
    keys = pd.Series(rng.choice([f"k{i}" for i in range(12)], size=N_API))
    return names, keys


def _assert_equal(a, b):
    if isinstance(a, pd.DataFrame):
        pd.testing.assert_frame_equal(a, b)
    else:
        pd.testing.assert_series_equal(a, b)


def _same_key_rows(frame, lkeys, rkeys, lcol="left_index", rcol="right_index"):
    return lkeys[frame[lcol].to_numpy()] == rkeys[frame[rcol].to_numpy()]


def test_api_one_key_is_the_unkeyed_call(api_data):
    from string_grouper_b200 import StringGrouper, group_similar_strings, match_most_similar, match_strings
    names, _ = api_data
    one = pd.Series(["all"] * N_API)
    sg_k = StringGrouper(names, master_keys=one).fit()
    sg_u = StringGrouper(names).fit()
    assert sg_k._last_stats["blocks"] and sg_k._last_stats["n_blocks_used"] == 1
    assert not sg_u._last_stats["blocks"]
    pd.testing.assert_frame_equal(sg_k._matches_list, sg_u._matches_list)
    assert sg_k._true_max_n_matches == sg_u._true_max_n_matches
    pd.testing.assert_frame_equal(match_strings(names, master_keys=one), match_strings(names))
    _assert_equal(group_similar_strings(names, keys=one), group_similar_strings(names))
    master, dupes = names[:12000], names[12000:].reset_index(drop=True)
    pd.testing.assert_frame_equal(
        match_strings(master, dupes, master_keys=one[:12000], duplicates_keys=one[12000:], min_similarity=0.6),
        match_strings(master, dupes, min_similarity=0.6))
    _assert_equal(match_most_similar(master, dupes, master_keys=one[:12000], duplicates_keys=one[12000:]),
                  match_most_similar(master, dupes))


def test_api_large_top_n_is_the_filtered_unkeyed_call(api_data):
    from string_grouper_b200 import group_similar_strings, match_strings
    names, keys = api_data
    k = keys.to_numpy()
    big = 4000
    for thr in (0.6, 0.8):
        got = match_strings(names, master_keys=keys, max_n_matches=big, min_similarity=thr)
        full = match_strings(names, max_n_matches=big, min_similarity=thr)
        want = full[_same_key_rows(full, k, k)].reset_index(drop=True)
        pd.testing.assert_frame_equal(got, want)
    master, dupes = names[:12000], names[12000:].reset_index(drop=True)
    mk, dk = keys[:12000], keys[12000:].reset_index(drop=True)
    got = match_strings(master, dupes, master_keys=mk, duplicates_keys=dk, max_n_matches=big, min_similarity=0.6)
    full = match_strings(master, dupes, max_n_matches=big, min_similarity=0.6)
    want = full[_same_key_rows(full, mk.to_numpy(), dk.to_numpy())].reset_index(drop=True)
    pd.testing.assert_frame_equal(got, want)
    groups = group_similar_strings(names, keys=keys, min_similarity=0.6)
    rep_pos = groups["group_rep_index"].to_numpy()                    # RangeIndex: labels are positions
    assert np.array_equal(k[rep_pos], k)                              # no group crosses a key


def test_api_keys_aligned_by_position_and_checked(api_data):
    from string_grouper_b200 import StringGrouper, match_strings
    names, keys = api_data
    small = names[:3000]
    shuffled = pd.Series(keys[:3000].to_numpy(), index=np.arange(3000)[::-1])   # index ignored: by position
    pd.testing.assert_frame_equal(match_strings(small, master_keys=shuffled),
                                  match_strings(small, master_keys=keys[:3000]))
    with pytest.raises(ValueError):
        match_strings(small, master_keys=keys[:10])
    with pytest.raises(ValueError):
        match_strings(small, duplicates_keys=keys[:3000])
    with pytest.raises(ValueError):
        match_strings(small, names[3000:4000], master_keys=keys[:3000])
    with pytest.raises(ValueError):
        match_strings(small, names[3000:4000], duplicates_keys=keys[:1000])
    sg = StringGrouper(small, master_keys=keys[:3000])
    sg.reset_data(small)                                               # keys go with the data
    assert sg.fit()._last_stats["blocks"] is False


# ---------------------------------------------------------------------------------------------------------------
# full size: the 663k benchmark names
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    from string_grouper_b200 import StringGrouper
    names = pd.Series(make_names(663_000, seed=0))
    A, _ = StringGrouper(names)._get_tf_idf_matrices()
    st = {}
    # the unkeyed product over every row: the keyed one does not take the identical-rows dedup, which the default
    # takes on this corpus (its candidates are those of the distinct rows)
    _D().cossim_topn(A, A, 20, 0.8, stats=st, dedup=False)
    return A, st["n_candidates"]


@pytest.mark.parametrize("n_keys", [50, 5000])
def test_full_size_blocked_sampled_rows(full, n_keys):
    D = _D()
    A, unblocked_candidates = full
    n = A.shape[0]
    ids = np.random.default_rng(n_keys).integers(0, n_keys, size=n).astype(np.int32)
    d = _ids(ids)
    got, st = _run(A, A, d, d, 20, 0.8, {"blocks": True, "triangle": True, "topn_floor": False, "dedup": False,
                                         "n_blocks_used": n_keys})
    assert st["n_candidates"] < unblocked_candidates
    r, c, s, _ = got
    host = A.to_scipy()
    rows = np.sort(np.random.default_rng(1).choice(n, size=2000, replace=False))
    pr, pc, ps = exact_pairs(host[rows], host, 0.8, block_rows=200)
    pr = rows[pr]
    want = blocked_exact((pr, pc, ps), ids, ids).topn(20, 0.8)
    sel = np.isin(r, rows)
    assert_same((r[sel], c[sel], s[sel]), want[:3], "663k, %d keys" % n_keys)

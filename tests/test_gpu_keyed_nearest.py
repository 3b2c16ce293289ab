"""-m gpu: the keyed arg-max (cossim_nearest's block_ids, match_nearest's blocking keys, keyed StringGrouperCorpus)
against an exact specification: tests/exact_nearest.py's arg-max over the exact pairs without the pairs of different
block ids.  Every device case compares the best column and its score bit for bit (np.array_equal), and asserts from
`stats` which path ran, the top-n floor included (sg_cossim_candidates_range_floor)."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix

from exact_nearest import nearest_from_pairs
from exact_topn import exact_pairs
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

N_NAMES = 6000
CLUSTER = 320                # identical names, split across two keys by the "cluster" layout
N_LEFT = 4000                # two matrices: the first N_LEFT rows (duplicates) against the rest (masters)
THRESHOLDS = (0.8, 0.3, 0.0)


def _D():
    from string_grouper_b200 import _device as D
    return D


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


def _ids(ids):
    import torch
    return torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int32)).cuda()


def keyed_nearest(pairs, ids_a, ids_b, thr, n_rows):
    """the specification: per left row the arg-max over the exact pairs above thr whose two ids are equal"""
    r, c, s = pairs
    keep = (ids_a[r] == ids_b[c]) & (s > thr)
    return nearest_from_pairs(r[keep], c[keep], s[keep], n_rows)


def keyed_nearest_rows(left, right, ids_a, ids_b, rows=None, block=500):
    """keyed_nearest at 0 for `rows` of left (default all) against right, the pairs of `block` rows at a time, reduced
    before the next block is formed"""
    rows = np.arange(left.shape[0]) if rows is None else rows
    best, score = np.full(len(rows), -1, np.int64), np.zeros(len(rows))
    for lo in range(0, len(rows), block):
        part = rows[lo:lo + block]
        b, sc = keyed_nearest(exact_pairs(left[part], right, 0.0), ids_a[part], ids_b, 0.0, len(part))
        best[lo:lo + len(part)], score[lo:lo + len(part)] = b, sc
    return best, score


def at_threshold(best0, thr):
    """keyed_nearest at thr from keyed_nearest at 0: a row's best pair passes thr or none of its pairs does"""
    best, score = best0
    hit = score > thr
    return np.where(hit, best, -1), np.where(hit, score, 0.0)


@pytest.fixture(scope="module")
def corpus():
    """dtype -> (host matrix, device matrix, device left block, device right block, self pairs, cross pairs), the
    pairs above 0 (every pair with a positive score)"""
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
        out[dtype] = (host, A, L, R, exact_pairs(host, host, 0.0), exact_pairs(hl, hr, 0.0))
    return out


def _case(corpus, dtype, layout, mode, seed=0):
    """(left, right, device ids pair, host ids pair, pairs) of one layout: 'self' one matrix and one id tensor,
    'two' the duplicates block against the masters block"""
    host, A, L, R, self_pairs, cross_pairs = corpus[dtype]
    ids = _layout(layout, host.shape[0], seed)
    if mode == "self":
        d = _ids(ids)
        return A, A, (d, d), (ids, ids), self_pairs
    return L, R, (_ids(ids[:N_LEFT]), _ids(ids[N_LEFT:])), (ids[:N_LEFT], ids[N_LEFT:]), cross_pairs


def _run(A, B, thr, block_ids, expect, **kw):
    st = {}
    got = _D().cossim_nearest(A, B, thr, stats=st, block_ids=block_ids, **kw)
    for k, v in expect.items():
        assert st.get(k) == v, "path: %s is %r, expected %r" % (k, st.get(k), v)
    return got, st


def _assert_same(got, want, label):
    assert np.array_equal(got[0], want[0]), "%s: best columns differ at %s" % (
        label, np.flatnonzero(got[0] != want[0])[:10])
    assert np.array_equal(got[1], want[1]), "%s: scores differ" % label


def _score_thresholds(best0):
    """row-best scores in (0, 1) and the next double below each: the threshold drops the pair, the one below keeps it"""
    best, score = best0
    s = np.unique(score[(best >= 0) & (score < 1.0)])
    picks = s[np.linspace(0, len(s) - 1, 3).astype(int)] if len(s) else []
    return [t for x in picks for t in (float(x), float(np.nextafter(x, -np.inf)))]


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("mode", ["self", "two"])
def test_keyed_nearest_exact(corpus, dtype, layout, mode):
    left, right, d_ids, (ha, hb), pairs = _case(corpus, dtype, layout, mode)
    n_used = len(np.unique(np.concatenate([ha, hb])))
    best0 = keyed_nearest(pairs, ha, hb, 0.0, left.shape[0])
    for thr in THRESHOLDS + tuple(_score_thresholds(best0)):
        want = at_threshold(best0, thr)
        for floor in (False, True):
            got, st = _run(left, right, thr, d_ids, {"blocks": True, "nearest": True, "topn_floor": floor,
                                                     "n_blocks_used": n_used}, floor=floor)
            _assert_same(got, want, "%s %s thr %r floor %s" % (layout, mode, thr, floor))


@pytest.mark.parametrize("layout", ["small", "cluster"])
def test_one_matrix_with_two_key_columns(corpus, layout):
    """the same matrix on both sides with different ids for the two sides (a corpus looked up against itself under
    other keys): no triangle, no self-match seed"""
    host, A, _, _, pairs, _ = corpus[np.float64]
    ia, ib = _layout(layout, host.shape[0], 1), _layout(layout, host.shape[0], 2)
    best0 = keyed_nearest(pairs, ia, ib, 0.0, host.shape[0])
    for thr in (0.3, 0.0):
        want = at_threshold(best0, thr)
        for floor in (False, True):
            got, _ = _run(A, A, thr, (_ids(ia), _ids(ib)), {"blocks": True, "topn_floor": floor}, floor=floor)
            _assert_same(got, want, "two key columns %s thr %r floor %s" % (layout, thr, floor))


@pytest.mark.parametrize("acc", ["u16", "f32"])
@pytest.mark.parametrize("refine", [True, False])
@pytest.mark.parametrize("mode", ["self", "two"])
def test_accumulators_and_refine(corpus, monkeypatch, acc, refine, mode):
    D = _D()
    monkeypatch.setattr(D, "REFINE", refine)
    left, right, d_ids, (ha, hb), pairs = _case(corpus, np.float64, "cluster", mode, seed=4)
    best0 = keyed_nearest(pairs, ha, hb, 0.0, left.shape[0])
    for thr in (0.8, 0.6, 0.3):
        want = at_threshold(best0, thr)
        for floor in (False, True):
            got, st = _run(left, right, thr, d_ids, {"blocks": True, "topn_floor": floor}, acc=acc, floor=floor)
            _assert_same(got, want, "%s refine=%s thr %r floor %s" % (acc, refine, thr, floor))
            if thr >= 0.6:          # the fixed-point tile needs a candidate threshold of at least 0.05
                assert st["acc"] == acc and ("n_refined" in st) == (refine and acc == "u16")


def test_floor_auto_and_default(corpus):
    left, right, d_ids, (ha, hb), pairs = _case(corpus, np.float64, "small", "two")
    best0 = keyed_nearest(pairs, ha, hb, 0.0, left.shape[0])
    for thr in (0.3, 0.0):
        want = at_threshold(best0, thr)
        for floor in ("auto", None):        # below FLOOR_MIN_ROWS rows auto keeps the usual path
            got, _ = _run(left, right, thr, d_ids, {"blocks": True, "topn_floor": False}, floor=floor)
            _assert_same(got, want, "floor %r thr %r" % (floor, thr))


def test_row_chunks_and_buffer_retry(corpus, monkeypatch):
    D = _D()
    for mode in ("self", "two"):
        left, right, d_ids, (ha, hb), pairs = _case(corpus, np.float64, "cluster", mode, seed=9)
        want = keyed_nearest(pairs, ha, hb, 0.3, left.shape[0])
        # a self-match's seed walks the row's own column-tile group unchunked: here that is every tile
        for floor in ((False, True) if mode == "two" else (False,)):
            _, st = _run(left, right, 0.3, d_ids, {"blocks": True, "topn_floor": floor}, floor=floor)
            # a quarter of the candidates the launches over all rows find: the first launch overflows, chunks follow
            n = st["n_candidates_main"] if floor else st["n_candidates"]
            monkeypatch.setattr(D, "CAND_CHUNK", max(n // 4, 1))
            got, st = _run(left, right, 0.3, d_ids, {"blocks": True, "topn_floor": floor}, floor=floor)
            monkeypatch.setattr(D, "CAND_CHUNK", 1 << 28)
            assert st["n_row_chunks"] > 1
            _assert_same(got, want, "row chunks %s floor %s" % (mode, floor))
        monkeypatch.setattr(D, "CAND_CHUNK", 1 << 28)
        monkeypatch.setenv("SG_B200_CAND_CAP", "1000")        # too small: the launch is repeated with the count
        before = D.LAUNCH_COUNTS["candidates"]
        got, st = _run(left, right, 0.3, d_ids, {"blocks": True, "topn_floor": False}, floor=False)
        assert D.LAUNCH_COUNTS["candidates"] - before >= 2 and st["n_candidates"] > 1000
        _assert_same(got, want, "retry %s" % mode)
        monkeypatch.delenv("SG_B200_CAND_CAP")


@pytest.fixture(scope="module")
def mid_group_keys():
    """48 000 names over 375 column tiles of 128 positions: key 0 holds 60 % of the rows (positions 0 .. 28 800), key 1
    30 % (28 800 .. 43 200, tiles 225 .. 337), 40 small keys the rest.  So key 1 starts more than 128 tiles into the first
    column-tile group and spans two of its 128-tile passes.  (device matrix, host ids, keyed self-match at 0)"""
    from oracle import pipeline as P
    D = _D()
    m, _, _ = P.tf_idf_matrices(make_names(48000, seed=13))
    m = csr_matrix(m)
    m.sort_indices()
    A = D.DeviceCSR.from_scipy(m)
    host = A.to_scipy()
    rng = np.random.default_rng(13)
    u = rng.random(host.shape[0])
    ids = np.where(u < 0.6, 0, np.where(u < 0.9, 1, rng.integers(2, 42, size=host.shape[0]))).astype(np.int32)
    return A, ids, keyed_nearest_rows(host, host, ids, ids)


def test_seed_starts_past_the_group_start(mid_group_keys, monkeypatch):
    """a self-match's seed with one large column-tile group: key 1's rows start their walk at the pass that holds
    their own position, counted from their first pass (tile 128), not from the group's first tile"""
    D = _D()
    A, ids, best0 = mid_group_keys
    monkeypatch.setattr(D, "GROUP_BYTES", 1 << 32)           # one group of every tile
    d = _ids(ids)
    for thr in (0.3, 0.0):
        got, st = _run(A, A, thr, (d, d), {"blocks": True, "topn_floor": True}, tile_w=128, floor=True)
        assert st["n_tiles"] > 256 and st["tiles_per_group"] >= st["n_tiles"]
        assert st["n_candidates_main"] == 0                  # one group: the seed walks every tile
        _assert_same(got, at_threshold(best0, thr), "seed past the group start thr %r" % thr)


def test_floor_row_chunks_and_retry_in_a_self_match(mid_group_keys, monkeypatch):
    """the keyed self-match with the floor over 64-tile groups: the seed and the main launches overflow a small
    buffer and are repeated with their count, the main launches then run in row chunks"""
    D = _D()
    A, ids, best0 = mid_group_keys
    monkeypatch.setattr(D, "GROUP_BYTES", 1)                 # the smallest groups: 64 tiles
    d = _ids(ids)
    _, st = _run(A, A, 0.3, (d, d), {"blocks": True, "topn_floor": True}, tile_w=128, floor=True)
    assert -(-st["n_tiles"] // st["tiles_per_group"]) > 1 and st["n_candidates_main"] > 0
    monkeypatch.setattr(D, "CAND_CHUNK", max(min(st["n_candidates_seed"], st["n_candidates_main"]) // 4, 1))
    before = D.LAUNCH_COUNTS["candidates"]
    got, st = _run(A, A, 0.3, (d, d), {"blocks": True, "topn_floor": True}, tile_w=128, floor=True)
    # the seed twice, the first main launch over all rows (it overflows), then one launch per chunk at least
    assert st["n_row_chunks"] > 1
    assert D.LAUNCH_COUNTS["candidates"] - before >= 3 + st["n_row_chunks"]
    _assert_same(got, at_threshold(best0, 0.3), "self-match floor chunks")


def test_key_spanning_column_tile_groups(monkeypatch):
    """one key of 17 000 rows over three groups of 64 column tiles (8 192 positions each), next to small keys"""
    from oracle import pipeline as P
    D = _D()
    monkeypatch.setattr(D, "GROUP_BYTES", 1)                 # the smallest groups: 64 tiles
    m, _, _ = P.tf_idf_matrices(make_names(24000, seed=12))
    m = csr_matrix(m)
    m.sort_indices()
    A = D.DeviceCSR.from_scipy(m)
    L = D.DeviceCSR.from_scipy(m[:3000])
    host, hl = A.to_scipy(), L.to_scipy()
    rng = np.random.default_rng(3)
    ids = np.where(rng.random(host.shape[0]) < 0.7, 0, rng.integers(1, 50, size=host.shape[0])).astype(np.int32)
    self0 = keyed_nearest(exact_pairs(host, host, 0.0), ids, ids, 0.0, host.shape[0])
    cross0 = keyed_nearest(exact_pairs(hl, host, 0.0), ids[:3000], ids, 0.0, 3000)
    d = _ids(ids)
    for thr in (0.8, 0.3, 0.0):
        for floor in (False, True):
            got, st = _run(A, A, thr, (d, d), {"blocks": True, "topn_floor": floor}, tile_w=128, floor=floor)
            assert st["tiles_per_group"] == 64 and -(-st["n_tiles"] // 64) == 3
            _assert_same(got, at_threshold(self0, thr), "self thr %r" % thr)
            got, _ = _run(L, A, thr, (_ids(ids[:3000]), d), {"blocks": True, "topn_floor": floor}, tile_w=128,
                          floor=floor)
            _assert_same(got, at_threshold(cross0, thr), "two thr %r" % thr)


def test_renumbered_ids_give_identical_output(corpus):
    left, right, _, (ha, hb), _ = _case(corpus, np.float64, "cluster", "two", seed=6)
    rng = np.random.default_rng(6)
    uniq = np.unique(np.concatenate([ha, hb]))
    image = rng.choice(2**31 - 1, size=len(uniq), replace=False).astype(np.int32)     # any bijection
    ra, rb = image[np.searchsorted(uniq, ha)], image[np.searchsorted(uniq, hb)]
    for thr in (0.3, 0.0):
        for floor in (False, True):
            a, _ = _run(left, right, thr, (_ids(ha), _ids(hb)), {}, floor=floor)
            b, _ = _run(left, right, thr, (_ids(ra), _ids(rb)), {}, floor=floor)
            _assert_same(a, b, "renumbered thr %r floor %s" % (thr, floor))


def test_topn_floor_with_block_ids_stays_refused_for_top_n(corpus):
    host, A, _, _, _, _ = corpus[np.float64]
    d = _ids(np.zeros(host.shape[0], np.int32))
    with pytest.raises(ValueError):
        _D().cossim_topn(A, A, 20, 0.3, block_ids=(d, d), floor=True)


# ---------------------------------------------------------------------------------------------------------------
# public API: keyed match_nearest and the keyed corpus
# ---------------------------------------------------------------------------------------------------------------
N_API = 20000


@pytest.fixture(scope="module")
def api_data():
    names = pd.Series(make_names(N_API, seed=8))
    rng = np.random.default_rng(8)
    keys = pd.Series(rng.choice([f"k{i}" for i in range(12)] + [None], size=N_API), dtype=object)
    return names, keys


def _assert_equal(a, b):
    (pd.testing.assert_frame_equal if isinstance(a, pd.DataFrame) else pd.testing.assert_series_equal)(a, b)


def _relation(lkeys, rkeys):
    """host ids of two key Series with the relation of blocking keys (equal present values; missing matches none)"""
    from string_grouper_b200.string_grouper import block_ids_of
    ids = block_ids_of(pd.Series(["x"] * len(lkeys)), pd.Series(["x"] * len(rkeys)), lkeys, rkeys)
    return ids[:len(lkeys)], ids[len(lkeys):]


def test_corpus_register_lookup_keyed(api_data):
    import string_grouper_b200 as api
    D = _D()
    names, keys = api_data
    register, rkeys = names[:15000], keys[:15000]
    batch = pd.Series([n + "s" for n in names[15000:17000]] + list(names[17000:]))
    bkeys = keys[15000:].reset_index(drop=True).copy()
    bkeys.iloc[:100] = "unknown key"                              # a key the register does not have
    corpus = api.StringGrouperCorpus(register, keys=rkeys)
    M, Mb = corpus._matrices(register, batch, {})
    ids_r, ids_b = _relation(rkeys, bkeys)
    want0 = keyed_nearest(exact_pairs(Mb.to_scipy(), M.to_scipy(), 0.0), ids_b, ids_r, 0.0, len(batch))
    for thr in THRESHOLDS:
        # match_nearest on the same matrices with the same key relation, numbered by a per-call factorisation
        st = {}
        best, _ = D.cossim_nearest(Mb, M, thr, stats=st, block_ids=(_ids(ids_b), _ids(ids_r)))
        assert st["blocks"]
        assert np.array_equal(best, at_threshold(want0, thr)[0])
        got = corpus.match_nearest(register, batch, duplicates_keys=bkeys, min_similarity=thr)
        _assert_equal(got, api.StringGrouper(register, batch)._nearest_frame(best, False, False))
        assert got["most_similar_index"][:100].isna().all()
        # a second call reuses the register's blocked order and postings
        before = dict(D.LAUNCH_COUNTS)
        again = corpus.match_nearest(register, batch, duplicates_keys=bkeys, min_similarity=thr)
        assert D.LAUNCH_COUNTS["postings"] == before["postings"]
        _assert_equal(again, got)


def test_keyed_corpus_equals_the_keyed_module_functions(api_data):
    import string_grouper_b200 as api
    names, keys = api_data
    m, d = names[:12000], names[12000:].reset_index(drop=True)
    mk, dk = keys[:12000], keys[12000:].reset_index(drop=True)
    whole = pd.concat([m, d], ignore_index=True)
    wkeys = pd.concat([mk, dk], ignore_index=True)
    corpus = api.StringGrouperCorpus(whole, keys=wkeys)
    for thr in (0.8, 0.5):
        kw = dict(master_keys=mk, duplicates_keys=dk, min_similarity=thr)
        _assert_equal(corpus.match_strings(m, d, **kw), api.match_strings(m, d, **kw))
        _assert_equal(corpus.match_nearest(m, d, **kw), api.match_nearest(m, d, **kw))
        _assert_equal(corpus.match_most_similar(m, d, **kw), api.match_most_similar(m, d, **kw))
        _assert_equal(corpus.group_similar_strings(whole, min_similarity=thr),
                      api.group_similar_strings(whole, keys=wkeys, min_similarity=thr))
        _assert_equal(corpus.match_strings(whole, min_similarity=thr),
                      api.match_strings(whole, master_keys=wkeys, min_similarity=thr))


def test_match_nearest_one_key_is_the_unkeyed_call(api_data):
    import string_grouper_b200 as api
    names, _ = api_data
    m, d = names[:12000], names[12000:].reset_index(drop=True)
    one_m, one_d = pd.Series(["all"] * len(m)), pd.Series(["all"] * len(d))
    for thr in THRESHOLDS:
        _assert_equal(api.match_nearest(m, d, master_keys=one_m, duplicates_keys=one_d, min_similarity=thr),
                      api.match_nearest(m, d, min_similarity=thr))


# ---------------------------------------------------------------------------------------------------------------
# config-4 shape (400k masters x 150k duplicates), seeded keys, sampled rows
# ---------------------------------------------------------------------------------------------------------------

def test_config4_shape_keyed_on_sampled_rows():
    from string_grouper_b200 import StringGrouper
    D = _D()
    base = make_names(480_000, seed=3)
    master, dupes = pd.Series(base[:400_000]), pd.Series(base[330_000:480_000])
    M, Dm = StringGrouper(master, duplicates=dupes)._get_tf_idf_matrices(shard=False)
    right, left = M.to_scipy(), Dm.to_scipy()
    import torch
    rng = np.random.default_rng(9)

    def one_key_70(n):                                # one key holds 70 % of the rows, 49 keys the rest
        return np.where(rng.random(n) < 0.7, 0, rng.integers(1, 50, size=n)).astype(np.int32)
    ids_m, ids_d = one_key_70(400_000), one_key_70(150_000)
    d_ids = (_ids(ids_d), _ids(ids_m))
    rows = np.sort(rng.choice(left.shape[0], 1500, replace=False))
    best0 = keyed_nearest_rows(left, right, ids_d, ids_m, rows, block=100)
    quarter = torch.cuda.get_device_properties(0).total_memory // 4
    for thr in THRESHOLDS:
        want = at_threshold(best0, thr)
        for floor in ((None, True) if thr < 0.5 else (None,)):
            st = {}
            best, score = D.cossim_nearest(Dm, M, thr, stats=st, block_ids=d_ids, floor=floor)
            print("keyed config 4 at %g (floor=%s): topn_floor %s, %d pairs written"
                  % (thr, floor, st["topn_floor"], st["n_nearest_written"]))
            assert st["blocks"] and st["n_blocks_used"] == 50
            if floor is True:
                assert st["topn_floor"] is True
            elif "n_candidates_estimate_usual" in st:
                # auto: the keyed floor exactly when the sampled estimate of the usual path needs a quarter of memory
                assert st["topn_floor"] == (st["n_candidates_estimate_usual"] * 24 > quarter)
            if floor is None and thr == 0.0:
                assert st["topn_floor"] is True and st["floor_init"] is True
            _assert_same((best[rows], score[rows]), want, "keyed config 4 thr=%g floor=%s" % (thr, floor))

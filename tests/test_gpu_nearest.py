"""-m gpu: match_nearest's device path (`_device.cossim_nearest`, the arg-max re-score) bit for bit against the
specification of tests/exact_nearest.py, the public function against the all-pairs oracle
`StringGrouper(..., max_n_matches=len(duplicates)).fit().get_groups()`, the config-4 shape on sampled rows, and the
register lookup of StringGrouperCorpus.  Every exact case compares `best` and the scores with np.array_equal and
asserts the path taken from `stats`."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix

from exact_nearest import exact_nearest, exact_nearest_many, nearest_from_pairs
from exact_topn import exact_pairs
from synth_corpus import make_names
from test_gpu_corpus import perturb

pytestmark = pytest.mark.gpu

LOWEST = 0.0          # the reference pairs are collected once above this
CLUSTER = 320         # identical masters: a duplicate of that name ties with all of them at the top


def _D():
    from string_grouper_b200 import _device as D
    return D


def _strings():
    rng = np.random.default_rng(31)
    masters = make_names(6000, seed=11) + ["acme global holdings llc"] * CLUSTER + ["acme global holding llc"] * 40
    masters += ["", "ab", "x"]                               # rows without an n-gram
    dupes = make_names(1500, seed=12) + [perturb(masters[i], rng) for i in rng.integers(0, 6000, 800)]
    dupes += ["acme global holdings llc"] * 5 + ["acme global holdings"] * 3 + ["", "q", "ab"]
    return masters, dupes


@pytest.fixture(scope="module", params=[np.float64, np.float32], ids=["f64", "f32"])
def mats(request):
    from oracle import pipeline as P
    masters, dupes = _strings()
    m, d, _ = P.tf_idf_matrices(masters, dupes, dtype=request.param)
    m, d = csr_matrix(m).astype(request.param), csr_matrix(d).astype(request.param)
    m.sort_indices()
    d.sort_indices()
    assert np.diff(m.indptr).min() == 0 and np.diff(d.indptr).min() == 0
    pairs = exact_pairs(d, m, LOWEST)
    D = _D()
    return d, m, D.DeviceCSR.from_scipy(d), D.DeviceCSR.from_scipy(m), pairs


def _want(pairs, n, thr):
    r, c, s = pairs
    keep = s > thr
    return nearest_from_pairs(r[keep], c[keep], s[keep], n)


def _run(A, B, thr, **kw):
    st = {}
    best, score = _D().cossim_nearest(A, B, thr, stats=st, **kw)
    assert st["nearest"] is True and st["select"] == "nearest", st
    return (best, score), st


def _assert_same(got, want, label):
    (gb, gs), (wb, ws) = got, want
    assert gb.dtype == np.int64 and gs.dtype == np.float64, label
    bad = np.flatnonzero((gb != wb) | (gs != ws))
    assert len(bad) == 0, "%s: %d rows differ, first %s: got %s want %s" % (
        label, len(bad), bad[:3].tolist(), list(zip(gb[bad[:3]], gs[bad[:3]])), list(zip(wb[bad[:3]], ws[bad[:3]])))
    assert np.array_equal(gb, wb) and np.array_equal(gs, ws), label


@pytest.mark.parametrize("floor", [False, True, "auto"])
@pytest.mark.parametrize("thr", [0.05, 0.3, 0.8])
def test_exact(mats, thr, floor):
    d, m, A, B, pairs = mats
    got, st = _run(A, B, thr, floor=floor)
    assert st["topn_floor"] is (floor is True), st["topn_floor"]    # auto: too few rows for the floor
    assert st["n_nearest_written"] >= int((got[0] >= 0).sum())
    _assert_same(got, _want(pairs, d.shape[0], thr), "thr=%g floor=%s" % (thr, floor))
    # ties at the top go to the lowest master: the copies of the cluster name take its first copy (master 6000)
    assert (got[0][1500 + 800:1500 + 805] == 6000).all()


def test_thresholds_on_pair_scores(mats):
    """thresholds equal to a row's best score (the pair must then be left out) and the next double below it"""
    d, m, A, B, pairs = mats
    best, score = _want(pairs, d.shape[0], LOWEST)
    tops = np.unique(score[score > 0.1])
    picks = [tops[int(q * (len(tops) - 1))] for q in (0.0, 0.25, 0.5, 0.75, 0.9)]
    for s in picks:
        for thr in (float(s), float(np.nextafter(s, -np.inf))):
            for floor in (False, True):
                got, _ = _run(A, B, thr, floor=floor)
                _assert_same(got, _want(pairs, d.shape[0], thr), "thr=%r floor=%s" % (thr, floor))


@pytest.mark.parametrize("acc,kernel", [("u16", "row"), ("f32", "row"), ("u16", "tiles")])
def test_accumulators_and_kernels(mats, acc, kernel):
    d, m, A, B, pairs = mats
    for thr in (0.3, 0.8):
        got, st = _run(A, B, thr, acc=acc, kernel=kernel, floor=False)
        assert st["acc"] == acc and st["kernel"] == kernel, (st["acc"], st["kernel"])
        _assert_same(got, _want(pairs, d.shape[0], thr), "acc=%s kernel=%s thr=%g" % (acc, kernel, thr))
    if kernel == "row":
        got, st = _run(A, B, 0.3, acc=acc, floor=True)
        _assert_same(got, _want(pairs, d.shape[0], 0.3), "acc=%s floor" % acc)


def test_no_threshold(mats):
    d, m, A, B, pairs = mats
    want = _want(pairs, d.shape[0], 0.0)
    for thr in (0.0, -1.0):
        for floor in (True, False):
            got, st = _run(A, B, thr, floor=floor)
            assert st["topn_floor"] is floor and st.get("floor_init", False) is floor
            _assert_same(got, want, "no threshold (%g) floor=%s" % (thr, floor))


def test_row_chunks_and_buffer_retry(mats, monkeypatch):
    d, m, A, B, pairs = mats
    D = _D()
    monkeypatch.setattr(D, "GROUP_BYTES", 1)
    monkeypatch.setattr(D, "CAND_CHUNK", 1000)
    for thr, floor in ((0.3, False), (0.3, True), (0.05, False), (0.0, True)):
        got, st = _run(A, B, thr, floor=floor, acc="f32", tile_w=64)
        assert st["n_row_chunks"] > 1, st["n_row_chunks"]
        _assert_same(got, _want(pairs, d.shape[0], thr), "row chunks thr=%g floor=%s" % (thr, floor))
    monkeypatch.undo()
    monkeypatch.setenv("SG_B200_CAND_CAP", "1000")       # the launch overflows its buffer and is repeated
    got, st = _run(A, B, 0.3, floor=False)
    assert st["n_candidates"] > 1000
    _assert_same(got, _want(pairs, d.shape[0], 0.3), "buffer retry")


def test_same_matrix_both_sides(mats):
    """A is B (a register looked up with itself): the full product, no triangle, no dedup"""
    d, m, A, B, pairs = mats
    want = exact_nearest(m, m, 0.5)
    for floor in (False, True):
        got, st = _run(B, B, 0.5, floor=floor)
        assert st["triangle"] is False and st.get("dedup", False) is False
        _assert_same(got, want, "A is B floor=%s" % floor)


def test_nearest_needs_all_rows_and_top_one(mats):
    d, m, A, B, pairs = mats
    D = _D()
    for kw in ({"row_begin": 5}, {"row_end": 100}):
        with pytest.raises(ValueError):
            D.cossim_topn(A, B, 1, 0.5, nearest=True, **kw)
    with pytest.raises(ValueError):
        D.cossim_topn(A, B, 2, 0.5, nearest=True)


# ---------------------------------------------------------------------------------------------------------------
# the public function against the all-pairs oracle
# ---------------------------------------------------------------------------------------------------------------

def _assert_equal(got, want):
    (pd.testing.assert_frame_equal if isinstance(want, pd.DataFrame) else pd.testing.assert_series_equal)(got, want)


@pytest.fixture(scope="module")
def synthetic20k():
    rng = np.random.default_rng(41)
    names = make_names(20_000, seed=42)
    batch = make_names(2000, seed=43) + [perturb(names[i], rng) for i in rng.integers(0, len(names), 1500)]
    batch += [names[7]] * 4 + [names[7] + " inc"] * 3
    return pd.Series(names, name="register"), pd.Series(batch, index=np.arange(len(batch)) * 3 + 1)


@pytest.mark.parametrize("thr", [0.8, 0.5])
def test_public_api_against_the_all_pairs_oracle(synthetic20k, thr):
    import string_grouper_b200 as api
    master, dupes = synthetic20k
    mid = pd.Series(np.arange(len(master)) + 100, name="mid")
    did = pd.Series(["d%d" % i for i in range(len(dupes))], name="did", index=dupes.index)
    want = api.StringGrouper(master, dupes, mid, did, min_similarity=thr,
                             max_n_matches=len(dupes)).fit().get_groups()
    got = api.match_nearest(master, dupes, mid, did, min_similarity=thr)
    _assert_equal(got, want)
    mms = api.match_most_similar(master, dupes, mid, did, min_similarity=thr)
    differ = int((mms["most_similar_register"] != got["most_similar_register"]).sum())
    print("min_similarity %g: %d of %d duplicates differ from match_most_similar" % (thr, differ, len(dupes)))
    assert differ > 0
    sg = api.StringGrouper(master, dupes)
    _assert_equal(sg.match_nearest(master, dupes, mid, did, min_similarity=thr), want)


# ---------------------------------------------------------------------------------------------------------------
# config-4 shape (400k masters x 150k duplicates), sampled rows
# ---------------------------------------------------------------------------------------------------------------

def test_config4_shape_exact_on_sampled_rows():
    from string_grouper_b200 import StringGrouper
    D = _D()
    base = make_names(480_000, seed=3)
    master, dupes = pd.Series(base[:400_000]), pd.Series(base[330_000:480_000])
    M, Dm = StringGrouper(master, duplicates=dupes)._get_tf_idf_matrices(shard=False)
    right, left = M.to_scipy(), Dm.to_scipy()
    rows = np.sort(np.random.default_rng(9).choice(left.shape[0], 2000, replace=False))
    want = exact_nearest_many(left[rows], right, (0.8, 0.3, 0.0))
    for thr in (0.8, 0.3, 0.0):
        st = {}
        best, score = D.cossim_nearest(Dm, M, thr, stats=st)
        print("config 4 at %g: floor %s, %d pairs written" % (thr, st["topn_floor"], st["n_nearest_written"]))
        _assert_same((best[rows], score[rows]), want[thr], "config 4 shape thr=%g" % thr)
        if thr == 0.0:
            assert st["topn_floor"] is True and st["floor_init"] is True


# ---------------------------------------------------------------------------------------------------------------
# register lookup on a corpus
# ---------------------------------------------------------------------------------------------------------------

def test_corpus_register_lookup(synthetic20k):
    import string_grouper_b200 as api
    from oracle import pipeline as P
    D = _D()
    register, batch = synthetic20k
    corpus = api.StringGrouperCorpus(register)
    vec = P.tf_idf_matrices(register.tolist())[2]
    Mr, Mb = vec.transform(register.tolist()), vec.transform(batch.tolist())
    b1, b2 = batch.iloc[:1800], batch.iloc[1800:]

    def delta(call):
        before = dict(D.LAUNCH_COUNTS)
        out = call()
        return out, {k: D.LAUNCH_COUNTS[k] - before[k] for k in before}

    for thr in (0.8, 0.5):
        for part, lo in ((b1, 0), (b2, 1800)):
            got, d = delta(lambda: corpus.match_nearest(register, part, min_similarity=thr))
            best, _ = exact_nearest(Mb[lo:lo + len(part)], Mr, thr)
            want = api.StringGrouper(register, part)._nearest_frame(best, False, False)
            _assert_equal(got, want)
            # the register is not vectorised again: one K1 transform of the batch (3 launches); its row order and
            # postings were built by the first call and carry over (the batch's own row order: 2 launches)
            assert d["tfidf"] == 3, d
            if (thr, lo) != (0.8, 0):
                assert d["postings"] == 0 and d["order"] == 2 and d["tiles"] == 0, d

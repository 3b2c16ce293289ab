"""not-gpu: host logic of match_nearest (StringGrouper, module function, StringGrouperCorpus) with the oracle standing in
for the device (tests/cpu_backend.py) and a numpy model of `_device.cossim_nearest` (tests/exact_nearest.py).

* match_nearest equals the oracle `StringGrouper(..., max_n_matches=len(duplicates)).fit().get_groups()` on every
  match_most_similar case of tests/golden/api_cases.json (index, ids, ignore_index, replace_na, unmatched rows,
  MultiIndex, unnamed Series);
* where every master is the best match of at most one duplicate it equals match_most_similar;
* the documented example: 'foooob' maps to 'foooo' under match_nearest, and match_most_similar still leaves it alone.
"""
import numpy as np
import pandas as pd
import pytest

import string_grouper_b200 as api
from cpu_backend import oracle_device
from exact_nearest import exact_nearest
from golden_util import fixtures, load_cases, resolve
from string_grouper_b200 import _device
from synth_corpus import make_names

CASES = load_cases()
MMS = sorted(k for k, c in CASES.items() if c["fn"] == "match_most_similar")


def _cossim_nearest(A, B, threshold, stats=None, **kw):
    if stats is not None:
        stats["nearest"] = True
    if A.shape[1] == 0 or A.shape[0] == 0 or B.shape[0] == 0:
        return np.full(A.shape[0], -1, dtype=np.int64), np.zeros(A.shape[0])
    return exact_nearest(A.m, B.m, threshold)


@pytest.fixture
def host(monkeypatch):
    with oracle_device():
        monkeypatch.setattr(_device, "cossim_nearest", _cossim_nearest)
        yield


def _assert_equal(got, want):
    (pd.testing.assert_frame_equal if isinstance(want, pd.DataFrame) else pd.testing.assert_series_equal)(got, want)


def _oracle(master, duplicates, master_id=None, duplicates_id=None, **kw):
    kw["max_n_matches"] = len(duplicates)
    return api.StringGrouper(master, duplicates=duplicates, master_id=master_id, duplicates_id=duplicates_id,
                             **kw).fit().get_groups()


def _case(key):
    fx = fixtures()
    args = [resolve(a, fx) for a in CASES[key]["series"]]
    kw = dict(CASES[key]["kwargs"])
    if kw.get("tfidf_matrix_dtype") == "float32":
        kw["tfidf_matrix_dtype"] = np.float32
    return args, kw


@pytest.mark.parametrize("key", MMS)
def test_equals_the_all_pairs_oracle(key, host):
    args, kw = _case(key)
    want = _oracle(*args, **kw)
    _assert_equal(api.match_nearest(*args, **kw), want)
    _assert_equal(api.match_nearest(*args, max_n_matches=1, **kw), want)        # accepted and ignored
    _assert_equal(api.StringGrouper(args[0], args[1]).match_nearest(*args, **kw), want)


@pytest.mark.parametrize("index", [None, "labels"])
@pytest.mark.parametrize("ids", [False, True])
def test_equals_match_most_similar_when_no_master_is_shared(index, ids, host):
    """duplicates that are near copies of distinct masters, plus unrelated names: no master is the best match of two
    duplicates, so the reference's one-duplicate-per-master product gives the same answer"""
    rng = np.random.default_rng(5)
    ms = make_names(300, seed=21)
    picks = rng.choice(len(ms), 40, replace=False)
    ds = [ms[i] + " inc" for i in picks] + make_names(30, seed=22)
    # drop the duplicates that share a master above the threshold with an earlier one
    pairs = api.StringGrouper(pd.Series(ms), pd.Series(ds), min_similarity=0.6).fit()._matches_list
    taken, keep = set(), []
    for j in range(len(ds)):
        hit = set(pairs.master_side[pairs.dupe_side == j])
        keep.append(not hit & taken)
        taken |= hit if keep[-1] else set()
    ds = [x for x, k in zip(ds, keep) if k]
    mi = None if index is None else pd.Index(["m%d" % i for i in range(len(ms))], name="mk")
    di = None if index is None else pd.Index(["d%d" % i for i in range(len(ds))], name="dk")
    m, d = pd.Series(ms, name="name", index=mi), pd.Series(ds, name="name", index=di)
    mid = pd.Series(np.arange(len(ms)), name="mid", index=mi) if ids else None
    did = pd.Series(np.arange(len(ds)) + 1000, name="did", index=di) if ids else None
    pairs = api.StringGrouper(m, d, min_similarity=0.6).fit()._matches_list
    assert len(pairs) >= 30 and pairs.master_side.value_counts().max() == 1
    got = api.match_nearest(m, d, mid, did, min_similarity=0.6)
    _assert_equal(got, _oracle(m, d, mid, did, min_similarity=0.6))
    _assert_equal(got, api.match_most_similar(m, d, mid, did, min_similarity=0.6))


def test_documented_example(host):
    master = pd.Series(["foooo", "bar", "baz"])
    dupes = pd.Series(["foooo", "bar", "baz", "foooob"])
    got = api.match_nearest(master, dupes)
    assert got["most_similar_master"].tolist() == ["foooo", "bar", "baz", "foooo"]
    assert got["most_similar_index"].tolist() == [0, 1, 2, 0]
    mms = api.match_most_similar(master, dupes)
    assert mms["most_similar_master"].tolist() == ["foooo", "bar", "baz", "foooob"]
    _assert_equal(got, _oracle(master, dupes))


def test_ties_go_to_the_lowest_master(host):
    master = pd.Series(["acme corp", "zeta", "acme corp", "acme corp"], index=[7, 3, 5, 1])
    dupes = pd.Series(["acme corp", "acme corpp"])
    got = api.match_nearest(master, dupes, min_similarity=0.5)
    assert got["most_similar_index"].tolist() == [7, 7]
    _assert_equal(got, _oracle(master, dupes, min_similarity=0.5))


@pytest.mark.parametrize("dtype", ["str", "string[pyarrow]", "string[python]", object])
@pytest.mark.parametrize("ids", [False, True])
@pytest.mark.parametrize("ignore_index,replace_na", [(False, False), (True, False), (False, True)])
def test_arrow_take_gives_the_object_path_frame(dtype, ids, ignore_index, replace_na, monkeypatch):
    """the result frame built with the Arrow take equals the one built through `to_numpy()`, for every string dtype
    (only pandas' inferred `str` takes the Arrow path), with string ids, unmatched duplicates, all index options"""
    from string_grouper_b200 import string_grouper as sgm
    rng = np.random.default_rng(7)
    ms = make_names(500, seed=25) + ["", "é ü 東京"]
    ds = make_names(120, seed=26) + ["東京", ""]
    m = pd.Series(ms, name="name", dtype=dtype, index=pd.Index(np.arange(len(ms)) * 2 + 5, name="k"))
    d = pd.Series(ds, dtype=dtype, index=pd.Index(["d%d" % i for i in range(len(ds))], name="k"))
    mid = pd.Series(["m%d" % i for i in range(len(ms))], name="mid", dtype=dtype) if ids else None
    did = pd.Series(["x%d" % i for i in range(len(ds))], name="did", dtype=dtype) if ids else None
    sg = api.StringGrouper(m, d, mid, did)
    for best in (rng.integers(-1, len(ms), len(ds)), np.full(len(ds), -1), rng.integers(0, len(ms), len(ds))):
        got = sg._nearest_frame(best, ignore_index, replace_na)
        monkeypatch.setattr(sgm, "_takes_as_str", lambda a, b: False)
        want = sg._nearest_frame(best, ignore_index, replace_na)
        monkeypatch.undo()
        _assert_equal(got, want)
    assert sgm._takes_as_str(m, d) == (pd.Series(m.to_numpy()).dtype == m.dtype and dtype != "string[python]")


def test_corpus_and_arguments(host, monkeypatch):
    names = make_names(200, seed=23)
    s = pd.Series(names)
    batch = pd.Series([n + "x" for n in names[:50]] + make_names(20, seed=24))
    corpus = api.StringGrouperCorpus(pd.concat([s, batch], ignore_index=True))
    monkeypatch.setattr(_device, "tfidf_transform", _transform_as_fit(corpus))
    got = corpus.match_nearest(s, batch, min_similarity=0.5)
    assert len(got) == len(batch)
    with pytest.raises(TypeError):
        api.match_nearest(s, None)
    with pytest.raises(ValueError):
        corpus.match_nearest(s, batch, ngram_size=4)


def _transform_as_fit(corpus):
    """the corpus was fitted on master ++ duplicates: its transform of them is the fit (the host stand-in re-fits)"""
    from cpu_backend import tfidf

    def transform(data, offsets, n_first, flags, vocab, stats=None):
        first, second, _ = tfidf(data, offsets, n_first, 3, flags, np.float64)
        return first, second
    return transform

"""not-gpu: the host side of keyed lookups (blocking keys through match_nearest and StringGrouperCorpus), with the
oracle standing in for the device (tests/cpu_backend.py), a scikit-learn vectoriser for the corpus transform, and
keyed stand-ins of cossim_topn / cossim_nearest that follow the specifications of tests/test_gpu_blocks.py and
tests/test_gpu_keyed_nearest.py (the exact pairs without the pairs of different ids).

* key mapping of a keyed corpus: corpus values keep the corpus ids, values the corpus lacks share ids after them,
  missing keys get one id each; the corpus Series carries the corpus keys; the ValueError / TypeError cases;
* keys are never dropped: every corpus method hands block ids to the product and equals the keyed module function;
* match_nearest with one key for every string is the unkeyed call, and keyed match_nearest is the keyed all-pairs
  arg-max.
"""
import copy

import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix
from sklearn.feature_extraction.text import TfidfVectorizer

import string_grouper_b200 as api
from cpu_backend import FakeCSR, FakeMatches, _device_analyzer, cossim_topn, oracle_device
from exact_nearest import nearest_from_pairs
from exact_topn import RankedPairs, exact_pairs
from string_grouper_b200 import StringGrouperCorpus, _device
from synth_corpus import make_names


class _Vocabulary:
    def __init__(self, vec, ngram):
        self.vec, self.ngram = vec, ngram
        self.idf_ = vec.idf_


class StandIn:
    """_device.tfidf / tfidf_transform on scikit-learn (transform with the fitted vectoriser), and keyed products
    that record the block ids they were given"""

    def __init__(self):
        self.calls = []        # (kind, block_ids) per product

    def tfidf(self, data, offsets, n_master, ngram, flags, dtype, device=None, stats=None):
        docs = _docs(data, offsets)
        vec = TfidfVectorizer(min_df=1, analyzer=lambda s: _device_analyzer(s, ngram, flags), dtype=dtype)
        m = vec.fit_transform(docs)
        dup = FakeCSR(m[n_master:]) if n_master < len(docs) else None
        return FakeCSR(m[:n_master]), dup, _Vocabulary(vec, ngram)

    def tfidf_transform(self, data, offsets, n_first, flags, vocab, stats=None):
        vec = copy.copy(vocab.vec)
        vec.analyzer = lambda s: _device_analyzer(s, vocab.ngram, flags)
        m = vec.transform(_docs(data, offsets))
        return FakeCSR(m[:n_first]), FakeCSR(m[n_first:])

    def cossim_topn(self, A, B, top_n, threshold, row_begin=0, row_end=None, block_ids=None, stats=None, **kw):
        self.calls.append(("topn", block_ids))
        if block_ids is None:
            return cossim_topn(A, B, top_n, threshold, row_begin, row_end, **kw)
        ids_a, ids_b = block_ids
        r, c, s = exact_pairs(A.m, B.m, threshold)
        keep = ids_a[r] == ids_b[c]
        row, col, score, max_row = RankedPairs(r[keep], c[keep], s[keep]).topn(min(top_n, B.shape[0]), threshold)
        indptr = np.zeros(A.shape[0] + 1, np.int64)
        np.cumsum(np.bincount(row, minlength=A.shape[0]), out=indptr[1:])
        return FakeMatches(csr_matrix((score, col, indptr), shape=(A.shape[0], B.shape[0])), max_row=max_row)

    def cossim_nearest(self, A, B, threshold, stats=None, block_ids=None, **kw):
        self.calls.append(("nearest", block_ids))
        r, c, s = exact_pairs(A.m, B.m, threshold)
        if block_ids is not None:
            keep = block_ids[0][r] == block_ids[1][c]
            r, c, s = r[keep], c[keep], s[keep]
        return nearest_from_pairs(r, c, s, A.shape[0])


def _docs(data, offsets):
    raw = bytes(np.asarray(data, dtype=np.uint8))
    return [raw[offsets[i]:offsets[i + 1]].decode("ascii") for i in range(len(offsets) - 1)]


@pytest.fixture
def standin(monkeypatch):
    s = StandIn()
    with oracle_device():
        for name in ("tfidf", "tfidf_transform", "cossim_topn", "cossim_nearest"):
            monkeypatch.setattr(_device, name, getattr(s, name))
        # host arrays for the device id tensors: a self-match takes one array twice
        monkeypatch.setattr(_device, "block_id_tensors",
                            lambda ids, n_left, same: (ids, ids) if same else (ids[:n_left], ids[n_left:]))
        yield s


@pytest.fixture(scope="module")
def data():
    rng = np.random.default_rng(5)
    names = make_names(300, seed=41)
    names += [n + " co" for n in names[:80]]
    s = pd.Series(names)
    keys = pd.Series(rng.choice(["US", "FR", "DE", None], size=len(s), p=[0.4, 0.3, 0.2, 0.1]), dtype=object)
    return s, keys


def _assert_equal(got, want):
    (pd.testing.assert_frame_equal if isinstance(want, pd.DataFrame) else pd.testing.assert_series_equal)(got, want)


# ---------------------------------------------------------------------------------------------------------------
# key mapping
# ---------------------------------------------------------------------------------------------------------------

def test_corpus_ids_and_mapping_of_known_new_and_missing_keys(standin):
    reg = pd.Series(["alpha one", "beta two", "gamma three", "delta four", "eps five"])
    corpus = StringGrouperCorpus(reg, keys=pd.Series(["US", "FR", None, "US", "DE"], dtype=object))
    assert corpus._ids.tolist() == [0, 1, 3, 0, 2] and corpus._ids.dtype == np.int32     # US FR DE, then missing
    batch = pd.Series(["a", "b", "c", "d", "e", "f"])
    bkeys = pd.Series(["FR", "IT", None, "IT", "US", np.nan], dtype=object, index=[9, 8, 7, 6, 5, 4])
    ids = corpus._block_ids(reg, batch, None, bkeys)
    assert ids.dtype == np.int32
    assert ids.tolist() == [0, 1, 3, 0, 2] + [1, 4, 5, 4, 0, 6]       # by position: the index is not read
    # two fresh Series: a value the corpus lacks shares one id over both of them
    m, d = pd.Series(["x", "y"]), pd.Series(["z"])
    ids = corpus._block_ids(m, d, pd.Series(["NL", "US"]), pd.Series(["NL"]))
    assert ids.tolist() == [4, 0, 4]
    assert corpus._block_ids(m, d) is None                            # no keys on either fresh Series: unkeyed


def test_tuple_and_numeric_keys_map_like_values(standin):
    reg = pd.Series(["alpha one", "beta two", "gamma three"])
    corpus = StringGrouperCorpus(reg, keys=pd.Series([("t", 1), ("t", 2), ("t", 1)], dtype=object))
    ids = corpus._block_ids(reg, pd.Series(["q", "r"]), None, pd.Series([("t", 2), ("u", 0)], dtype=object))
    assert ids.tolist() == [0, 1, 0, 1, 2]
    corpus = StringGrouperCorpus(reg, keys=pd.Series([3, 1, 3]))
    ids = corpus._block_ids(reg, pd.Series(["q", "r"]), None, pd.Series([1, 7]))
    assert ids.tolist() == [0, 1, 0, 1, 2]


def test_corpus_series_carries_the_corpus_keys(standin, data):
    s, keys = data
    corpus = StringGrouperCorpus(s, keys=keys)
    batch = pd.Series(["x one", "y two"])
    bkeys = pd.Series(["US", "FR"])
    base = corpus._block_ids(s, batch, None, bkeys)
    assert np.array_equal(base[:len(s)], corpus._ids)
    # the same keys again (another index) are accepted; other keys for the corpus Series are not
    same = pd.Series(keys.to_numpy(), index=np.arange(len(s))[::-1], dtype=object)
    assert np.array_equal(corpus._block_ids(s, batch, same, bkeys), base)
    with pytest.raises(ValueError):
        corpus._block_ids(s, batch, keys.shift(1), bkeys)
    with pytest.raises(ValueError):
        corpus.match_nearest(s, batch, master_keys=pd.Series(["US"] * len(s)), duplicates_keys=bkeys)
    # the other Series of a keyed call needs keys of its own
    with pytest.raises(ValueError):
        corpus.match_nearest(s, batch)
    with pytest.raises(ValueError):
        corpus.match_strings(batch, s)
    # a self-match of the corpus Series is keyed by the corpus keys
    assert np.array_equal(corpus._block_ids(s), corpus._ids)
    assert np.array_equal(corpus._block_ids(s, s), np.concatenate([corpus._ids, corpus._ids]))


def test_key_argument_errors(standin, data):
    s, keys = data
    batch, bkeys = pd.Series(["x one", "y two"]), pd.Series(["US", "FR"])
    for corpus in (StringGrouperCorpus(s, keys=keys), StringGrouperCorpus(s)):
        with pytest.raises(ValueError):
            corpus.match_nearest(s, batch, duplicates_keys=bkeys[:1])                  # wrong length
        with pytest.raises(TypeError):
            corpus.match_nearest(s, batch, master_keys=keys, duplicates_keys=["US", "FR"])
        with pytest.raises(ValueError):
            corpus.match_strings(batch, duplicates_keys=bkeys)                         # no duplicates
        with pytest.raises(ValueError):
            corpus.match_strings(batch, pd.Series(["z"]), master_keys=bkeys)           # one fresh side only
        with pytest.raises(TypeError):                                                 # keys are keyword-only
            corpus.match_nearest(s, batch, None, None, keys, bkeys)
    with pytest.raises(ValueError):
        StringGrouperCorpus(s, keys=keys[:10])
    with pytest.raises(TypeError):
        StringGrouperCorpus(s, keys=list(keys))


def test_unkeyed_corpus_factorises_per_call(standin, data):
    from string_grouper_b200.string_grouper import block_ids_of
    s, keys = data
    corpus = StringGrouperCorpus(s)
    batch, bkeys = pd.Series(["x one", "y two"]), pd.Series(["US", "FR"])
    grouper = corpus._grouper(s, batch, master_keys=keys, duplicates_keys=bkeys)
    assert np.array_equal(grouper._block_ids, block_ids_of(s, batch, keys, bkeys))
    assert corpus._grouper(s, batch)._block_ids is None


# ---------------------------------------------------------------------------------------------------------------
# keys reach the product from every corpus method
# ---------------------------------------------------------------------------------------------------------------

def _halves(s, keys):
    n = len(s) * 2 // 3
    m, d = s[:n], s[n:].reset_index(drop=True)
    return m, d, keys[:n], keys[n:].reset_index(drop=True)


@pytest.mark.parametrize("keyed_corpus", [False, True])
def test_every_corpus_method_is_keyed(standin, data, keyed_corpus):
    s, keys = data
    m, d, mk, dk = _halves(s, keys)
    whole = pd.concat([m, d], ignore_index=True)
    corpus = StringGrouperCorpus(whole, keys=pd.concat([mk, dk], ignore_index=True) if keyed_corpus else None)
    kw = dict(min_similarity=0.5)
    cases = [
        (lambda: corpus.match_strings(m, d, master_keys=mk, duplicates_keys=dk, **kw),
         lambda: api.match_strings(m, d, master_keys=mk, duplicates_keys=dk, **kw)),
        (lambda: corpus.match_most_similar(m, d, master_keys=mk, duplicates_keys=dk, **kw),
         lambda: api.match_most_similar(m, d, master_keys=mk, duplicates_keys=dk, **kw)),
        (lambda: corpus.match_nearest(m, d, master_keys=mk, duplicates_keys=dk, **kw),
         lambda: api.match_nearest(m, d, master_keys=mk, duplicates_keys=dk, **kw)),
        (lambda: corpus.fit(m, d, master_keys=mk, duplicates_keys=dk, **kw).get_matches(),
         lambda: api.StringGrouper(m, d, master_keys=mk, duplicates_keys=dk, **kw).fit().get_matches()),
        (lambda: corpus.group_similar_strings(whole, keys=pd.concat([mk, dk], ignore_index=True), **kw),
         lambda: api.group_similar_strings(whole, keys=pd.concat([mk, dk], ignore_index=True), **kw)),
    ]
    for got, want in cases:
        standin.calls.clear()
        g = got()
        assert standin.calls and all(ids is not None for _, ids in standin.calls)
        _assert_equal(g, want())
    # and the keys change the answer: the unkeyed lookup differs on this data
    assert not corpus.match_nearest(m, d, **kw).equals(api.match_nearest(m, d, master_keys=mk, duplicates_keys=dk,
                                                                        **kw))


def test_register_lookup_on_a_keyed_corpus(standin, data):
    """the corpus Series as master takes the corpus keys and its own id array (the device tensor) as the right ids"""
    s, keys = data
    corpus = StringGrouperCorpus(s, keys=keys)
    batch = pd.Series([n + "x" for n in s[:60]] + ["zzz qqq"])
    bkeys = pd.Series(list(keys[:30]) + ["US"] * 15 + ["IT"] * 15 + [None], dtype=object)
    standin.calls.clear()
    got = corpus.match_nearest(s, batch, duplicates_keys=bkeys, min_similarity=0.3)
    (kind, (ids_dup, ids_reg)), = standin.calls
    assert kind == "nearest" and ids_reg is corpus._d_ids
    # the keyed all-pairs arg-max on the corpus transform: match_most_similar with room for every duplicate
    want = corpus.fit(s, batch, duplicates_keys=bkeys, min_similarity=0.3, max_n_matches=len(batch)).get_groups()
    _assert_equal(got, want)
    # a duplicate with a key the corpus lacks, or a missing key, comes back as itself
    assert (got["most_similar_master"][45:].to_numpy() == batch[45:].to_numpy()).all()
    assert got["most_similar_index"][45:].isna().all()


def test_grouper_from_a_keyed_corpus_keeps_the_rule(standin, data):
    s, keys = data
    corpus = StringGrouperCorpus(s, keys=keys)
    sg = corpus.fit(s)
    assert np.array_equal(sg._block_ids, corpus._ids)
    with pytest.raises(ValueError):
        sg.match_nearest(s, pd.Series(["x one"]))                # reset_data goes through the corpus rule
    sg.match_nearest(s, pd.Series(["x one"]), duplicates_keys=pd.Series(["US"]))
    assert sg._block_ids[-1] == corpus._ids[keys.to_numpy() == "US"][0]


def test_pairwise_similarities_take_no_keys(standin, data):
    s, keys = data
    corpus = StringGrouperCorpus(s, keys=keys)
    got = corpus.compute_pairwise_similarities(s[:5], s[5:10].reset_index(drop=True))
    assert len(got) == 5


# ---------------------------------------------------------------------------------------------------------------
# match_nearest
# ---------------------------------------------------------------------------------------------------------------

def test_match_nearest_one_key_is_the_unkeyed_call(standin, data):
    s, _ = data
    m, d, _, _ = _halves(s, pd.Series(["k"] * len(s)))
    one_m, one_d = pd.Series(["k"] * len(m)), pd.Series(["k"] * len(d))
    for thr in (0.0, 0.3, 0.8):
        _assert_equal(api.match_nearest(m, d, master_keys=one_m, duplicates_keys=one_d, min_similarity=thr),
                      api.match_nearest(m, d, min_similarity=thr))
        sg = api.StringGrouper(m, d)
        _assert_equal(sg.match_nearest(m, d, master_keys=one_m, duplicates_keys=one_d, min_similarity=thr),
                      api.match_nearest(m, d, min_similarity=thr))


def test_keyed_match_nearest_is_the_keyed_all_pairs_argmax(standin, data):
    s, keys = data
    m, d, mk, dk = _halves(s, keys)
    for thr in (0.0, 0.5):
        standin.calls.clear()
        got = api.match_nearest(m, d, master_keys=mk, duplicates_keys=dk, min_similarity=thr)
        (kind, (ids_d, ids_m)), = standin.calls
        assert len(ids_d) == len(d) and len(ids_m) == len(m)       # the duplicates are the left operand
        want = api.StringGrouper(m, d, master_keys=mk, duplicates_keys=dk, min_similarity=thr,
                                 max_n_matches=len(d)).fit().get_groups()
        _assert_equal(got, want)
    with pytest.raises(ValueError):
        api.match_nearest(m, d, master_keys=mk)


def test_corpus_keys_compared_by_value_not_dtype(standin, data):
    s, keys = data
    corpus = StringGrouperCorpus(s, keys=keys)
    batch, bkeys = pd.Series(["x one", "y two"]), pd.Series(["US", "FR"])
    base = corpus._block_ids(s, batch, None, bkeys)
    for same in (keys.astype("category"), keys.astype("string[pyarrow]"), keys.astype("string[python]"),
                 pd.Series(keys.to_numpy(), index=np.arange(len(keys))[::-1], dtype=object)):
        assert np.array_equal(corpus._block_ids(s, batch, same, bkeys), base), same.dtype
    other = keys.copy()
    other.iloc[0] = "NL" if other.iloc[0] != "NL" else "US"
    moved = keys.copy()
    moved.iloc[int(np.flatnonzero(keys.isna().to_numpy())[0])] = "US"      # a missing key given a value
    for bad in (other, moved, keys[:-1]):
        with pytest.raises(ValueError):
            corpus._block_ids(s, batch, bad, bkeys)


def test_the_corpus_series_is_the_object_itself(standin, data):
    """the README's pattern: the corpus Series kept in a variable carries the corpus keys; a column selected again
    from its DataFrame is another Series, and the error says so"""
    s, keys = data
    df = pd.DataFrame({"name": s, "country": keys})
    names = df["name"]
    register = StringGrouperCorpus(names, keys=df["country"])
    batch = pd.DataFrame({"name": ["x one", "y two"], "country": ["US", "FR"]})
    got = register.match_nearest(names, batch["name"], duplicates_keys=batch["country"], min_similarity=0.3)
    assert len(got) == 2
    if df["name"] is not names:              # pandas' copy-on-write: every selection is a new Series
        with pytest.raises(ValueError, match="identity"):
            register.match_nearest(df["name"], batch["name"], duplicates_keys=batch["country"])

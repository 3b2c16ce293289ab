"""not-gpu: host logic of StringGrouperCorpus (option handling, the identity rule, frame shapes) with a scikit-learn
stand-in for the device vectoriser, and the host mapping of new symbols through a fitted alphabet.

The stand-in fits like tests/cpu_backend.py and transforms with the SAME fitted TfidfVectorizer (vocabulary, idf),
which is what the CUDA transform computes; tests/test_gpu_corpus.py checks the CUDA path itself against scikit-learn.
"""
import copy

import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix
from sklearn.feature_extraction.text import TfidfVectorizer

import string_grouper_b200 as api
from cpu_backend import FakeCSR, _device_analyzer, oracle_device
from oracle import pipeline as P
from string_grouper_b200 import StringGrouperConfig, StringGrouperCorpus, _device, _ingest, _lib
from synth_corpus import make_names


def _docs(data, offsets):
    if np.asarray(data).dtype == np.uint32:
        raw = np.asarray(data, dtype=np.uint32)
        return [raw[offsets[i]:offsets[i + 1]].tobytes().decode("utf-32-le", "surrogatepass")
                for i in range(len(offsets) - 1)]
    raw = bytes(np.asarray(data, dtype=np.uint8))
    return [raw[offsets[i]:offsets[i + 1]].decode("ascii") for i in range(len(offsets) - 1)]


class FakeVocabulary:
    def __init__(self, vec, ngram, n_docs):
        self.vec, self.ngram, self.n_docs = vec, ngram, n_docs
        self.idf_ = vec.idf_ if vec is not None else np.zeros(0)
        self.size = len(self.idf_)

    def feature_names(self):
        return self.vec.get_feature_names_out().tolist()


class StandIn:
    """_device.tfidf / _device.tfidf_transform on scikit-learn; records the rows every transform received"""

    def __init__(self):
        self.transformed = []

    def tfidf(self, data, offsets, n_master, ngram, flags, dtype, device=None, stats=None):
        docs = _docs(data, offsets)
        vec = TfidfVectorizer(min_df=1, analyzer=lambda s: _device_analyzer(s, ngram, flags), dtype=dtype)
        if any(len(_device_analyzer(d, ngram, flags)) for d in docs):
            m = vec.fit_transform(docs)
        else:
            vec, m = None, csr_matrix((len(docs), 0), dtype=dtype)
        dup = FakeCSR(m[n_master:]) if n_master < len(docs) else None
        return FakeCSR(m[:n_master]), dup, FakeVocabulary(vec, ngram, len(docs))

    def tfidf_transform(self, data, offsets, n_first, flags, vocab, stats=None):
        docs = _docs(data, offsets)
        self.transformed.append(len(docs))
        vec = copy.copy(vocab.vec)
        # this batch's own analyzer flags (ingest may fold on the host for one call and on the device for another)
        vec.analyzer = lambda s: _device_analyzer(s, vocab.ngram, flags)
        m = vec.transform(docs)
        return FakeCSR(m[:n_first]), FakeCSR(m[n_first:])


@pytest.fixture
def standin(monkeypatch):
    s = StandIn()
    with oracle_device():
        monkeypatch.setattr(_device, "tfidf", s.tfidf)
        monkeypatch.setattr(_device, "tfidf_transform", s.tfidf_transform)
        yield s


@pytest.fixture(scope="module")
def names():
    base = make_names(400, seed=11)
    return base + [n.upper() + " Ltd." for n in base[:60]]


def _series(strings, name=None, index=None):
    return pd.Series(strings, name=name, index=index)


# ---------------------------------------------------------------------------------------------------------------
# identities with the module-level functions
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ids", [False, True])
@pytest.mark.parametrize("index", [None, "shifted"])
def test_self_match_identities(standin, names, ids, index):
    idx = None if index is None else pd.Index(np.arange(len(names)) * 3 + 7, name="k")
    s = _series(names, "name", idx)
    sid = _series(["id%d" % i for i in range(len(names))], "id", idx) if ids else None
    corpus = StringGrouperCorpus(s, min_similarity=0.6)
    pd.testing.assert_frame_equal(corpus.match_strings(s, master_id=sid),
                                  api.match_strings(s, master_id=sid, min_similarity=0.6))
    for rep in ("centroid", "first"):
        got = corpus.group_similar_strings(s, string_ids=sid, group_rep=rep)
        want = api.group_similar_strings(s, string_ids=sid, group_rep=rep, min_similarity=0.6)
        (pd.testing.assert_frame_equal if isinstance(want, pd.DataFrame) else pd.testing.assert_series_equal)(got, want)
    assert standin.transformed == []          # the corpus Series itself is never vectorised again


@pytest.mark.parametrize("ids", [False, True])
@pytest.mark.parametrize("index", [None, "labels"])
def test_two_series_identities(standin, names, ids, index):
    m_strings, d_strings = names[:300], names[300:] + names[:20]
    mi = None if index is None else pd.Index(["m%d" % i for i in range(len(m_strings))])
    di = None if index is None else pd.Index(["d%d" % i for i in range(len(d_strings))])
    m, d = _series(m_strings, "m", mi), _series(d_strings, None, di)
    mid = _series(np.arange(len(m_strings)), "mid", mi) if ids else None
    did = _series(np.arange(len(d_strings)) + 1000, "did", di) if ids else None
    corpus = StringGrouperCorpus(pd.concat([m, d]), min_similarity=0.5)
    pd.testing.assert_frame_equal(corpus.match_strings(m, d, mid, did),
                                  api.match_strings(m, d, mid, did, min_similarity=0.5))
    got = corpus.match_most_similar(m, d, mid, did)
    want = api.match_most_similar(m, d, mid, did, min_similarity=0.5)
    (pd.testing.assert_frame_equal if isinstance(want, pd.DataFrame) else pd.testing.assert_series_equal)(got, want)
    left = m[:len(d)]
    pair_corpus = StringGrouperCorpus(pd.concat([left, d]))
    pd.testing.assert_series_equal(pair_corpus.compute_pairwise_similarities(left, d),
                                   api.compute_pairwise_similarities(left, d))
    # each call transformed its own Series (master ++ duplicates in one pass), nothing else
    assert standin.transformed == [len(m) + len(d), len(m) + len(d), 2 * len(d)]


# ---------------------------------------------------------------------------------------------------------------
# new data against the corpus
# ---------------------------------------------------------------------------------------------------------------

def test_new_batch_against_the_corpus_uses_the_corpus_vocabulary(standin, names):
    s = _series(names)
    corpus = StringGrouperCorpus(s, min_similarity=0.4)
    batch = _series(make_names(80, seed=12) + ["Zyx Qwv", ""] + names[:5])
    sg = corpus.fit(batch, s)
    assert standin.transformed == [len(batch)]           # the corpus is the right operand, not vectorised again
    vec = TfidfVectorizer(min_df=1, analyzer=P.n_grams).fit(names)
    M, D = vec.transform(batch.tolist()), vec.transform(names)
    want = P.matches_list(P.build_matches(M, D, None, 20, 0.4))
    for col in ("master_side", "dupe_side"):
        assert np.array_equal(sg._matches_list[col].to_numpy(), want[col].to_numpy()), col
    # the stand-in product sums in its own order; the CUDA path is checked bit for bit in tests/test_gpu_corpus.py
    np.testing.assert_allclose(sg._matches_list.similarity.to_numpy(), want.similarity.to_numpy(), rtol=1e-12)
    frame = corpus.match_strings(batch, s)
    assert list(frame.columns) == ["left_index", "left_side", "similarity", "right_side", "right_index"]
    assert corpus.n_docs == len(names)
    assert corpus.feature_names() == vec.get_feature_names_out().tolist()
    assert np.array_equal(corpus.idf_, vec.idf_)


def test_fit_returns_a_fitted_string_grouper(standin, names):
    s = _series(names)
    corpus = StringGrouperCorpus(s)
    batch = _series(names[:40])
    sg = corpus.fit(batch, s)
    assert isinstance(sg, api.StringGrouper) and sg.is_build
    n = len(sg._matches_list)
    sg.add_match(names[0], names[1])
    assert len(sg._matches_list) > n
    sg.remove_match(names[0], names[1])
    assert len(sg.get_matches()) <= n


def test_method_kwargs_override_the_corpus_defaults(standin, names):
    s = _series(names)
    corpus = StringGrouperCorpus(s, min_similarity=0.95, max_n_matches=2)
    assert corpus.fit(s)._config.min_similarity == 0.95
    sg = corpus.fit(s, min_similarity=0.5)
    assert sg._config.min_similarity == 0.5 and sg._config.max_n_matches == 2
    assert corpus._config.min_similarity == 0.95          # the defaults themselves do not change
    assert len(corpus.match_strings(s, min_similarity=0.5)) > len(corpus.match_strings(s))


# ---------------------------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("option", [{"ngram_size": 2}, {"regex": r"[aeiou]"}, {"ignore_case": False},
                                    {"normalize_to_ascii": False}, {"tfidf_matrix_dtype": np.float32}])
def test_changing_a_vectoriser_option_raises(standin, names, option):
    s = _series(names)
    corpus = StringGrouperCorpus(s)
    with pytest.raises(ValueError, match=next(iter(option))):
        corpus.match_strings(s, **option)
    with pytest.raises(ValueError):
        corpus.compute_pairwise_similarities(s, s, **option)
    with pytest.raises(ValueError):
        corpus.fit(s).update_options(**option)
    same = {k: getattr(corpus._config, k) for k in option}
    corpus.match_strings(s, **same)                          # restating the corpus's own value is allowed


def test_unknown_option_raises_like_the_config(standin, names):
    with pytest.raises(Exception) as ref:
        StringGrouperConfig(no_such_option=1)
    s = _series(names)
    with pytest.raises(ref.type):
        StringGrouperCorpus(s, no_such_option=1)
    corpus = StringGrouperCorpus(s)
    with pytest.raises(ref.type):
        corpus.match_strings(s, no_such_option=1)


def test_empty_vocabulary_raises_value_error(standin):
    with pytest.raises(ValueError, match="empty vocabulary"):
        StringGrouperCorpus(_series(["", "ab", " . "]))
    with pytest.raises(TypeError):
        StringGrouperCorpus(pd.Series([1, 2]))


# ---------------------------------------------------------------------------------------------------------------
# new symbols through a fitted alphabet (the host half of the sorted transform)
# ---------------------------------------------------------------------------------------------------------------

def test_fitted_byte_lut():
    alphabet = np.array([ord(c) for c in "abcz"], dtype=np.uint32)
    data = np.frombuffer(b"A b,cZy-q", dtype=np.uint8)
    flags = _lib.SG_FLAG_IGNORE_CASE | _lib.SG_FLAG_STRIP_DEFAULT
    lut = _ingest.fitted_byte_lut(data, flags, alphabet)
    assert lut[ord("A")] == 0 and lut[ord("b")] == 1 and lut[ord("c")] == 2 and lut[ord("Z")] == 3
    assert lut[ord(" ")] == lut[ord(",")] == lut[ord("-")] == 0xff            # deleted by the default regex
    # 'y' sits between 'c' and 'z': a nearest id would alias one of them
    assert lut[ord("y")] == lut[ord("q")] == _lib.SG_LUT_UNKNOWN
    assert lut[ord("x")] == 0xff                                                 # absent from the data
    assert _ingest.fitted_byte_lut(data, 0, alphabet)[ord("A")] == _lib.SG_LUT_UNKNOWN   # not folded: no 'A'


def test_fitted_symbol_ids():
    alphabet = np.array([0x61, 0x62, 0xe9, 0x4e2d], dtype=np.uint32)
    cps = np.array([0x61, 0xe9, 0xe8, 0x4e2d, 0x10000, 0x60, 0x62], dtype=np.uint32)
    ids = _ingest.fitted_symbol_ids(cps, alphabet)
    U = _lib.SG_SYMBOL_UNKNOWN
    assert ids.dtype == np.uint32 and ids.tolist() == [0, 2, U, 3, U, U, 1]
    assert _ingest.fitted_symbol_ids(cps, np.zeros(0, np.uint32)).tolist() == [U] * len(cps)

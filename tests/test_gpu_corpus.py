"""-m gpu: StringGrouperCorpus — the K1 transform bit for bit against scikit-learn, the identities with the
module-level functions, new data against the exact pipeline, and the reuse of the corpus's device state.

* K1 transform: `TfidfVectorizer(analyzer=oracle.pipeline.n_grams(...)).fit(corpus).transform(x)` on every
  vectoriser path, with n-grams and characters the corpus does not have (chosen so that mapping an unknown character
  to a neighbouring symbol id would alias a real n-gram), rows without a known n-gram, empty and long strings, and
  both representation mismatches of normalize_to_ascii=False (an ASCII corpus queried with non-ASCII text, a
  code-point corpus queried with ASCII text).
* New data: `corpus.fit(batch, corpus_series)` / `corpus.fit(batch)` against sklearn's transformed matrices, the exact
  top-n product (tests/exact_topn.py) and, for a self-match, the reference's fix-diagonal / symmetrise.
* Reuse: launch counters across calls whose argument is the corpus Series object.
"""
import numpy as np
import pandas as pd
import pytest
from sklearn.feature_extraction.text import TfidfVectorizer

from exact_topn import exact_topn, to_csr
from synth_corpus import make_names
from test_gpu_pipeline_exact import K1_PATHS, edge_corpus
from test_gpu_tfidf import EDGE, UNICODE

pytestmark = pytest.mark.gpu

ABSENT_ASCII = "j"     # removed from the corpus; 'k' (its neighbour in any alphabet holding 'i' and 'k') stays


def perturb(name, rng):
    """a near copy of `name`: one character dropped, doubled or swapped with its neighbour, or a suffix"""
    if len(name) < 4:
        return name + " co"
    i = int(rng.integers(1, len(name) - 2))
    op = int(rng.integers(4))
    if op == 0:
        return name[:i] + name[i + 1:]
    if op == 1:
        return name[:i] + name[i] + name[i:]
    if op == 2:
        return name[:i] + name[i + 1] + name[i] + name[i + 2:]
    return name + " inc"


def _no_j(s):
    return s.replace(ABSENT_ASCII, "i").replace(ABSENT_ASCII.upper(), "I")


@pytest.fixture(scope="module")
def corpora():
    """(ASCII-only corpus, corpus with non-ASCII text), neither holding 'j' / 'J' nor 'ó'"""
    ascii_ = [_no_j(s) for s in make_names(3000, seed=61) + [e for e in edge_corpus() if e.isascii()]]
    mixed = ascii_[:2000] + [_no_j(s) for s in edge_corpus() + EDGE + UNICODE]
    assert not any("ó" in s for s in mixed)
    return ascii_, mixed


@pytest.fixture(scope="module")
def queries(corpora):
    """(ASCII-only batch, batch with non-ASCII text)"""
    ascii_, mixed = corpora
    rng = np.random.default_rng(62)
    # 'j' where the corpus has 'k' / 'i': a nearest-id mapping of 'j' would turn these rows into corpus n-grams
    aliasing = [s.replace("k", "j").replace("K", "J") for s in ascii_[:300] if "k" in s.lower()]
    aliasing += [s.replace("i", "j") for s in ascii_[300:400]]
    unknown_ngrams = ["zqzqzq xvxv", "qqqqqqqqqq", "jjjj", "@@@ ###", "x", "", "", "  ", "jjjjjjjj" * 40]
    long_rows = [" ".join(ascii_[i:i + 20]) for i in range(0, 400, 20)]        # well over 256 bytes
    perturbed = [perturb(s, rng) for s in ascii_[:500]]
    batch_ascii = (make_names(800, seed=63) + aliasing + unknown_ngrams + long_rows + perturbed
                   + [e for e in EDGE + edge_corpus() if e.isascii()])
    # 'ó' lies between the corpus's 'é' and 'ø': a nearest id would alias 'ø'
    non_ascii = ["Straße 7 & Són", "Són", "són søn", "óóóó",
                 "東京ЖЖЖ", "Ж" * 300, "café müller", "Café Müller GmbH"]
    batch_mixed = batch_ascii[:600] + non_ascii + EDGE + UNICODE + edge_corpus()[:12]
    return batch_ascii, batch_mixed


def _sklearn(corpus, kw):
    from oracle import pipeline as P
    dtype = kw.get("tfidf_matrix_dtype", np.float64)
    akw = {k: v for k, v in kw.items() if k != "tfidf_matrix_dtype"}
    return TfidfVectorizer(min_df=1, analyzer=lambda s: P.n_grams(s, **akw), dtype=dtype).fit(corpus)


def _device_transform(corpus, strings):
    m, _ = corpus._matrices(pd.Series(strings), None, {})
    return m


def _assert_same_csr(got, want, dtype, label):
    got, want = got.to_scipy(), want.tocsr()
    assert got.shape == want.shape, label
    assert got.dtype == want.dtype == dtype, label
    assert np.array_equal(got.indptr, want.indptr), label
    assert np.array_equal(got.indices, want.indices), label
    bad = np.flatnonzero(got.data != want.data)
    assert len(bad) == 0, "%s: %d of %d values differ" % (label, len(bad), len(want.data))


@pytest.mark.parametrize("kw", K1_PATHS)
def test_k1_transform_equals_sklearn(kw, corpora, queries):
    from string_grouper_b200 import StringGrouperCorpus
    dtype = kw.get("tfidf_matrix_dtype", np.float64)
    for c_label, strings in zip(("ascii corpus", "non-ascii corpus"), corpora):
        vec = _sklearn(strings, kw)
        corpus = StringGrouperCorpus(pd.Series(strings), **kw)
        names, idf = vec.get_feature_names_out().tolist(), vec.idf_
        assert corpus.feature_names() == names
        assert corpus.idf_.dtype == idf.dtype == dtype and np.array_equal(corpus.idf_, idf)
        assert corpus.n_docs == len(strings)
        for q_label, batch in zip(("ascii batch", "non-ascii batch"), queries):
            got = _device_transform(corpus, batch)
            _assert_same_csr(got, vec.transform(batch), dtype, "%s / %s / %s" % (kw, c_label, q_label))
            assert np.diff(got.to_scipy().indptr).min() == 0          # rows without a known n-gram are there
        # the corpus matrix is transform(corpus); the vocabulary and idf did not move
        _assert_same_csr(_device_transform(corpus, strings), vec.transform(strings), dtype, "%s / self" % kw)
        assert corpus.feature_names() == names and np.array_equal(corpus.idf_, idf)


def test_k1_transform_long_rows_and_runs():
    """documents far above the 256-symbol shared-memory cap, and long runs of one n-gram, on both forms"""
    from string_grouper_b200 import StringGrouperCorpus
    corpus = [_no_j(s) for s in make_names(2000, seed=64)] + ["ab" * 3000]
    batch = ["ab" * 50_000, "ab" * 128 + "j" + "ab" * 128, "j" * 1000, ("ab" * 20 + "j") * 40, "q" * 5000]
    for kw in ({}, {"ngram_size": 5}, {"ngram_size": 2, "tfidf_matrix_dtype": np.float32}):
        vec = _sklearn(corpus, kw)
        c = StringGrouperCorpus(pd.Series(corpus), **kw)
        _assert_same_csr(_device_transform(c, batch), vec.transform(batch), kw.get("tfidf_matrix_dtype", np.float64),
                         str(kw))


# ---------------------------------------------------------------------------------------------------------------
# identities with the module-level functions
# ---------------------------------------------------------------------------------------------------------------

def _assert_equal(got, want):
    (pd.testing.assert_frame_equal if isinstance(want, pd.DataFrame) else pd.testing.assert_series_equal)(got, want)


@pytest.mark.parametrize("ids", [False, True])
@pytest.mark.parametrize("index", [None, "shifted"])
def test_identities_self_match(ids, index):
    import string_grouper_b200 as api
    names = make_names(3000, seed=65)
    names += [perturb(s, np.random.default_rng(66)) for s in names[:300]]
    idx = None if index is None else pd.Index(np.arange(len(names)) * 5 + 3, name="key")
    s = pd.Series(names, name="name", index=idx)
    sid = pd.Series(["id%d" % i for i in range(len(names))], name="id", index=idx) if ids else None
    corpus = api.StringGrouperCorpus(s, min_similarity=0.7)
    _assert_equal(corpus.match_strings(s, master_id=sid), api.match_strings(s, master_id=sid, min_similarity=0.7))
    for rep in ("centroid", "first"):
        _assert_equal(corpus.group_similar_strings(s, string_ids=sid, group_rep=rep),
                      api.group_similar_strings(s, string_ids=sid, group_rep=rep, min_similarity=0.7))


@pytest.mark.parametrize("ids", [False, True])
@pytest.mark.parametrize("index", [None, "labels"])
def test_identities_two_series(ids, index):
    import string_grouper_b200 as api
    rng = np.random.default_rng(67)
    ms = make_names(2500, seed=68)
    ds = make_names(700, seed=69) + [perturb(s, rng) for s in ms[:500]]
    mi = None if index is None else pd.Index(["m%d" % i for i in range(len(ms))], name="mk")
    di = None if index is None else pd.Index(["d%d" % i for i in range(len(ds))])
    m, d = pd.Series(ms, name="master", index=mi), pd.Series(ds, index=di)
    mid = pd.Series(np.arange(len(ms)), name="mid", index=mi) if ids else None
    did = pd.Series(np.arange(len(ds)) + 10**6, name="did", index=di) if ids else None
    corpus = api.StringGrouperCorpus(pd.concat([m, d]), min_similarity=0.6)
    _assert_equal(corpus.match_strings(m, d, mid, did), api.match_strings(m, d, mid, did, min_similarity=0.6))
    _assert_equal(corpus.match_most_similar(m, d, mid, did),
                  api.match_most_similar(m, d, mid, did, min_similarity=0.6))
    left = m.iloc[:len(d)]
    pair = api.StringGrouperCorpus(pd.concat([left, d]))
    _assert_equal(pair.compute_pairwise_similarities(left, d), api.compute_pairwise_similarities(left, d))


# ---------------------------------------------------------------------------------------------------------------
# new data, exact
# ---------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def corpus20k():
    from string_grouper_b200 import StringGrouperCorpus
    names = make_names(20_000, seed=91)
    s = pd.Series(names)
    rng = np.random.default_rng(70)
    batch = make_names(2000, seed=71) + [perturb(names[i], rng) for i in rng.integers(0, len(names), 1500)]
    return s, StringGrouperCorpus(s), _sklearn(names, {}), batch


def _exact_list(M, D, self_match, max_n_matches=20, min_similarity=0.8):
    from oracle import pipeline as P
    top_n = min(int(max_n_matches), D.shape[0])
    r, c, sc, max_row = exact_topn(M, D, top_n, min_similarity)
    C = to_csr((r, c, sc), (M.shape[0], D.shape[0]))
    if self_match:
        C = P.fix_diagonal_and_symmetrize(C)
    return P.matches_list(C), max_row


def _assert_same_list(got, want, label):
    for col in ("master_side", "dupe_side", "similarity"):
        g, w = got[col].to_numpy(), want[col].to_numpy()
        assert g.shape == w.shape and np.array_equal(g, w), "%s: %s differs (%d vs %d rows)" % (label, col, len(g),
                                                                                              len(w))


@pytest.mark.parametrize("min_similarity,floor", [(0.8, None), (0.3, True)])
def test_new_data_exact(min_similarity, floor, corpus20k, monkeypatch):
    from string_grouper_b200 import _device as D
    s, corpus, vec, batch = corpus20k
    if floor is not None:
        monkeypatch.setattr(D, "TOPN_FLOOR", floor)
    b = pd.Series(batch)
    Mb, Ms = vec.transform(batch), vec.transform(s.tolist())
    for label, (left, right), (M, R) in (("batch x corpus", (b, s), (Mb, Ms)), ("batch self-match", (b, None), (Mb, Mb)),
                                         ("corpus x batch", (s, b), (Ms, Mb))):
        sg = corpus.fit(left, right, min_similarity=min_similarity)
        want, true_max = _exact_list(M, R, right is None, min_similarity=min_similarity)
        _assert_same_list(sg._matches_list, want, "%s at %s" % (label, min_similarity))
        assert sg._true_max_n_matches == true_max, label
        if floor:
            assert sg._last_stats["topn_floor"] is True


# ---------------------------------------------------------------------------------------------------------------
# reuse of the corpus's device state
# ---------------------------------------------------------------------------------------------------------------

def test_reuse_from_counters(corpus20k):
    """the corpus Series as an argument costs no K1 launch; as the right operand its row order and postings are built
    once.  A second batch adds its own K1 transform (dense form: count, known keys, values) and its own left-row order
    (sg_row_order: 2 launches), nothing for the corpus."""
    from string_grouper_b200 import _device as D
    s, corpus, _, batch = corpus20k
    b1, b2 = pd.Series(batch[:1500]), pd.Series(batch[1500:3000])

    def delta(call):
        before = dict(D.LAUNCH_COUNTS)
        call()
        return {k: D.LAUNCH_COUNTS[k] - before[k] for k in before}

    d = delta(lambda: corpus.match_strings(b1, s))
    assert d["tfidf"] == 3
    d = delta(lambda: corpus.match_strings(b2, s))
    assert d["tfidf"] == 3 and d["postings"] == 0 and d["order"] == 2, d
    d = delta(lambda: corpus.match_most_similar(s, b2))
    assert d["tfidf"] == 3, d
    corpus.match_strings(s)
    d = delta(lambda: corpus.match_strings(s))
    assert d["tfidf"] == 0 and d["postings"] == 0 and d["order"] == 0 and d["dedup"] == 0, d


def test_sorted_form_launches():
    from string_grouper_b200 import StringGrouperCorpus
    from string_grouper_b200 import _device as D
    names = make_names(3000, seed=72)
    s = pd.Series(names)
    corpus = StringGrouperCorpus(s, ngram_size=5)
    before = D.LAUNCH_COUNTS["tfidf"]
    corpus.match_strings(pd.Series(names[:100]), s)
    assert D.LAUNCH_COUNTS["tfidf"] - before == 4          # count, known keys, place, values


# ---------------------------------------------------------------------------------------------------------------
# argument checks
# ---------------------------------------------------------------------------------------------------------------

def test_argument_checks():
    from string_grouper_b200 import StringGrouperConfig, StringGrouperCorpus
    s = pd.Series(make_names(500, seed=73))
    corpus = StringGrouperCorpus(s)
    for option in ({"ngram_size": 4}, {"regex": "x"}, {"ignore_case": False}, {"normalize_to_ascii": False},
                   {"tfidf_matrix_dtype": np.float32}):
        with pytest.raises(ValueError):
            corpus.match_strings(s, **option)
    with pytest.raises(Exception) as ref:
        StringGrouperConfig(bogus=1)
    with pytest.raises(ref.type):
        corpus.match_most_similar(s, s, bogus=1)
    with pytest.raises(ValueError, match="empty vocabulary"):
        StringGrouperCorpus(pd.Series(["", "a", "b."]))

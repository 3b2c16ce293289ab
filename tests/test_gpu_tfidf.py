"""-m gpu: K1 (device n-gram TF-IDF) against sklearn driven by the reference analyzer (the oracle), bit for bit, and
against the reference's own matrix stored in tests/golden/synthetic.npz."""
import os

import numpy as np
import pandas as pd
import pytest

from synth_corpus import make_names

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "synthetic.npz"), allow_pickle=True)

EDGE = ["", "ab", "abc", "A.B,C-D/E F\tG", "ÀbracâDABRÀ", "ﬁ½① İstanbul", "x" * 300 + " inc", "aaa aaa aaa aaaa"]


def _device_matrices(master, dupes=None, **kw):
    from string_grouper_b200 import StringGrouper
    sg = StringGrouper(pd.Series(master), None if dupes is None else pd.Series(dupes), **kw)
    m, d = sg._get_tf_idf_matrices()
    return sg, m, d


def _assert_same_csr(got, ref):
    """equal bit for bit: K1 computes idf with numpy on the host exactly as scikit-learn does"""
    got, ref = got.to_scipy(), ref.tocsr()
    assert got.shape == ref.shape
    assert np.array_equal(got.indptr, ref.indptr)
    assert np.array_equal(got.indices, ref.indices)
    assert got.dtype == ref.dtype
    assert np.array_equal(got.data, ref.data), "%d values differ" % (got.data != ref.data).sum()


def test_matrix_equals_reference_golden():
    """The golden matrix was written on another host: its idf carries that host's numpy `log` (picked by CPU
    dispatch), which may differ from this host's in the last bit, so the values are compared with a tolerance here;
    the exact comparisons are against live scikit-learn below."""
    texts = make_names(500, seed=14) + EDGE
    sg, m, _ = _device_matrices(texts)
    got = m.to_scipy()
    assert np.array_equal(got.indptr, GOLD["tfidf_indptr"]) and np.array_equal(got.indices, GOLD["tfidf_indices"])
    np.testing.assert_allclose(got.data, GOLD["tfidf_data"], rtol=1e-14, atol=0)
    assert sg._vocabulary.feature_names() == GOLD["tfidf_vocab"].tolist()
    _, m32, _ = _device_matrices(texts, tfidf_matrix_dtype=np.float32)
    assert m32.to_scipy().dtype == np.float32
    np.testing.assert_allclose(m32.to_scipy().data, GOLD["tfidf32_data"], rtol=2e-6, atol=0)


@pytest.mark.parametrize("kw", [{}, {"ngram_size": 2}, {"ngram_size": 4}, {"ngram_size": 1}, {"ignore_case": False},
                                {"tfidf_matrix_dtype": np.float32}, {"regex": r"[aeiou\s]"},
                                # sorted-vocabulary vectoriser (csrc/sg_tfidf64.cu): keys beyond 21 bits
                                {"ngram_size": 5}, {"ngram_size": 7, "tfidf_matrix_dtype": np.float32},
                                {"ngram_size": 9, "ignore_case": False}, {"ngram_size": 4, "regex": r"[aeiou\s]"}])
def test_matrix_equals_sklearn_oracle(kw):
    from oracle import pipeline as P
    master = make_names(6000, seed=31) + EDGE + ["Q" * 1000, "lorem ipsum " * 60]
    dupes = make_names(2500, seed=32) + ["zzzz", ""]
    _, m, d = _device_matrices(master, dupes, **kw)
    okw = dict(kw)
    dtype = okw.pop("tfidf_matrix_dtype", np.float64)
    rm, rd, _ = P.tf_idf_matrices(master, dupes, dtype=dtype, **okw)
    _assert_same_csr(m, rm)
    _assert_same_csr(d, rd)


UNICODE = ["Caf\u00e9 M\u00fcller GmbH", "Cafe Muller GmbH", "CAF\u00c9 M\u00dcLLER GMBH", "\u6771\u4eac\u682a\u5f0f\u4f1a\u793e",
           "\u6771\u4eac\u682a\u5f0f\u4f1a\u793e\u30db\u30fc\u30eb\u30c7\u30a3\u30f3\u30b0\u30b9", "\u0130stanbul A.\u015e.", "istanbul a.s.",
           "Stra\u00dfe 7 & S\u00f8n", "strasse\u00a07\u2003& son", "\U0001F600 emoji co", "emoji co", "", "\u00e9"]


@pytest.mark.parametrize("kw", [{}, {"ngram_size": 2}, {"ignore_case": False}, {"tfidf_matrix_dtype": np.float32},
                                {"ngram_size": 4}])
def test_code_point_ngrams_equal_sklearn_oracle(kw):
    """normalize_to_ascii=False keeps the non-ASCII characters: n-grams over code points (string_grouper.py:374-378),
    Python's lower() and the regex's Unicode white space handled like the reference."""
    from oracle import pipeline as P
    master = make_names(800, seed=33) + UNICODE
    dupes = UNICODE[:5] + make_names(100, seed=34)
    sg, m, d = _device_matrices(master, dupes, normalize_to_ascii=False, **kw)
    okw = dict(kw)
    dtype = okw.pop("tfidf_matrix_dtype", np.float64)
    rm, rd, vec = P.tf_idf_matrices(master, dupes, dtype=dtype, normalize_to_ascii=False, **okw)
    _assert_same_csr(m, rm)
    _assert_same_csr(d, rd)
    vocab = vec.vocabulary_
    assert sg._vocabulary.feature_names() == sorted(vocab, key=vocab.get)


def test_sorted_vocabulary_feature_names_and_key_limit():
    from oracle import pipeline as P
    from string_grouper_b200 import StringGrouper
    names = make_names(3000, seed=35)
    sg = StringGrouper(pd.Series(names), ngram_size=6)
    sg._get_tf_idf_matrices()
    _, _, vec = P.tf_idf_matrices(names, ngram_size=6)
    vocab = vec.vocabulary_
    assert sg._vocabulary.feature_names() == sorted(vocab, key=vocab.get)
    assert "64-bit" in sg._last_stats.get("vectoriser", "") or "bit keys" in sg._last_stats.get("vectoriser", "")
    # n * ceil(log2(alphabet)) > 64: a clear error instead of a wrong answer
    with pytest.raises(NotImplementedError):
        StringGrouper(pd.Series(names), ngram_size=14)._get_tf_idf_matrices()


def test_capital_ascii_from_nfkd_is_not_folded_again():
    """str.lower() runs before NFKD in the reference analyzer (:372-375); NFKD of the trade-mark / numero / degree
    signs yields CAPITAL ASCII that must survive ('acmeTMcorp', not 'acmetmcorp')."""
    from oracle import pipeline as P
    texts = ["Acme\u2122 Corp", "ACME TM CORP", "AcmeTM Corp", "\u2116 5 Ltd", "No 5 Ltd", "Degree \u2103 Inc",
             "plain ascii"] + make_names(200, seed=36)
    sg, m, _ = _device_matrices(texts)
    rm, _, vec = P.tf_idf_matrices(texts)
    _assert_same_csr(m, rm)
    assert "eTM" in sg._vocabulary.feature_names()


def test_reference_fixture_build_matrix():
    """test_build_matrix / test_build_matrix_master_and_duplicates (reference tests :519-544): exact values."""
    _, m, d = _device_matrices(['foo', 'bar', 'baz'])
    np.testing.assert_array_equal(m.toarray(), np.array([[0., 0., 1.], [1., 0., 0.], [0., 1., 0.]]))
    _, m, d = _device_matrices(['foo', 'bar', 'baz'], ['foo', 'bar', 'bop'])
    np.testing.assert_array_equal(m.toarray(), np.array([[0., 0., 0., 1.], [1., 0., 0., 0.], [0., 1., 0., 0.]]))
    np.testing.assert_array_equal(d.toarray(), np.array([[0., 0., 0., 1.], [1., 0., 0., 0.], [0., 0., 1., 0.]]))


def test_full_pipeline_matches_oracle_fit():
    from oracle import pipeline as P
    from parity import compare_triples
    from string_grouper_b200 import StringGrouper
    names = make_names(20000, seed=41)
    sg = StringGrouper(pd.Series(names)).fit()
    got = sg._matches_list
    ref, true_max = P.fit(names, n_threads=4, fast_symmetrize=True)
    m, d, _ = P.tf_idf_matrices(names)
    C = P.build_matches(m, d, None, 20, 0.8, n_threads=4)
    from parity import row_cutoffs
    cut = row_cutoffs(C.indptr, C.data, 20, len(names))
    st = compare_triples((ref.master_side, ref.dupe_side, ref.similarity),
                         (got.master_side, got.dupe_side, got.similarity), len(names), 0.8, tol=1e-9,
                         cutoff_row=cut, cutoff_col=cut, label="fit 20k")
    assert st["common"] >= 0.97 * st["pairs_ref"]     # the rest are top-n ties inside clusters of identical names
    assert sg._true_max_n_matches == true_max
    # storage order of the symmetrised list: row ascending, column ascending (ref test_get_matches_single)
    key = got.master_side.to_numpy() * len(names) + got.dupe_side.to_numpy()
    assert np.all(np.diff(key) > 0)


def test_match_strings_two_series_frame_equals_oracle():
    from oracle import pipeline as P
    import string_grouper_b200 as api
    master = pd.Series(make_names(5000, seed=51), name="company")
    dupes = pd.Series(make_names(1500, seed=52) + make_names(5000, seed=51)[:500])
    out = api.match_strings(master, dupes, min_similarity=0.75, max_n_matches=3)
    ref, _ = P.fit(master.tolist(), dupes.tolist(), min_similarity=0.75, max_n_matches=3, n_threads=4)
    assert list(out.columns) == ["left_index", "left_company", "similarity", "right_side", "right_index"]
    a = set(zip(out.left_index.tolist(), out.right_index.tolist()))
    b = set(zip(ref.master_side.tolist(), ref.dupe_side.tolist()))
    assert len(a ^ b) <= 0.01 * len(b)         # top-3 ties between identical strings may differ
    assert (out.left_company.to_numpy() == master.to_numpy()[out.left_index.to_numpy()]).all()


@pytest.mark.parametrize("group_rep", ["centroid", "first"])
def test_group_representatives_equal_host_rule(group_rep):
    """device connected components / centroid choice (csrc/sg_groups.cu) vs the scipy statement of
    StringGrouper._deduplicate (reference string_grouper.py:851-904) on the same match list."""
    from string_grouper_b200 import StringGrouper
    names = pd.Series(make_names(30000, seed=61), name="name")
    sg = StringGrouper(names, min_similarity=0.8, group_rep=group_rep).fit()
    assert sg._matches_device is not None
    dev = sg.get_groups()
    sg._matches_device = None          # same object, host rule
    host = sg.get_groups()
    pd.testing.assert_frame_equal(dev, host)
    assert (dev["group_rep_index"] != np.arange(len(names))).sum() > 1000


def test_device_string_gather_equals_host_take():
    """get_matches with the strings gathered on the device (csrc/sg_gather.cu) vs pandas/Arrow take."""
    import string_grouper_b200 as api
    master = pd.Series(make_names(20000, seed=71), name="company")
    dupes = pd.Series(make_names(6000, seed=72) + make_names(20000, seed=71)[:500] + ["", "x"])
    for args in [(master,), (master, dupes)]:
        sg = api.StringGrouper(*args, min_similarity=0.75).fit()
        assert sg._raw_device is not None and sg._matches_device is not None
        dev = sg.get_matches()
        sg._raw_device = None
        host = sg.get_matches()
        pd.testing.assert_frame_equal(dev, host)
        assert len(dev) > 2000
    # non-ASCII input is normalised on the host: the device copy is not the callers' text, so the host path is taken
    odd = pd.Series(["Ünited Çorp", "United Corp", "Ünited Çorp."])
    sg = api.StringGrouper(odd, min_similarity=0.5).fit()
    assert sg._raw_device is None
    assert sg.get_matches()["left_side"].tolist()[0] == "Ünited Çorp"


def test_degenerate_inputs():
    import string_grouper_b200 as api
    # strings shorter than ngram_size give empty rows but still match themselves (reference fit(), :419-427)
    out = api.match_strings(pd.Series(["ab", "abc", "abc.", "x", ""]))
    pairs = set(zip(out.left_index.tolist(), out.right_index.tolist()))
    assert pairs == {(0, 0), (1, 1), (1, 2), (2, 1), (2, 2), (3, 3), (4, 4)}
    assert out.similarity.min() >= 1.0 - 1e-12
    # one row
    assert len(api.match_strings(pd.Series(["hello world"]))) == 1
    # nothing to vectorise at all: scikit-learn's error, as in the reference
    with pytest.raises(ValueError):
        api.match_strings(pd.Series(["a", "b"]))
    # no match above the threshold between two Series
    out = api.match_strings(pd.Series(["alpha beta"]), pd.Series(["gamma delta", "epsilon"]))
    assert len(out) == 0 and list(out.columns) == ["left_index", "left_side", "similarity", "right_side", "right_index"]
    # groups on a tiny input
    g = api.group_similar_strings(pd.Series(["foo inc", "foo inc.", "bar"]))
    assert g["group_rep_index"].tolist() == [0, 0, 2]


@pytest.mark.parametrize("kw", [{}, {"ngram_size": 2}, {"ngram_size": 5}, {"normalize_to_ascii": False}])
def test_vectoriser_df_is_the_feature_df_of_the_matrix(kw):
    """Self-match: the matrix holds exactly the fitted rows, so K1 hands its document frequencies (column order)
    to K2 instead of a second count (sg_feature_df); with two Series nothing is handed over."""
    import ctypes
    from string_grouper_b200 import _device as D, _lib
    texts = make_names(3000, seed=5) + EDGE
    _, m, _ = _device_matrices(texts, **kw)
    assert m._df is not None
    handed = m._df.cpu().numpy()[:m.shape[1]].copy()
    m._df = None
    counted = D.feature_df(m).cpu().numpy()
    ref = np.bincount(m.to_scipy().indices, minlength=m.shape[1])
    assert np.array_equal(counted, ref) and np.array_equal(handed, ref)
    # the heavy-feature ranks are the same whether sg_heavy_features counts or is given the frequencies
    t, L = D.torch(), _lib.load()
    ws_bytes = int(L.sg_order_workspace_bytes(m.shape[0], m.shape[1]))
    ws = t.empty(ws_bytes, dtype=t.uint8, device=m.device)
    own = t.empty(m.shape[1], dtype=t.int8, device=m.device)
    _lib.check(L.sg_heavy_features(m.shape[0], m.shape[1], ctypes.c_void_p(m.d_indptr.data_ptr()),
                                   ctypes.c_void_p(m.d_indices.data_ptr()), None, 64,
                                   ctypes.c_void_p(own.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ws_bytes, D._stream()))
    t.cuda.synchronize()
    assert np.array_equal(own.cpu().numpy(), D.heavy_features(m).cpu().numpy())
    _, master, dup = _device_matrices(texts[:2000], texts[2000:], **kw)
    assert master._df is None and dup._df is None

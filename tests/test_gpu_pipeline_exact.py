"""-m gpu: from strings to the match list with no tolerance.

* K1 against live scikit-learn (oracle.pipeline.tf_idf_matrices, the real TfidfVectorizer): indptr, indices and
  values bit for bit, the dtype, the feature names and `vocab.idf_ == vec.idf_`, on every vectoriser path and on a
  corpus built for K1's edges (shared memory / HBM scratch at 256 raw bytes, run-length carries across 32-key
  chunks, the grid-stride loops, a 64-bit key that is all ones).
* The whole pipeline against tests/exact_pipeline.py: `_matches_list` and `_true_max_n_matches`, then
  get_groups, match_most_similar and compute_pairwise_similarities on that exact list.
* 663k: K1's matrix of the benchmark corpus is scikit-learn's, so tests/test_gpu_fullsize.py's comparisons hold
  from the strings on.
"""
import time

import numpy as np
import pandas as pd
import pytest

from exact_pipeline import COMMON_COUNTS, common_count_pairs, distinct_ngram_word, exact_match_list
from synth_corpus import make_names

pytestmark = pytest.mark.gpu


def edge_corpus(seed=0):
    """Strings at K1's edges (see the module docstring), in no particular order."""
    rng = np.random.default_rng(seed)
    letters = list("abcdefghijklmnopqrstuvwxyz     ")

    def text(n):
        return "".join(rng.choice(letters, n))

    out = [text(n) for n in (255, 256, 257, 5000)]                # raw bytes around the 256-byte shared-memory cap
    out.append("ab. " * 75)                                       # 300 raw bytes that clean to 150 characters
    for r in (1, 31, 32, 33, 64, 65, 1000):                       # one n-gram's run over r positions, after others
        out += ["q" * (r + 2), "bcd" + "q" * (r + 2) + "xy"]
    for k in (31, 32, 33, 64, 65):                                # exactly k distinct n-grams (the norm loop)
        out.append(distinct_ngram_word(k, rng))
    out.append("ab" * 50_000)
    out += ["", "", "a", "ab", " ,.-/ \t", "-/-/", "A.B,C-D/E F\tG", "ÀbracâDABRÀ", "ﬁ½① İstanbul"]
    return out


def _k1(master, dupes=None, **kw):
    from string_grouper_b200 import StringGrouper
    sg = StringGrouper(pd.Series(master), None if dupes is None else pd.Series(dupes), **kw)
    m, d = sg._get_tf_idf_matrices()
    return sg, m, d


def _assert_k1_is_sklearn(master, dupes=None, **kw):
    """K1 and scikit-learn's TfidfVectorizer on the same strings: equal matrices, vocabularies and idf."""
    from oracle import pipeline as P
    sg, m, d = _k1(master, dupes, **kw)
    okw = dict(kw)
    dtype = okw.pop("tfidf_matrix_dtype", np.float64)
    rm, rd, vec = P.tf_idf_matrices(master, dupes, dtype=dtype, **okw)
    for got, ref in ((m, rm), (d, rd)) if dupes is not None else ((m, rm),):
        got, ref = got.to_scipy(), ref.tocsr()
        assert got.shape == ref.shape and got.dtype == ref.dtype == dtype
        assert np.array_equal(got.indptr, ref.indptr)
        assert np.array_equal(got.indices, ref.indices)
        bad = np.flatnonzero(got.data != ref.data)
        assert len(bad) == 0, "%d of %d values differ" % (len(bad), len(ref.data))
    assert sg._vocabulary.feature_names() == vec.get_feature_names_out().tolist()
    idf = sg._vocabulary.idf_
    assert idf.dtype == vec.idf_.dtype == dtype
    bad = np.flatnonzero(idf != vec.idf_)
    assert len(bad) == 0, "%d of %d idf values differ" % (len(bad), len(idf))
    return sg, vec


K1_PATHS = [
    {"ngram_size": 1}, {"ngram_size": 2}, {}, {"tfidf_matrix_dtype": np.float32},
    {"ngram_size": 2, "tfidf_matrix_dtype": np.float32}, {"ignore_case": False}, {"regex": r"[aeiou\s]"},
    # sorted-vocabulary vectoriser (csrc/sg_tfidf64.cu)
    {"ngram_size": 4}, {"ngram_size": 5}, {"ngram_size": 7}, {"ngram_size": 9, "ignore_case": False},
    {"ngram_size": 5, "tfidf_matrix_dtype": np.float32},
    {"normalize_to_ascii": False, "ngram_size": 2}, {"normalize_to_ascii": False},
    {"normalize_to_ascii": False, "ngram_size": 4}, {"normalize_to_ascii": False, "tfidf_matrix_dtype": np.float32},
]


@pytest.fixture(scope="module")
def k1_corpus():
    """30 000 names (the count and values kernels' grid-stride loops wrap more than three times on 132 SMs) and the
    edge corpus spread through them"""
    names = make_names(30_000, seed=81)
    edges = edge_corpus()
    for i, e in enumerate(edges):
        names.insert((i * 7919) % len(names), e)
    return names


@pytest.mark.parametrize("kw", K1_PATHS)
def test_k1_equals_sklearn_master_only(kw, k1_corpus):
    _assert_k1_is_sklearn(k1_corpus, **kw)


@pytest.mark.parametrize("kw", K1_PATHS[::2])
def test_k1_equals_sklearn_master_and_duplicates(kw, k1_corpus):
    _assert_k1_is_sklearn(k1_corpus[:20_000], k1_corpus[20_000:] + make_names(500, seed=82), **kw)


def test_k1_feature_in_every_document_has_idf_one():
    names = [s + " zzq" for s in make_names(3000, seed=83)]
    sg, vec = _assert_k1_is_sklearn(names)
    col = vec.vocabulary_["zzq"]
    assert sg._vocabulary.idf_[col] == 1.0


@pytest.mark.parametrize("kw", [{"ngram_size": 16}, {"ngram_size": 8, "normalize_to_ascii": False, "ignore_case": False}])
def test_k1_all_ones_64_bit_key(kw):
    """n * bits = 64 and the largest symbol repeated n times is present: its key is all ones, like the sort's
    padding.  16 symbols at n = 16; 256 code points at n = 8 (U+0100..U+01FF, case kept: lower() would merge
    some)."""
    rng = np.random.default_rng(84)
    n = kw["ngram_size"]
    if n == 16:
        alphabet = list("abcdefghijklmnop")
    else:
        alphabet = [chr(c) for c in range(0x100, 0x200)]
    top = alphabet[-1]
    docs = ["".join(rng.choice(alphabet, int(rng.integers(n, 3 * n)))) for _ in range(3000)]
    docs += [top * n, top * (n + 40), "".join(alphabet) + top * n, alphabet[0] * n]
    sg, vec = _assert_k1_is_sklearn(docs, **kw)
    assert "bit keys" in sg._last_stats["vectoriser"] and "64-bit" in sg._last_stats["vectoriser"]
    assert vec.get_feature_names_out()[-1] == top * n


# ---------------------------------------------------------------------------------------------------------------
# strings -> match list, no tolerance
# ---------------------------------------------------------------------------------------------------------------

def _assert_same_list(got, want, label):
    for col in ("master_side", "dupe_side", "similarity"):
        g, w = got[col].to_numpy(), want[col].to_numpy()
        assert g.shape == w.shape and np.array_equal(g, w), "%s: %s differs (%d vs %d rows)" % (label, col, len(g),
                                                                                              len(w))


def _fit_exact(master, dupes=None, monkeypatch=None, floor=None, **kw):
    from string_grouper_b200 import StringGrouper
    from string_grouper_b200 import _device as D
    if floor is not None:
        monkeypatch.setattr(D, "TOPN_FLOOR", floor)
    sg = StringGrouper(pd.Series(master), None if dupes is None else pd.Series(dupes), **kw).fit()
    rkw = dict(kw)
    dtype = rkw.pop("tfidf_matrix_dtype", np.float64)
    rkw.pop("group_rep", None)
    want, true_max, mats = exact_match_list(master, dupes, dtype=dtype, **rkw)
    _assert_same_list(sg._matches_list, want, str(kw))
    assert sg._true_max_n_matches == true_max
    return sg, want, mats


@pytest.fixture(scope="module")
def names20k():
    return make_names(20_000, seed=91)


@pytest.fixture(scope="module")
def default_fit(names20k):
    return _fit_exact(names20k)


def test_match_list_20k_self_match_defaults(default_fit):
    sg, want, _ = default_fit
    assert sg._last_stats["triangle"] is True
    assert len(want) > 20_000


@pytest.mark.parametrize("kw", [{"tfidf_matrix_dtype": np.float32}, {"ngram_size": 2, "min_similarity": 0.85},
                                {"ngram_size": 5, "min_similarity": 0.7}])
def test_match_list_self_match(kw, names20k):
    _fit_exact(names20k[:8000], **kw)


def test_match_list_two_series_top3():
    master = make_names(5000, seed=51)
    dupes = make_names(1500, seed=52) + master[:500]
    _fit_exact(master, dupes, min_similarity=0.75, max_n_matches=3)


def test_match_list_non_ascii():
    names = make_names(4000, seed=92)
    odd = ["Café Müller GmbH", "Cafe Muller GmbH", "CAFÉ MÜLLER GMBH", "İstanbul A.Ş.",
           "istanbul a.s.", "Straße 7 & Søn", "strasse 7 & son", "東京株式会社"]
    names = names + odd + [o + " ltd" for o in odd]
    _fit_exact(names, min_similarity=0.6)
    _fit_exact(names, normalize_to_ascii=False, min_similarity=0.6)


@pytest.mark.parametrize("min_similarity", [0.3, 0.0])
def test_match_list_low_threshold_with_floor(min_similarity, monkeypatch):
    names = make_names(4000, seed=93)
    sg, _, _ = _fit_exact(names, monkeypatch=monkeypatch, floor=True, min_similarity=min_similarity)
    assert sg._last_stats["topn_floor"] is True


@pytest.mark.parametrize("group_rep", ["centroid", "first"])
def test_groups_on_the_exact_list(group_rep, names20k):
    from oracle import pipeline as P
    sg, want, _ = _fit_exact(names20k[:12_000], group_rep=group_rep)
    got = sg.get_groups()["group_rep_index"].to_numpy()
    assert np.array_equal(got, P.deduplicate(want, 12_000, group_rep))


def test_match_most_similar_on_the_exact_list():
    master = make_names(6000, seed=94)
    dupes = make_names(2000, seed=95) + master[:800]
    sg, want, _ = _fit_exact(master, dupes, min_similarity=0.7)
    assert sg._matches_device is not None
    dev = sg._get_nearest_matches()
    sg._matches_device = None               # same exact list, host rule (highest score, lowest master index)
    host = sg._get_nearest_matches()
    pd.testing.assert_frame_equal(dev, host)


def test_compute_pairwise_similarities_bit_equal_to_scipy():
    """the reference's dot(): master.multiply(dup).sum(axis=1), rows with 0 to 3 000 common trigrams"""
    import string_grouper_b200 as api
    from oracle import pipeline as P
    left, right = common_count_pairs(seed=3)
    for dtype in (np.float64, np.float32):
        got = api.compute_pairwise_similarities(pd.Series(left), pd.Series(right), tfidf_matrix_dtype=dtype)
        M, D, _ = P.tf_idf_matrices(left, right, dtype=dtype)
        want = np.asarray(M.multiply(D).sum(axis=1)).squeeze(axis=1)
        assert got.to_numpy().dtype == want.dtype == dtype
        bad = np.flatnonzero(got.to_numpy() != want)
        assert len(bad) == 0, "%s: %d of %d rows differ (first %s)" % (dtype.__name__, len(bad), len(want), bad[:5])
        assert len(COMMON_COUNTS) < len(want)


# ---------------------------------------------------------------------------------------------------------------
# 663k
# ---------------------------------------------------------------------------------------------------------------

def test_k1_663k_is_sklearn():
    """K1's matrix of the benchmark corpus (make_names(663_000, seed=0)) is scikit-learn's, bit for bit."""
    names = make_names(663_000, seed=0)
    t0 = time.perf_counter()
    _assert_k1_is_sklearn(names)
    print("663k: K1 + scikit-learn fit / transform + comparison %.1f s" % (time.perf_counter() - t0))

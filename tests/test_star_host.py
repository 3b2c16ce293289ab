"""not-gpu: linkage='star' of group_similar_strings on the host path (the numpy rounds of
string_grouper.star_representatives behind StringGrouper._host_star_reps), through the scikit-learn stand-in of
tests/cpu_backend.py, against the serial statement of tests/exact_star.py."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

import exact_star as X
from cpu_backend import oracle_device
from string_grouper_b200 import StringGrouper, _device, group_similar_strings
from string_grouper_b200.string_grouper import star_representatives
from synth_corpus import make_names


@pytest.fixture
def oracle():
    with oracle_device():
        yield


@pytest.fixture
def keyed_oracle(monkeypatch):
    from test_blocks_host import _keyed_cossim_topn
    with oracle_device():
        monkeypatch.setattr(_device, "cossim_topn", _keyed_cossim_topn)
        monkeypatch.setattr(_device, "block_id_tensors", lambda ids, n_left, same: (ids, ids))
        yield


def _assert_same(a, b):
    (pd.testing.assert_frame_equal if isinstance(a, pd.DataFrame) else pd.testing.assert_series_equal)(a, b)


def _components(n, pairs):
    graph = csr_matrix((np.ones(len(pairs)), (pairs.master_side, pairs.dupe_side)), shape=(n, n))
    return connected_components(graph, directed=True, connection="weak")[1]


def _check_guarantees(sg, rep):
    """every string is its own representative or listed with it; every star group inside one component"""
    n = len(sg._master)
    pairs = sg._matches_list
    listed = set(zip(pairs.master_side.tolist(), pairs.dupe_side.tolist()))
    for i in np.nonzero(rep != np.arange(n))[0].tolist():
        assert (i, int(rep[i])) in listed or (int(rep[i]), i) in listed
    comp = _components(n, pairs)
    assert np.array_equal(comp[rep], comp)


@pytest.mark.parametrize("min_similarity", [0.8, 0.6])
@pytest.mark.parametrize("group_rep", ["centroid", "first"])
@pytest.mark.parametrize("force_symmetries", [True, False])
def test_host_rule_equals_serial_spec(oracle, min_similarity, group_rep, force_symmetries):
    names = make_names(3000, seed=5) + [n.upper() + " inc" for n in make_names(300, seed=5)]
    sg = StringGrouper(pd.Series(names), min_similarity=min_similarity, group_rep=group_rep, linkage="star",
                       force_symmetries=force_symmetries).fit()
    rep = sg._representatives(len(names))
    assert np.array_equal(rep, X.star_of_grouper(sg))
    _check_guarantees(sg, rep)
    frame = sg.get_groups()
    assert np.array_equal(frame["group_rep_index"].to_numpy(), rep)
    assert (frame["group_rep"].to_numpy() == np.asarray(names, dtype=object)[rep]).all()
    single = sg._host_group_reps(len(names), group_rep == "centroid")
    assert (rep != np.arange(len(names))).sum() > 100
    if min_similarity == 0.6:        # chains exist at 0.6: star splits some components
        assert len(np.unique(rep)) > len(np.unique(single))


def test_rounds_equal_serial_rule_on_adversarial_inputs():
    """the numpy rounds against the serial rule: a path whose ranks increase along it (one round per string) in
    both directions, a star (two rounds), random graphs with weights that tie"""
    rng = np.random.default_rng(3)
    n = 300
    path = (np.arange(n - 1), np.arange(1, n))
    for w in (None, np.arange(n, dtype=np.float64)):
        rep, rounds = star_representatives(n, *path, weight=w)
        assert np.array_equal(rep, X.serial_star(n, *path, weight=w)) and rounds == n
    star = (np.full(n - 1, 7), np.delete(np.arange(n), 7))
    w = np.ones(n)
    w[7] = 2.0
    rep, rounds = star_representatives(n, *star, weight=w)
    assert rep.tolist() == [7] * n and rounds == 2
    for trial in range(20):
        m = int(rng.integers(0, 4 * n))
        r, c = rng.integers(0, n, m), rng.integers(0, n, m)
        w = rng.integers(0, 4, n).astype(np.float64) if trial % 2 else None
        assert np.array_equal(star_representatives(n, r, c, w)[0], X.serial_star(n, r, c, w))


def test_three_string_chain():
    """A ~ B and B ~ C above the threshold, A and C unmatched: one group under 'single', two under 'star'"""
    with oracle_device():
        names = pd.Series(["abcdefghij", "abcdefghijklmn", "efghijklmn"])
        sg = StringGrouper(names, min_similarity=0.7, group_rep="first").fit()
        pairs = sg._matches_list
        score = {(a, b): s for a, b, s in zip(pairs.master_side, pairs.dupe_side, pairs.similarity)}
        assert score[(0, 1)] > 0.7 and score[(1, 2)] > 0.7 and (0, 2) not in score and (2, 0) not in score
        single = group_similar_strings(names, min_similarity=0.7, group_rep="first")
        star = group_similar_strings(names, min_similarity=0.7, group_rep="first", linkage="star")
        centroid = group_similar_strings(names, min_similarity=0.7, linkage="star")
    assert single["group_rep_index"].tolist() == [0, 0, 0]
    assert star["group_rep_index"].tolist() == [0, 0, 2]
    assert star["group_rep"].tolist() == ["abcdefghij", "abcdefghij", "efghijklmn"]
    assert centroid["group_rep_index"].tolist() == [1, 1, 1]       # the middle has the largest similarity sum


@pytest.mark.parametrize("group_rep", ["centroid", "first"])
@pytest.mark.parametrize("kw", [{}, {"ignore_index": True}])
def test_cliques_give_the_single_linkage_frame(oracle, group_rep, kw):
    ids = pd.Series(["A0", "A1", "A2"], name="id")
    _assert_same(group_similar_strings(pd.Series(["foooo", "foooob", "bar"]), linkage="star", **kw),
                 group_similar_strings(pd.Series(["foooo", "foooob", "bar"]), **kw))
    _assert_same(
        group_similar_strings(pd.Series(["foooo", "foooob", "bar"]), ids, linkage="star", group_rep=group_rep, **kw),
        group_similar_strings(pd.Series(["foooo", "foooob", "bar"]), ids, group_rep=group_rep, **kw))
    exact = pd.Series(["acme corp", "zeta ltd", "acme corp", "qux gmbh", "zeta ltd", "acme corp", "lone name"],
                      index=[10, 11, 12, 13, 14, 15, 16], name="company")
    _assert_same(group_similar_strings(exact, linkage="star", group_rep=group_rep, **kw),
                 group_similar_strings(exact, group_rep=group_rep, **kw))


def test_edited_lists(oracle):
    names = pd.Series(make_names(400, seed=9) + ["abcdefghij", "abcdefghijklmn", "efghijklmn"])
    sg = StringGrouper(names, min_similarity=0.7, linkage="star").fit()
    sg.add_match("abcdefghij", "efghijklmn")
    rep = sg._representatives(len(names))
    assert np.array_equal(rep, X.star_of_grouper(sg))
    assert rep[400] == rep[401] == rep[402]          # a triangle now: one star group
    sg.remove_match("abcdefghij", "abcdefghijklmn")
    rep = sg._representatives(len(names))
    assert np.array_equal(rep, X.star_of_grouper(sg))
    _check_guarantees(sg, rep)
    assert np.array_equal(sg.get_groups()["group_rep_index"].to_numpy(), rep)


def test_no_pairs_and_tiny_inputs(oracle):
    assert star_representatives(0, [], [])[0].shape == (0,)
    assert star_representatives(4, [], [])[0].tolist() == [0, 1, 2, 3]
    assert star_representatives(3, [2, 1], [2, 1], np.zeros(3))[0].tolist() == [0, 1, 2]    # the diagonal only
    one = group_similar_strings(pd.Series(["abc"]), linkage="star")
    assert one["group_rep"].tolist() == ["abc"] and one["group_rep_index"].tolist() == [0]
    sg = StringGrouper(pd.Series(["abc def", "xyz uvw"]), linkage="star").fit()
    sg.remove_match("abc def", "abc def").remove_match("xyz uvw", "xyz uvw")
    assert len(sg._matches_list) == 0
    assert sg.get_groups()["group_rep_index"].tolist() == [0, 1]
    with pytest.raises(ValueError):          # no strings: the vectoriser's error, as with linkage='single'
        group_similar_strings(pd.Series([], dtype=object), linkage="star")


def test_linkage_validation(oracle):
    names = pd.Series(["foooo", "foooob", "bar"])
    for bad in ("complete", "Star", "", None, 1):
        with pytest.raises(Exception, match=r"(?s)Invalid option value for linkage.*\('single', 'star'\)"):
            StringGrouper(names, linkage=bad)
        with pytest.raises(Exception, match="Invalid option value for linkage"):
            group_similar_strings(names, linkage=bad)
        with pytest.raises(Exception, match="Invalid option value for linkage"):
            StringGrouper(names).update_options(linkage=bad)
    assert StringGrouper(names)._config.linkage == "single"


def test_duplicates_ignore_linkage(oracle):
    master = pd.Series(["foooo", "bar", "baz"])
    dupes = pd.Series(["foooo", "bar", "baz", "foooob"])
    _assert_same(StringGrouper(master, dupes, linkage="star").fit().get_groups(),
                 StringGrouper(master, dupes).fit().get_groups())


def test_keys(keyed_oracle):
    names = make_names(600, seed=4)
    keys = pd.Series(np.arange(600) % 3)
    sg = StringGrouper(pd.Series(names), master_keys=keys, min_similarity=0.6, linkage="star").fit()
    rep = sg._representatives(600)
    assert np.array_equal(rep, X.star_of_grouper(sg))
    assert np.array_equal(keys.to_numpy()[rep], keys.to_numpy())
    assert np.array_equal(group_similar_strings(pd.Series(names), keys=keys, min_similarity=0.6,
                                                linkage="star")["group_rep_index"].to_numpy(), rep)

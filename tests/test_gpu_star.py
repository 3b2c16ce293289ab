"""-m gpu: star groups on the device (csrc/sg_star.cu, _device.group_star) against the serial statement of
tests/exact_star.py, compared exactly (representatives are integers): match lists of real fits (plain, keyed,
records, corpus), lists in other orders, asymmetric lists, empty lists, and a path graph of 20 000 strings whose
ranks increase along it (20 000 rounds)."""
import time

import numpy as np
import pandas as pd
import pytest
import torch

import exact_star as X
from string_grouper_b200 import (StringGrouper, StringGrouperCorpus, _device, group_similar_records,
                                 group_similar_strings)
from string_grouper_b200.records import _RecordsGrouper
from synth_corpus import make_names
from synth_records import make_records

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def names():
    base = make_names(30_000, seed=61)
    return pd.Series(base[:29_000] + [s.upper() + " ltd" for s in base[:1_000]], name="name")


def _device_list(n, row, col, score):
    dev = torch.device("cuda")
    t = lambda a, dt: torch.as_tensor(np.asarray(a), dtype=dt, device=dev)     # noqa: E731
    return _device.DeviceMatches((n, n), t(row, torch.int32), t(col, torch.int32), t(score, torch.float64), len(row),
                                 0)


def _assert_direct(sg, rep):
    """every string is its own representative or one of its pairs in get_matches() holds the representative"""
    m = sg.get_matches()
    pairs = set(zip(m.left_index.tolist(), m.right_index.tolist()))
    idx = sg._master.index.to_numpy()
    for i in np.nonzero(rep != np.arange(len(rep)))[0].tolist():
        assert (idx[i], idx[rep[i]]) in pairs or (idx[rep[i]], idx[i]) in pairs


@pytest.mark.parametrize("min_similarity", [0.8, 0.6])
@pytest.mark.parametrize("group_rep", ["centroid", "first"])
def test_device_equals_serial_spec(names, min_similarity, group_rep):
    sg = StringGrouper(names, min_similarity=min_similarity, group_rep=group_rep, linkage="star").fit()
    assert sg._matches_device is not None
    n = len(names)
    before = _device.LAUNCH_COUNTS["groups"]
    rep = _device.group_star(sg._matches_device, n, group_rep == "centroid")
    assert _device.LAUNCH_COUNTS["groups"] > before
    want = X.star_of_grouper(sg)
    assert np.array_equal(rep, want)
    assert (rep != np.arange(n)).sum() > 1000
    single = _device.group_reps(sg._matches_device, n, group_rep == "centroid")
    if min_similarity == 0.6:
        assert len(np.unique(rep)) > len(np.unique(single))
    _assert_direct(sg, rep)
    # device path (with the device string gather) and host path give one frame
    dev = sg.get_groups()
    assert np.array_equal(dev["group_rep_index"].to_numpy(), rep)
    sg._matches_device = None
    pd.testing.assert_frame_equal(dev, sg.get_groups())


def test_list_order_asymmetric_and_empty_lists(names):
    sg = StringGrouper(names, min_similarity=0.6, group_rep="first", linkage="star").fit()
    r, c, s = sg._matches_device.host_triples()
    n = len(names)
    want = X.serial_star(n, r, c)
    perm = np.random.default_rng(0).permutation(len(r))       # 'first' needs no row order
    assert np.array_equal(_device.group_star(_device_list(n, r[perm], c[perm], s[perm]), n, False), want)
    # one direction of every pair only (rows still ascending): the same graph, the same groups
    upper = r < c
    for centroid in (False, True):
        got = _device.group_star(_device_list(n, r[upper], c[upper], s[upper]), n, centroid)
        assert np.array_equal(got, X.star_of_pairs(n, r[upper], c[upper], s[upper], centroid))
    assert np.array_equal(_device.group_star(_device_list(n, r[upper], c[upper], s[upper]), n, False), want)
    # force_symmetries=False: the list as the product left it (rows by score), asymmetric at the top-n cut
    for group_rep in ("centroid", "first"):
        sg = StringGrouper(names, min_similarity=0.6, max_n_matches=3, group_rep=group_rep, linkage="star",
                           force_symmetries=False).fit()
        rep = _device.group_star(sg._matches_device, n, group_rep == "centroid")
        assert np.array_equal(rep, X.star_of_grouper(sg))
        dev = sg.get_groups()
        sg._matches_device = None
        pd.testing.assert_frame_equal(dev, sg.get_groups())
    empty = _device_list(0, [], [], [])
    assert _device.group_star(empty, 0, True).shape == (0,)
    for centroid in (False, True):
        assert np.array_equal(_device.group_star(_device_list(7, [], [], []), 7, centroid), np.arange(7))


@pytest.mark.parametrize("centroid", [False, True])
def test_path_of_increasing_ranks(centroid):
    """one stored pair per string, i -> i + 1; ranks increase along the path ('first': by index; 'centroid': row sums
    that fall along it), so every round decides one string"""
    n = 20_000
    row, col = np.arange(n - 1), np.arange(1, n)
    score = 1.0 - 1e-5 * np.arange(n - 1)
    M = _device_list(n, row, col, score)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rep = _device.group_star(M, n, centroid)
    ms = 1e3 * (time.perf_counter() - t0)
    want = np.arange(n) - np.arange(n) % 2
    assert np.array_equal(rep, want)
    assert np.array_equal(rep, X.star_of_pairs(n, row, col, score, centroid))
    print("path of %d strings, centroid=%s: %.1f ms" % (n, centroid, ms))


def test_keyed_records_and_corpus(names):
    keys = pd.Series(np.arange(len(names)) % 4)
    sg = StringGrouper(names, master_keys=keys, min_similarity=0.6, linkage="star").fit()
    rep = sg._representatives(len(names))
    assert np.array_equal(rep, X.star_of_grouper(sg))
    assert np.array_equal(keys.to_numpy()[rep], keys.to_numpy())
    out = group_similar_strings(names, keys=keys, min_similarity=0.6, linkage="star")
    assert np.array_equal(out["group_rep_index"].to_numpy(), rep)

    df = make_records(20_000, seed=5)
    weights = {"name": 0.6, "address": 0.4}
    for group_rep in ("centroid", "first"):
        rg = _RecordsGrouper(df, None, weights, min_similarity=0.7, group_rep=group_rep, linkage="star").fit()
        assert rg._matches_device is not None
        rep = rg._representatives(len(df))
        assert np.array_equal(rep, X.star_of_grouper(rg))
        frame = group_similar_records(df, weights=weights, min_similarity=0.7, group_rep=group_rep, linkage="star")
        assert (frame["group_rep_name"].to_numpy() == df["name"].to_numpy()[rep]).all()
        rg._matches_device = None
        pd.testing.assert_frame_equal(frame, rg.get_groups())

    corpus = StringGrouperCorpus(names, min_similarity=0.6)
    batch = pd.Series(make_names(8_000, seed=62) + names.tolist()[:2_000])
    cg = corpus.fit(batch, linkage="star")
    assert cg._matches_device is not None
    rep = cg._representatives(len(batch))
    assert np.array_equal(rep, X.star_of_grouper(cg))
    assert np.array_equal(corpus.group_similar_strings(batch, linkage="star")["group_rep_index"].to_numpy(), rep)

"""not-gpu: the host side of blocking keys: key factorisation, argument checks, the blocked order and position
ranges (torch on the CPU against a numpy restatement), and the result frames through the oracle-backed stand-in of
tests/cpu_backend.py with a keyed product that follows the specification of tests/test_gpu_blocks.py."""
import os

import numpy as np
import pandas as pd
import pytest
import torch
from scipy.sparse import csr_matrix

from cpu_backend import FakeMatches, oracle_device
from exact_topn import RankedPairs, exact_pairs
from string_grouper_b200 import StringGrouper, _device, group_similar_strings, match_most_similar, match_strings
from string_grouper_b200.string_grouper import block_ids_of

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_factorisation_joint_and_missing():
    m, d = pd.Series(["a", "b", "c", "d", "e"]), pd.Series(["x", "y", "z"])
    ids = block_ids_of(m, d, pd.Series(["US", None, "FR", np.nan, "US"]), pd.Series([pd.NA, "FR", "US"]))
    assert ids.dtype == np.int32 and len(ids) == 8
    assert ids[0] == ids[4] == ids[7] and ids[2] == ids[6] and ids[0] != ids[2]
    missing = ids[[1, 3, 5]]
    assert len(set(missing)) == 3 and not set(missing) & set(ids[[0, 2, 4, 6, 7]])


def test_factorisation_mixed_dtypes():
    m = pd.Series(["a", "b", "c", "d", "e"])
    ids = block_ids_of(m, None, pd.Series([1, "1", 2, ("t", 1), ("t", 1)], dtype=object))
    assert ids[0] != ids[1] and ids[3] == ids[4] and len(set(ids[:4])) == 4
    ids = block_ids_of(m[:3], m[3:], pd.Series([1, 2, 3]), pd.Series(["1", "2"]))     # int64 against str
    assert len(set(ids)) == 5
    ids = block_ids_of(m[:3], m[3:], pd.Series([1.5, np.nan, 2.0]), pd.Series([2.0, np.nan]))
    assert ids[2] == ids[3] and ids[1] != ids[4]


def test_no_keys_no_block_ids():
    assert block_ids_of(pd.Series(["a"]), None, None, None) is None
    assert block_ids_of(pd.Series(["a"]), pd.Series(["b"]), None, None) is None
    assert StringGrouper(pd.Series(["a", "b"]))._block_ids is None


def test_argument_checks():
    m, d = pd.Series(["a", "b", "c"]), pd.Series(["x", "y"])
    with pytest.raises(ValueError):
        StringGrouper(m, master_keys=pd.Series([1, 2]))
    with pytest.raises(ValueError):
        StringGrouper(m, duplicates_keys=pd.Series([1, 2, 3]))
    with pytest.raises(ValueError):
        StringGrouper(m, d, master_keys=pd.Series([1, 2, 3]))
    with pytest.raises(ValueError):
        StringGrouper(m, d, duplicates_keys=pd.Series([1, 2]))
    with pytest.raises(ValueError):
        StringGrouper(m, d, master_keys=pd.Series([1, 2, 3]), duplicates_keys=pd.Series([1]))
    with pytest.raises(TypeError):
        StringGrouper(m, master_keys=[1, 2, 3])
    sg = StringGrouper(m, master_keys=pd.Series([1, 2, 3]))
    with pytest.raises(ValueError):
        sg.reset_data(m, master_keys=pd.Series([1]))
    sg.reset_data(m)
    assert sg._block_ids is None
    with pytest.raises(TypeError):           # keys are keyword-only
        match_strings(m, None, None, None, pd.Series([1, 2, 3]))


def test_keys_aligned_by_position():
    m = pd.Series(["a", "b", "c"], index=[10, 11, 12])
    ids = block_ids_of(m, None, pd.Series(["p", "q", "p"], index=[2, 1, 0]))
    assert ids[0] == ids[2] != ids[1]


@pytest.mark.parametrize("seed", range(4))
def test_blocked_order_and_ranges(seed):
    rng = np.random.default_rng(seed)
    n_right, n_left = int(rng.integers(1, 400)), int(rng.integers(1, 400))
    ids_b = rng.integers(0, 1 + n_right // 7, size=n_right).astype(np.int32)
    ids_a = rng.integers(0, 2 + n_right // 7, size=n_left).astype(np.int32)
    perm = rng.permutation(n_right).astype(np.int32)
    got = _device.blocked_order(torch.from_numpy(perm), torch.from_numpy(ids_b)).numpy()
    want = perm[np.argsort(ids_b[perm], kind="stable")]
    assert np.array_equal(got, want)
    sorted_ids = ids_b[want]
    lo, hi = (x.numpy() for x in _device.block_ranges(torch.from_numpy(sorted_ids), torch.from_numpy(ids_a)))
    assert lo.dtype == hi.dtype == np.int32
    for r in range(n_left):
        at = np.flatnonzero(sorted_ids == ids_a[r])
        if len(at):
            assert (lo[r], hi[r]) == (at[0], at[-1] + 1)
        else:
            assert lo[r] == hi[r]
    # in the blocked order of the left rows both ends grow: the work items of each column-tile group are one range
    order = np.argsort(ids_a, kind="stable")
    assert np.all(np.diff(lo[order]) >= 0) and np.all(np.diff(hi[order]) >= 0)


def _keyed_cossim_topn(A, B, top_n, threshold, row_begin=0, row_end=None, block_ids=None, stats=None, **kw):
    """stand-in for the keyed product: the exact pairs of equal ids, cut by the top-n rule (row kernel spec)"""
    from cpu_backend import cossim_topn
    if block_ids is None:
        return cossim_topn(A, B, top_n, threshold, row_begin, row_end, **kw)
    ids_a, ids_b = block_ids
    r, c, s = exact_pairs(A.m, B.m, threshold)
    keep = ids_a[r] == ids_b[c]
    row, col, score, max_row = RankedPairs(r[keep], c[keep], s[keep]).topn(min(top_n, B.shape[0]), threshold)
    indptr = np.zeros(A.shape[0] + 1, np.int64)
    np.cumsum(np.bincount(row, minlength=A.shape[0]), out=indptr[1:])
    if stats is not None:
        stats["blocks"] = True
    return FakeMatches(csr_matrix((score, col, indptr), shape=(A.shape[0], B.shape[0])), max_row=max_row)


@pytest.fixture
def keyed_oracle(monkeypatch):
    with oracle_device():
        monkeypatch.setattr(_device, "cossim_topn", _keyed_cossim_topn)
        monkeypatch.setattr(_device, "block_id_tensors",
                            lambda ids, n_left, same: (ids, ids) if same else (ids[:n_left], ids[n_left:]))
        yield


def _accounts():
    acc = pd.read_csv(os.path.join(GOLDEN, "accounts_input.csv"))
    keys = pd.Series(np.where(np.arange(len(acc)) % 3 == 0, "A", "B"))
    return acc["name"], keys


def test_accounts_one_key_identity(keyed_oracle):
    names, _ = _accounts()
    one = pd.Series(["x"] * len(names))
    for thr in (0.1, 0.5, 0.8):
        k = StringGrouper(names, master_keys=one, min_similarity=thr).fit()
        u = StringGrouper(names, min_similarity=thr).fit()
        pd.testing.assert_frame_equal(k._matches_list, u._matches_list)
        assert k._true_max_n_matches == u._true_max_n_matches
        pd.testing.assert_frame_equal(k.get_matches(), u.get_matches())
        pd.testing.assert_frame_equal(k.get_groups(), u.get_groups())
    pd.testing.assert_frame_equal(group_similar_strings(names, keys=one, min_similarity=0.5),
                                  group_similar_strings(names, min_similarity=0.5))


def test_accounts_filtered_identity(keyed_oracle):
    names, keys = _accounts()
    k = keys.to_numpy()
    for thr in (0.1, 0.5, 0.8):
        got = match_strings(names, master_keys=keys, min_similarity=thr, max_n_matches=len(names))
        full = match_strings(names, min_similarity=thr, max_n_matches=len(names))
        same = k[full["left_index"].to_numpy()] == k[full["right_index"].to_numpy()]
        pd.testing.assert_frame_equal(got, full[same].reset_index(drop=True))
    master, dupes = names[:9], names[9:].reset_index(drop=True)
    mk, dk = keys[:9], keys[9:].reset_index(drop=True)
    got = match_strings(master, dupes, master_keys=mk, duplicates_keys=dk, min_similarity=0.3, max_n_matches=9)
    full = match_strings(master, dupes, min_similarity=0.3, max_n_matches=9)
    same = mk.to_numpy()[full["left_index"].to_numpy()] == dk.to_numpy()[full["right_index"].to_numpy()]
    pd.testing.assert_frame_equal(got, full[same].reset_index(drop=True))
    groups = group_similar_strings(names, keys=keys, min_similarity=0.1)
    assert np.array_equal(k[groups["group_rep_index"].to_numpy()], k)
    best = match_most_similar(master, dupes, master_keys=mk, duplicates_keys=dk, min_similarity=0.3)
    assert len(best) == len(dupes)

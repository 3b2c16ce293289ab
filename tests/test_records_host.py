"""not-gpu: the host side of match_records / group_similar_records — argument checks, missing values, the result
frames — through the scikit-learn stand-in of tests/cpu_backend.py, with a numpy stand-in for the weighted stacking
and the per-field pair scores (the specification of tests/exact_records.py)."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import csr_matrix

import exact_records as X
from cpu_backend import FakeCSR, oracle_device
from string_grouper_b200 import _device, group_similar_records, group_similar_strings, match_records, match_strings
from synth_records import make_records


def _stack_fields(parts, scales):
    return FakeCSR(X.stack([p.m for p in parts], scales))


def _pair_scores(A, B, M):
    r, c, _ = M.host_triples()
    return X.pair_scores(A.m, B.m, r, c) if len(r) else np.zeros(0)


@pytest.fixture
def records_oracle(monkeypatch):
    with oracle_device():
        monkeypatch.setattr(_device, "stack_fields", _stack_fields)
        monkeypatch.setattr(_device, "pair_scores", _pair_scores)
        monkeypatch.setattr(_device, "mark", lambda stats, name: None)
        yield


W2 = {"name": 0.6, "address": 0.4}


def _df(n=300, seed=0):
    return make_records(n, seed=seed)


def test_argument_checks(records_oracle):
    df = _df(40)
    with pytest.raises(TypeError):
        match_records(df["name"], weights={"name": 1.0})
    with pytest.raises(TypeError):
        match_records(df, df["name"], weights={"name": 1.0})
    for bad in ({}, {"nope": 1.0}, {"name": 0.0}, {"name": -1.0}, {"name": float("nan")}, {"name": float("inf")},
                {"name": "1"}, {"name": True}, [("name", 1.0)]):
        with pytest.raises(ValueError):
            match_records(df, weights=bad)
    with pytest.raises(ValueError):          # a column missing from the duplicates only
        match_records(df, df[["name"]], weights=W2)
    with pytest.raises(ValueError, match="address"):
        match_records(df.assign(address=["..."] * len(df)), weights=W2)
    with pytest.raises(TypeError, match="Master input does not consist"):
        match_records(df.assign(address=[1] * len(df)), weights=W2)
    with pytest.raises(TypeError, match="Duplicates input does not consist"):
        match_records(df, df.assign(name=[1.5] * len(df)), weights=W2)
    with pytest.raises(ValueError):          # left_index would collide
        match_records(df.rename(columns={"name": "index"}), weights={"index": 1.0})
    with pytest.raises(ValueError):          # left_id would collide
        match_records(df.rename(columns={"name": "id"}), weights={"id": 1.0},
                      master_id=pd.Series(np.arange(len(df))))
    with pytest.raises(TypeError):           # unknown option
        match_records(df, weights=W2, no_such_option=1)


def test_missing_values_read_as_empty(records_oracle):
    df = pd.DataFrame({"name": ["ACME INC", "ACME INC.", "BETA LLC", "ACME INC"],
                       "address": ["1 MAIN ST, X", None, np.nan, pd.NA]}, dtype=object)
    got = match_records(df, weights=W2, min_similarity=0.1)
    same = match_records(df.assign(address=["1 MAIN ST, X", "", "", ""]), weights=W2, min_similarity=0.1)
    cols = [c for c in got.columns if not c.endswith("address")]
    pd.testing.assert_frame_equal(got[cols], same[cols])
    assert pd.isna(got["left_address"].iloc[-1])      # the frame shows the records' own values
    assert (got.loc[got.left_index != got.right_index, "similarity_address"] == 0).all()
    s = pd.Series(["1 MAIN ST, X", None, None, None], dtype="str")
    got = match_records(df.assign(address=s), weights=W2, min_similarity=0.1)
    pd.testing.assert_frame_equal(got[cols], same[cols])


def _spec_frame(df, dup, weights, **kw):
    ml, _, _ = X.exact_record_list(df, dup, weights=weights, **kw)
    return ml


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_self_match_layout_and_scores(records_oracle, dtype):
    df = _df(300)
    got = match_records(df, weights=W2, min_similarity=0.5, tfidf_matrix_dtype=dtype)
    assert list(got.columns) == ["left_index", "left_name", "left_address", "similarity", "similarity_name",
                                 "similarity_address", "right_name", "right_address", "right_index"]
    want = _spec_frame(df, None, W2, min_similarity=0.5, dtype=dtype)
    assert np.array_equal(got.left_index, want.master_side) and np.array_equal(got.right_index, want.dupe_side)
    for c in ("similarity", "similarity_name", "similarity_address"):
        assert np.array_equal(got[c].to_numpy(), want[c].to_numpy()), c
    assert got.left_name.tolist() == df.name.to_numpy()[want.master_side].tolist()
    diag = got.left_index == got.right_index
    assert (got.similarity[diag] == 1).all() and diag.sum() == len(df)


def test_two_frames_ids_multiindex_ignore_index(records_oracle):
    df = _df(200)
    m, d = df[:120], df[120:]
    m = m.set_index(pd.MultiIndex.from_arrays([np.arange(120) % 7, np.arange(120)], names=["a", "b"]))
    got = match_records(m, d, weights=W2, min_similarity=0.3, master_id=pd.Series(np.arange(120), name="mid"),
                        duplicates_id=pd.Series(np.arange(80) + 1000, name="did"))
    assert list(got.columns) == ["left_a", "left_b", "left_name", "left_address", "left_mid", "similarity",
                                 "similarity_name", "similarity_address", "right_did", "right_name", "right_address",
                                 "right_index"]
    want = _spec_frame(m, d, W2, min_similarity=0.3)
    assert np.array_equal(got.left_b, want.master_side) and np.array_equal(got.right_index, want.dupe_side + 120)
    assert np.array_equal(got.right_did, want.dupe_side + 1000)
    for c in ("similarity", "similarity_name", "similarity_address"):
        assert np.array_equal(got[c].to_numpy(), want[c].to_numpy()), c
    got = match_records(m, d, weights=W2, min_similarity=0.3, ignore_index=True)
    assert list(got.columns) == ["left_name", "left_address", "similarity", "similarity_name", "similarity_address",
                                 "right_name", "right_address"]


def test_include_zeroes(records_oracle):
    df = _df(30)
    got = match_records(df, weights=W2, min_similarity=0, max_n_matches=30)
    assert len(got) == 30 * 30
    zero = got.similarity == 0
    assert zero.any() and (got.loc[zero, ["similarity_name", "similarity_address"]] == 0).all().all()
    got = match_records(df, weights=W2, min_similarity=0, max_n_matches=30, include_zeroes=False)
    assert (got.similarity > 0).all()


def test_one_field_equals_match_strings(records_oracle):
    df = _df(400, seed=3)
    for kw in ({}, {"min_similarity": 0.3, "max_n_matches": 5}, {"tfidf_matrix_dtype": np.float32}):
        got = match_records(df[["name"]], weights={"name": 3.0}, **kw)
        pd.testing.assert_frame_equal(got.drop(columns="similarity_name"), match_strings(df["name"], **kw))
        off = got.left_index != got.right_index          # the diagonal's similarity is set to 1
        assert np.array_equal(got.similarity_name[off], got.similarity[off])
        pd.testing.assert_frame_equal(group_similar_records(df[["name"]], weights={"name": 3.0}, **kw),
                                      group_similar_strings(df["name"], **kw))


@pytest.mark.parametrize("rep", ["centroid", "first"])
def test_group_similar_records_frame(records_oracle, rep):
    df = _df(300, seed=5)
    ids = pd.Series(np.arange(300) + 7, name="rid")
    got = group_similar_records(df, weights=W2, string_ids=ids, group_rep=rep, min_similarity=0.5)
    assert list(got.columns) == ["group_rep_rid", "group_rep_index", "group_rep_name", "group_rep_address"]
    assert got.index.equals(df.index)
    ml = _spec_frame(df, None, W2, min_similarity=0.5)
    from oracle import pipeline as P
    rep_pos = P.deduplicate(ml, len(df), group_rep=rep)
    assert np.array_equal(got.group_rep_index.to_numpy(), rep_pos)
    assert np.array_equal(got.group_rep_rid.to_numpy(), rep_pos + 7)
    got = group_similar_records(df, weights=W2, ignore_index=True, min_similarity=0.5)
    assert list(got.columns) == ["group_rep_name", "group_rep_address"]


def test_keys_and_stats(records_oracle, monkeypatch):
    from test_blocks_host import _keyed_cossim_topn
    monkeypatch.setattr(_device, "cossim_topn", _keyed_cossim_topn)
    monkeypatch.setattr(_device, "block_id_tensors",
                        lambda ids, n_left, same: (ids, ids) if same else (ids[:n_left], ids[n_left:]))
    df = _df(200, seed=9)
    keys = pd.Series(np.where(np.arange(200) % 3 == 0, "A", None))
    got = match_records(df, weights=W2, master_keys=keys, min_similarity=0.2, max_n_matches=200)
    full = match_records(df, weights=W2, min_similarity=0.2, max_n_matches=200)
    k = keys.to_numpy()
    l, r = full.left_index.to_numpy(), full.right_index.to_numpy()
    same = (k[l] == k[r]) & (k[l] != None) | (l == r)     # noqa: E711  a missing key matches only itself
    pd.testing.assert_frame_equal(got, full[same].reset_index(drop=True))
    from string_grouper_b200.records import _RecordsGrouper
    sg = _RecordsGrouper(df, None, W2).fit()
    assert sg._last_stats["fields"] == 2

"""gpu: match_records / group_similar_records against the specification of tests/exact_records.py, bit for bit
(np.array_equal, as tests/test_gpu_k2_exact.py compares): the stacking kernel (csrc/sg_fields.cu), the one-field
identity with match_strings, two and three fields over thresholds set on the scores themselves, blocking keys, groups,
the other K1 paths, and sampled rows of large inputs on whichever K2 path runs."""
import numpy as np
import pandas as pd
import pytest
from scipy.sparse import random as sparse_random

import exact_records as X
from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn
from synth_records import make_records, perturb

pytestmark = pytest.mark.gpu

W2 = {"name": 0.6, "address": 0.4}
W3 = {"name": 5.0, "address": 2.0, "city": 1.0}
WTINY = {"name": 1.0, "address": 1e6}     # the name's postings fall into fp16's subnormal range


def _three(df):
    city = df["address"].str.split(", ").str[-1]
    return df.assign(city=city)


def _grouper(master, dup=None, weights=W2, **kw):
    from string_grouper_b200.records import _RecordsGrouper
    return _RecordsGrouper(master, dup, weights, **kw)


# ------------------------------------------------------------------ the stacking kernel

def _field(rng, n, dtype, empty_rows):
    m = sparse_random(n, int(rng.integers(5, 300)), density=float(rng.uniform(0.01, 0.2)), format="csr",
                      dtype=dtype, random_state=int(rng.integers(1 << 30)))
    m.data = np.abs(m.data) + dtype(1e-3)
    m = m.tolil()
    m[empty_rows] = 0
    m = m.tocsr()
    m.eliminate_zeros()
    m.sort_indices()
    return m


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_stack_kernel(dtype, k):
    from string_grouper_b200 import _device as D
    rng = np.random.default_rng(k)
    n = 1000 + 7 * k                                    # not a multiple of 32
    all_empty = rng.choice(n, 40, replace=False)        # rows empty in every field
    mats = [_field(rng, n, dtype, np.union1d(all_empty, rng.choice(n, 100, replace=False))) for _ in range(k)]
    for weights in (rng.uniform(0.5, 7.0, size=k), np.array([1.0] + [1e6] * (k - 1)), np.array([1e6] + [1.0] * (k - 1))):
        scale = D.field_scales(weights, dtype)
        assert np.array_equal(scale.astype(dtype), X.scales(dict(zip(range(k), weights)), dtype))
        got = D.stack_fields([D.DeviceCSR.from_scipy(m) for m in mats], scale)
        want = X.stack(mats, scale.astype(dtype))
        n_got = got.nnz
        assert got.shape == want.shape and n_got == want.nnz
        assert np.array_equal(got.d_indptr.cpu().numpy(), want.indptr)
        assert np.array_equal(got.d_indices[:n_got].cpu().numpy(), want.indices)
        val = got.d_val[:n_got].cpu().numpy()
        assert val.dtype == dtype and np.array_equal(val, want.data)
        assert np.array_equal(got.d_val32[:n_got].cpu().numpy(), want.data.astype(np.float32))
        if k > 1 and weights[0] == 1.0:
            small = want.data[want.indices < mats[0].shape[1]].astype(np.float16)
            assert (np.abs(small[small > 0]) < 6.2e-5).any()     # fp16-subnormal postings of the light field


def test_stack_kernel_row_range_views():
    """the duplicate rows of a K1 call are a view whose indptr starts inside the arrays"""
    from string_grouper_b200 import _device as D
    df = make_records(3000, seed=4)
    sg = _grouper(df[:2000], df[2000:])
    A, B = sg._get_tf_idf_matrices()
    fields = X.field_matrices(df[:2000], df[2000:], W2)
    sc = X.scales(W2, np.float64)
    for got, want in ((A, X.stack([m for m, _ in fields], sc)), (B, X.stack([d for _, d in fields], sc))):
        h = got.to_scipy()
        assert np.array_equal(h.indptr, want.indptr) and np.array_equal(h.indices, want.indices)
        assert np.array_equal(h.data, want.data)


# ------------------------------------------------------------------ one field

def test_one_field_equals_match_strings():
    from string_grouper_b200 import match_records, match_strings
    df = make_records(20_000, seed=1)
    for kw in ({}, {"min_similarity": 0.5, "max_n_matches": 7}, {"tfidf_matrix_dtype": np.float32}):
        got = match_records(df[["name"]], weights={"name": 3.0}, **kw)
        want = match_strings(df["name"], **kw)
        pd.testing.assert_frame_equal(got.drop(columns="similarity_name"), want)
        off = got.left_index != got.right_index
        assert np.array_equal(got.similarity_name[off].to_numpy(), got.similarity[off].to_numpy())


# ------------------------------------------------------------------ two and three fields against the specification

def _check(got, want, fields):
    assert np.array_equal(got.left_index.to_numpy(), want.master_side.to_numpy())
    assert np.array_equal(got.right_index.to_numpy(), want.dupe_side.to_numpy())
    for c in ["similarity"] + ["similarity_%s" % f for f in fields]:
        assert np.array_equal(got[c].to_numpy(), want[c].to_numpy()), c


def _thresholds(df, dup, weights, dtype):
    """one pair's exact combined score and the next double below it"""
    _, _, (_, M, D) = X.exact_record_list(df, dup, weights=weights, dtype=dtype, min_similarity=0.5)
    r, c, s = exact_pairs(M, D, 0.5)
    s = s[r != c] if dup is None else s
    t = float(np.sort(s)[len(s) // 2])
    return [t, float(np.nextafter(t, -np.inf))]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("weights", [W2, W3, WTINY], ids=["two", "three", "tiny"])
def test_self_match_against_spec(dtype, weights):
    from string_grouper_b200 import match_records
    df = _three(make_records(4000, seed=2))
    for thr in _thresholds(df, None, weights, dtype):
        for top in (1, 20, 33, 2048):
            sg = _grouper(df, None, weights, min_similarity=thr, max_n_matches=top, tfidf_matrix_dtype=dtype).fit()
            assert sg._last_stats["triangle"] and sg._last_stats["fields"] == len(weights)
            want, max_row, _ = X.exact_record_list(df, None, weights=weights, dtype=dtype, min_similarity=thr,
                                                   max_n_matches=top)
            _check(sg.get_matches(), want, weights)
            assert sg._true_max_n_matches == max_row
    got = match_records(df[:50], weights=weights, min_similarity=0, max_n_matches=50, tfidf_matrix_dtype=dtype)
    assert len(got) == 50 * 50
    zero = got.similarity == 0
    assert zero.any() and (got.loc[zero, ["similarity_%s" % f for f in weights]] == 0).all().all()
    nz = got[~zero].reset_index(drop=True)
    want, _, _ = X.exact_record_list(df[:50], None, weights=weights, dtype=dtype, min_similarity=0, max_n_matches=50)
    _check(nz, want, weights)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_two_frames_against_spec(dtype):
    df = _three(make_records(5000, seed=6))
    m, d = df[:3000], _three(perturb(df[3000:].reset_index(drop=True), seed=9)).set_index(np.arange(3000, 5000))
    for weights in (W2, W3):
        for thr in _thresholds(m, d, weights, dtype):
            for top in (1, 20, 33, 2048):
                sg = _grouper(m, d, weights, min_similarity=thr, max_n_matches=top, tfidf_matrix_dtype=dtype).fit()
                want, max_row, _ = X.exact_record_list(m, d, weights=weights, dtype=dtype, min_similarity=thr,
                                                       max_n_matches=top)
                got = sg.get_matches()
                got = got.assign(right_index=got.right_index - 3000)
                _check(got, want, weights)
                assert sg._true_max_n_matches == max_row


def test_keys_against_spec():
    from string_grouper_b200 import match_records
    df = make_records(6000, seed=11)
    m, d = df[:4000], df[4000:].reset_index(drop=True)
    rng = np.random.default_rng(3)
    mk = pd.Series(rng.choice(["A", "B", "C", None], size=4000))
    dk = pd.Series(rng.choice(["A", "B", "D", None], size=2000))
    for top in (1, 20):
        got = match_records(m, d, weights=W2, master_keys=mk, duplicates_keys=dk, min_similarity=0.4,
                            max_n_matches=top)
        _, _, (fields, M, D) = X.exact_record_list(m, d, weights=W2, min_similarity=0.4)
        r, c, s = exact_pairs(M, D, 0.4)
        a, b = mk.to_numpy(), dk.to_numpy()
        keep = (a[r] == b[c]) & pd.notna(a[r])
        row, col, score, _ = RankedPairs(r[keep], c[keep], s[keep]).topn(top, 0.4)
        assert np.array_equal(got.left_index, row) and np.array_equal(got.right_index, col)
        assert np.array_equal(got.similarity, score)
        for f, (A, B) in zip(W2, fields):
            assert np.array_equal(got["similarity_%s" % f], X.pair_scores(A, B, row, col))


@pytest.mark.parametrize("rep", ["centroid", "first"])
def test_groups_against_host_rule(rep):
    from oracle import pipeline as P
    from string_grouper_b200 import group_similar_records
    df = make_records(8000, seed=12)
    got = group_similar_records(df, weights=W2, group_rep=rep, min_similarity=0.6)
    want, _, _ = X.exact_record_list(df, None, weights=W2, min_similarity=0.6)
    assert np.array_equal(got.group_rep_index.to_numpy(), P.deduplicate(want, len(df), group_rep=rep))
    assert got.group_rep_name.tolist() == df.name.to_numpy()[got.group_rep_index.to_numpy()].tolist()


def test_other_k1_paths():
    df = make_records(3000, seed=13)
    accents = np.array(["É", "ö", "ñ", "ç", "ü"])
    rng = np.random.default_rng(0)
    name = [s[:3] + accents[rng.integers(5)] + s[3:] for s in df.name]
    dfa = df.assign(name=name)
    for d, kw in ((dfa, {"normalize_to_ascii": False}), (df, {"ngram_size": 4})):
        sg = _grouper(d, None, W2, min_similarity=0.5, **kw).fit()
        want, _, _ = X.exact_record_list(d, None, weights=W2, min_similarity=0.5, **kw)
        _check(sg.get_matches(), want, W2)


# ------------------------------------------------------------------ large inputs

def _sampled_exact(A_spec, got, n, top, thr, seed):
    rows = np.sort(np.random.default_rng(seed).choice(n, 2000, replace=False))
    r, c, s, _ = exact_topn(A_spec[rows], A_spec, top, thr, block_rows=128)
    gr, gc, gs = got.host_triples()
    sel = np.isin(gr, rows)
    assert_same((gr[sel], gc[sel], gs[sel]), (rows[r], c, s), "sampled rows")


def test_large_dedup_sampled():
    from string_grouper_b200 import _device as D
    base = make_records(100_000, seed=21)
    df = pd.concat([base, base[:40_000]], ignore_index=True)           # 140 000 records, 40 000 repeated
    A, _ = _grouper(df)._get_tf_idf_matrices()
    fields = X.field_matrices(df, None, W2)
    spec = X.stack([m for m, _ in fields], X.scales(W2, np.float64))
    h = A.to_scipy()
    assert np.array_equal(h.indptr, spec.indptr) and np.array_equal(h.indices, spec.indices)
    assert np.array_equal(h.data, spec.data)
    st = {}
    got = D.cossim_topn(A, A, 20, 0.8, stats=st)
    assert st["dedup"]
    _sampled_exact(spec, got, len(df), 20, 0.8, 8)


def test_large_low_threshold_sampled():
    from string_grouper_b200 import _device as D
    df = make_records(70_000, seed=22)
    A, _ = _grouper(df)._get_tf_idf_matrices()
    spec = A.to_scipy()
    st = {}
    got = D.cossim_topn(A, A, 20, 0.3, stats=st)
    print("path: floor %s, dedup %s, triangle %s" % (st.get("topn_floor"), st.get("dedup"), st.get("triangle")))
    _sampled_exact(spec, got, len(df), 20, 0.3, 9)

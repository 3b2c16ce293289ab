"""not-gpu: the dedup path of a self-match (DESIGN.md §4 "Identical rows") restated in numpy / scipy and compared with
the exact reference (tests/exact_topn.py) bit for bit.  The CUDA path is checked end to end by tests/test_gpu_dedup.py;
this file pins the ALGORITHM: group the bit-identical rows, take the top n of every distinct row over the columns
expanded to the members of each group, copy the list to every member.
"""
import numpy as np
import pytest
from scipy.sparse import csr_matrix

from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn, topn_from_pairs
from oracle import pipeline as P
from synth_corpus import make_names


def row_groups(m):
    """(uid, members): groups of bit-identical rows (indices and value bits), numbered by their first member"""
    first, uid = {}, np.empty(m.shape[0], np.int64)
    for r in range(m.shape[0]):
        lo, hi = m.indptr[r], m.indptr[r + 1]
        uid[r] = first.setdefault(m.indices[lo:hi].tobytes() + m.data[lo:hi].tobytes(), len(first))
    members = [np.flatnonzero(uid == u) for u in range(len(first))] if len(first) < 2000 else \
        np.split(np.argsort(uid, kind="stable"), np.cumsum(np.bincount(uid))[:-1])
    return uid, members


def dedup_topn(m, top_n, threshold):
    """the product over the distinct rows U, each kept (u, v, s) expanded to (u, c, s) for every member c of v,
    ranked per u, and every row given its group's list"""
    m = csr_matrix(m)
    uid, members = row_groups(m)
    reps = np.array([g[0] for g in members], dtype=np.int64)
    U = m[reps]
    u, v, s = exact_pairs(U, U, threshold)
    size = np.array([len(g) for g in members])
    cols = np.concatenate([members[x] for x in v]) if len(v) else np.zeros(0, np.int64)
    gr, gc, gs, _ = topn_from_pairs(np.repeat(u, size[v]), cols, np.repeat(s, size[v]), top_n)
    start = np.searchsorted(gr, np.arange(len(members) + 1))
    out = [(np.full(start[uid[r] + 1] - start[uid[r]], r), gc[start[uid[r]]:start[uid[r] + 1]],
            gs[start[uid[r]]:start[uid[r] + 1]]) for r in range(m.shape[0])]
    r, c, sc = (np.concatenate([o[k] for o in out]) for k in range(3))
    max_row = int(np.diff(start).max()) if len(gr) else 0
    return r.astype(np.int64), c.astype(np.int64), sc, max_row


def _dup_corpus(n, seed):
    rng = np.random.default_rng(seed)
    names = make_names(n, seed=seed)
    pick = rng.choice(n, n // 3, replace=True)
    names += [names[i].upper() if i % 2 else names[i] + "." for i in pick] + ["acme global holdings llc"] * 60
    return [names[i] for i in rng.permutation(len(names))]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_corpus_with_groups(dtype):
    m, _, _ = P.tf_idf_matrices(_dup_corpus(2500, 3), dtype=dtype)
    uid, members = row_groups(m)
    assert len(members) < 0.85 * m.shape[0] and max(len(g) for g in members) >= 60
    for thr in (0.5, 0.8, 0.95):
        for top_n in (1, 20, 32, 2048):
            assert_same(dedup_topn(m, top_n, thr), exact_topn(m, m, top_n, thr),
                        "%s thr=%r top_n=%d" % (np.dtype(dtype).name, thr, top_n))


def test_dyadic_ties_across_groups():
    """four features of weight 0.5 out of 10, so every score is a multiple of 1/4; groups of different sizes, members shuffled, tie exactly at the cut, so the
    cut and the ascending order of tied columns interleave the members of several groups"""
    rng = np.random.default_rng(11)
    base = [np.sort(rng.choice(10, 4, replace=False)) for _ in range(30)]
    rows = [base[i % 30] for i in range(30 * 7)] + [base[i] for i in rng.choice(30, 90)]
    rows = [rows[i] for i in rng.permutation(len(rows))]
    m = csr_matrix((np.full(4 * len(rows), 0.5), np.concatenate(rows), np.arange(0, 4 * len(rows) + 1, 4)),
                   shape=(len(rows), 10))
    uid, members = row_groups(m)
    assert len(members) >= 20 and len({len(g) for g in members}) > 3
    for thr in (0.25, float(np.nextafter(0.25, 0)), 0.5, float(np.nextafter(0.5, 0))):
        # the cut of top 20 falls inside a run of equal scores that spans groups
        t = RankedPairs(*exact_pairs(m, m, thr))
        at, past = (t.rank == 19), (t.rank == 20)
        cut = dict(zip(t.row[at], zip(t.col[at], t.score[at])))
        assert any(s == cut[r][1] and uid[c] != uid[cut[r][0]]
                   for r, c, s in zip(t.row[past], t.col[past], t.score[past]))
        for top_n in (1, 20, 32, 2048):
            assert_same(dedup_topn(m, top_n, thr), exact_topn(m, m, top_n, thr), "dyadic thr=%r top_n=%d" % (thr,
                                                                                                         top_n))


def test_empty_rows():
    m, _, _ = P.tf_idf_matrices(_dup_corpus(600, 5) + ["", "", "--", "  "])
    assert np.any(np.diff(m.indptr) == 0)
    for top_n in (1, 20, 32, 2048):
        assert_same(dedup_topn(m, top_n, 0.8), exact_topn(m, m, top_n, 0.8), "empty rows top_n=%d" % top_n)


def test_split_groups_are_still_exact():
    """a vector split over two groups (what a hash collision may cause on the device) keeps the result: expansion
    takes the union of the groups' members"""
    m, _, _ = P.tf_idf_matrices(_dup_corpus(800, 7))
    m = csr_matrix(m)
    uid, members = row_groups(m)
    big = max(range(len(members)), key=lambda u: len(members[u]))
    split = members[:big] + [members[big][::2], members[big][1::2]] + members[big + 1:]
    reps = np.array([g[0] for g in split])
    U = m[reps]
    u, v, s = exact_pairs(U, U, 0.8)
    size = np.array([len(g) for g in split])
    cols = np.concatenate([split[x] for x in v])
    gr, gc, gs, _ = topn_from_pairs(np.repeat(u, size[v]), cols, np.repeat(s, size[v]), 20)
    want = exact_topn(m, m, 20, 0.8)
    for g, grp in enumerate(split):
        for r in grp[:3]:
            w = want[0] == r
            assert np.array_equal(gc[gr == g], want[1][w]) and np.array_equal(gs[gr == g], want[2][w])

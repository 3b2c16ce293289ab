"""-m gpu: BASELINE.json's full-size configuration (663 000 names, self-match @0.8, top 20) checked through
size-independent properties plus an oracle spot check on sampled rows."""
import numpy as np
import pandas as pd
import pytest

from synth_corpus import make_names

pytestmark = pytest.mark.gpu
N = 663_000


@pytest.fixture(scope="module")
def fitted():
    from string_grouper_b200 import StringGrouper
    names = pd.Series(make_names(N, seed=0))
    sg = StringGrouper(names).fit()
    return names, sg


def test_full_size_structure(fitted):
    names, sg = fitted
    ml = sg._matches_list
    r, c, s = ml.master_side.to_numpy(), ml.dupe_side.to_numpy(), ml.similarity.to_numpy()
    key = r * N + c
    assert np.all(np.diff(key) > 0)                               # (row, col) ascending, no duplicates
    assert np.all(s > 0.8) and np.all(s <= 1.0 + 1e-9)            # strict threshold
    diag = r == c
    assert diag.sum() == N and np.all(s[diag] == 1.0)             # _fix_diagonal: every row, exactly 1
    rev = np.searchsorted(key, c * N + r)                         # _symmetrize_matrix: (c, r) present, same score
    assert np.array_equal(key[rev], c * N + r)
    assert np.array_equal(s[rev][~diag], s[~diag])
    assert sg._true_max_n_matches == 20                           # clusters of identical names fill top-n
    assert len(ml) > 4_000_000


def _threads():
    import bench_cpu
    return min(bench_cpu.usable_cores(), 16)


def test_full_size_kernels_and_pruning_levels_agree(fitted):
    """663k: the row kernel at the default pruning level, the TMA-staged tile kernel, and the UNPRUNED fp32 traversal
    return bit-identical triples (block invariance, reference tests :191-336; a pruning bug at scale cannot cancel)."""
    from string_grouper_b200 import _device as D
    names, sg = fitted
    A, _ = sg._get_tf_idf_matrices()
    st = {}
    a = D.cossim_topn(A, A, 20, 0.8, stats=st)
    assert st["kernel"] == "row" and st["prune"] > 0
    b = D.cossim_topn(A, A, 20, 0.8, kernel="row", prune=0.0, acc="f32")
    st2 = {}
    c = D.cossim_topn(A, A, 20, 0.8, kernel="tiles", stats=st2)
    assert st2["kernel"] == "tiles"
    ta = a.host_triples()
    assert a.nnz == b.nnz == c.nnz
    for other in (b.host_triples(), c.host_triples()):
        for x, y in zip(ta, other):
            assert np.array_equal(x, y)


def test_full_size_exact_on_sampled_rows(fitted):
    """663k: 2 000 sampled rows of the default product against the exact reference (tests/exact_topn.py), bit for bit
    with no exemption; at this size the row kernel uses 128-column tiles walked in column-tile groups."""
    from exact_topn import assert_same, exact_topn
    from string_grouper_b200 import _device as D
    names, sg = fitted
    A, _ = sg._get_tf_idf_matrices()
    st = {}
    got = D.cossim_topn(A, A, 20, 0.8, stats=st)
    assert st["kernel"] == "row" and st["acc"] == "u16" and st["select"] == "rows" and "n_refined" in st
    assert st["tile_w"] == 128 and st["tiles_per_group"] < st["n_tiles"]        # several column-tile groups
    host = A.to_scipy()
    rows = np.sort(np.random.default_rng(8).choice(N, 2000, replace=False))
    r, c, s, _ = exact_topn(host[rows], host, 20, 0.8, block_rows=128)
    gr, gc, gs = got.host_triples()
    sel = np.isin(gr, rows)
    assert_same((gr[sel], gc[sel], gs[sel]), (rows[r], c, s), "663k, sampled rows")


def test_full_size_all_pairs_equal_cpu_port(fitted):
    """BASELINE.json's headline configuration, EVERY pair: the whole 663k product on the CPU port with the reference's
    own block split (string_grouper.py:387-394 -> n_blocks (1, 166)), then fix-diagonal / symmetrise, against the CUDA
    match list (SURVEY.md §8c parity definition, all 4.36 M pairs)."""
    import bench_cpu
    from oracle import pipeline as P
    from string_grouper_b200 import _device as D
    names, sg = fitted
    A, _ = sg._get_tf_idf_matrices()
    full = A.to_scipy()                 # bit-equal to the sklearn matrix: tests/test_gpu_pipeline_exact.py (663k)
    C = P.build_matches(full, full, P.guess_blocks(N, N), 20, 0.8, _threads())
    S = P.symmetrize_fast(C)            # vectorised twin of the LIL restatement (tests/test_oracle.py)
    ml = P.matches_list(S)
    job = {"rows": N, "c_indptr": C.indptr.astype(np.int64), "c_indices": C.indices, "c_data": C.data,
           "row": ml.master_side.to_numpy(), "col": ml.dupe_side.to_numpy(), "score": ml.similarity.to_numpy()}
    pre = D.cossim_topn(A, A, 20, 0.8).host_triples()
    got = sg._matches_list
    par = bench_cpu.compare(job, pre, (got.master_side.to_numpy(), got.dupe_side.to_numpy(), got.similarity.to_numpy()))
    assert par["ok"], par
    assert par["product"]["max_abs_err"] <= 1e-9 and par["match_list"]["max_abs_err"] <= 1e-9
    assert par["match_list"]["pairs_ref"] > 4_000_000
    assert par["product"]["common"] >= 0.97 * par["product"]["pairs_ref"]     # the rest: top-n ties in clusters of identical names
    assert sg._true_max_n_matches == int(np.diff(C.indptr).max())


def test_config2_100k_all_pairs_equal_cpu_port():
    """BASELINE.json configs[1]: 100 000 names self-match @0.8, float32 on the GPU side is NOT used — the reference
    default float64 — every pair against the CPU port."""
    import bench_cpu
    from oracle import pipeline as P
    from string_grouper_b200 import StringGrouper, _device as D
    n = 100_000
    names = make_names(n, seed=0)
    sg = StringGrouper(pd.Series(names)).fit()
    m, d, _ = P.tf_idf_matrices(names)
    C = P.build_matches(m, d, P.guess_blocks(n, n), 20, 0.8, _threads())
    ml = P.matches_list(P.symmetrize_fast(C))
    job = {"rows": n, "c_indptr": C.indptr.astype(np.int64), "c_indices": C.indices, "c_data": C.data,
           "row": ml.master_side.to_numpy(), "col": ml.dupe_side.to_numpy(), "score": ml.similarity.to_numpy()}
    A, _ = sg._get_tf_idf_matrices()
    pre = D.cossim_topn(A, A, 20, 0.8).host_triples()
    got = sg._matches_list
    par = bench_cpu.compare(job, pre, (got.master_side.to_numpy(), got.dupe_side.to_numpy(), got.similarity.to_numpy()))
    assert par["ok"] and par["match_list"]["pairs_ref"] > 400_000, par


def test_config4_shape_two_series_all_pairs_equal_cpu_port():
    """BASELINE.json configs[3] shape (master x duplicates, min_similarity 0.7) at 400k x 150k: every pair."""
    from oracle import pipeline as P
    from parity import compare_triples, csr_triples, row_cutoffs
    from string_grouper_b200 import StringGrouper
    base = make_names(480_000, seed=3)
    master = pd.Series(base[:400_000])
    dupes = pd.Series(base[380_000:] + make_names(50_000, seed=4))          # 20k shared + 80k + 50k new
    sg = StringGrouper(master, dupes, min_similarity=0.7).fit()
    ml = sg._matches_list
    r, c, s = ml.master_side.to_numpy(), ml.dupe_side.to_numpy(), ml.similarity.to_numpy()
    assert np.all(np.diff(r) >= 0) and np.all(s > 0.7)
    same = r[1:] == r[:-1]
    assert np.all(s[1:][same] <= s[:-1][same])                       # sort=True inside a row
    assert np.bincount(r).max() <= 20 and c.max() < len(dupes)
    A, B = sg._get_tf_idf_matrices()
    fa, fb = A.to_scipy(), B.to_scipy()
    ref = P.build_matches(fa, fb, P.guess_blocks(len(master), len(dupes)), 20, 0.7, _threads())
    cut = row_cutoffs(ref.indptr, ref.data, 20, len(master))
    st = compare_triples(csr_triples(ref), (r, c, s), len(dupes), 0.7, tol=1e-9, cutoff_row=cut,
                         label="400k x 150k")
    assert st["common"] >= 0.97 * st["pairs_ref"] and st["pairs_ref"] > 100_000


def test_config5_shape_groups_equal_cpu_port():
    """BASELINE.json configs[4] shape: group_similar_strings @0.85 end to end (fit + dedupe) at 250k names against the
    CPU port.  (1) the match list equals the CPU port's (all pairs, boundary ties exempt); (2) the device group kernel
    equals the reference's _deduplicate restated (oracle/pipeline.deduplicate) on the SAME list, for both group_rep
    rules; (3) the groups agree with those of the CPU port's list except where top-n ties inside clusters of identical
    names moved a pair."""
    import bench_cpu
    from oracle import pipeline as P
    from string_grouper_b200 import StringGrouper, _device as D
    n = 250_000
    names = pd.Series(make_names(n, seed=5), name="name")
    ml = None
    for rep in ("centroid", "first"):
        sg = StringGrouper(names, min_similarity=0.85, group_rep=rep).fit()
        have = sg.get_groups()["group_rep_index"].to_numpy()
        mine = sg._matches_list
        assert np.array_equal(have, P.deduplicate(mine, n, rep)), rep          # (2)
        if ml is None:
            A, _ = sg._get_tf_idf_matrices()
            full = A.to_scipy()
            C = P.build_matches(full, full, P.guess_blocks(n, n), 20, 0.85, _threads())
            ml = P.matches_list(P.symmetrize_fast(C))
            job = {"rows": n, "c_indptr": C.indptr.astype(np.int64), "c_indices": C.indices, "c_data": C.data,
                   "row": ml.master_side.to_numpy(), "col": ml.dupe_side.to_numpy(), "score": ml.similarity.to_numpy()}
            pre = D.cossim_topn(A, A, 20, 0.85).host_triples()
            par = bench_cpu.compare(job, pre, (mine.master_side.to_numpy(), mine.dupe_side.to_numpy(),
                                               mine.similarity.to_numpy()), min_sim=0.85)
            assert par["ok"], par                                              # (1)
        # (3) same partition: label every string by the smallest index of its group
        def canon(reps):
            _, inv = np.unique(reps, return_inverse=True)
            first = np.full(inv.max() + 1, n, dtype=np.int64)
            np.minimum.at(first, inv, np.arange(n))
            return first[inv]
        want = P.deduplicate(ml, n, rep)
        assert (canon(have) != canon(want)).mean() < 0.005, rep
        assert (have != np.arange(n)).sum() > 10_000

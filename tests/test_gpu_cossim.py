"""-m gpu: K2 (postings -> candidates -> exact re-score -> top-n select) and K4 (symmetrise)
through the C ABI, against the CPU oracle on the same seeded inputs."""
import numpy as np
import pytest

from exact_topn import assert_same, exact_topn
from parity import compare_triples, csr_triples, row_cutoffs
from synth_corpus import make_names

pytestmark = pytest.mark.gpu


def _oracle():
    from oracle import pipeline
    return pipeline


def _run(master, dupes, top_n, thr, dtype=np.float64, tile_w=None, warps=None, prune=None, acc=None, stats=None,
         kernel=None):
    from string_grouper_b200 import _device as D
    P = _oracle()
    m, d, _ = P.tf_idf_matrices(master, dupes, dtype=dtype)
    ref = P.build_matches(m, d, None, top_n, thr, n_threads=4)
    A = D.DeviceCSR.from_scipy(m)
    B = A if dupes is None else D.DeviceCSR.from_scipy(d)
    got = D.cossim_topn(A, B, top_n, thr, tile_w=tile_w, warps=warps, prune=prune, acc=acc, stats=stats,
                        kernel=kernel)
    return m, d, ref, got


@pytest.mark.parametrize("n,top_n,thr,dtype", [
    (2000, 20, 0.8, np.float64),
    (2000, 20, 0.8, np.float32),
    (5000, 5, 0.6, np.float64),
    (3000, 1, 0.5, np.float64),
    (20000, 20, 0.8, np.float64),
])
@pytest.mark.parametrize("kernel", ["tiles", "row"])
def test_self_match_matches_oracle(n, top_n, thr, dtype, kernel):
    names = make_names(n, seed=1)
    st = {}
    m, d, ref, got = _run(names, None, top_n, thr, dtype, kernel=kernel, stats=st)
    assert st["kernel"] == kernel          # both K2 formulations against the oracle
    if kernel == "tiles":
        assert st["postings_walked"] > 0 and st["pairs_walked"] > 0
    gr, gc, gs = got.host_triples()
    cut = row_cutoffs(ref.indptr, ref.data, top_n, n)
    st = compare_triples(csr_triples(ref), (gr, gc, gs), n, thr, cutoff_row=cut, label="self %d" % n)
    assert st["common"] + st["boundary_ties"] >= n * 0.95   # at least the diagonal (ties may swap it)
    assert got.max_row == int(np.diff(ref.indptr).max())
    # bit for bit the exact reference (tests/exact_topn.py), ties and scores at the threshold included
    assert_same((gr, gc, gs, got.max_row), exact_topn(m, m, top_n, thr), "self %d exact" % n)
    # entries of a row come out by descending score (sort=True, string_grouper.py:730)
    same_row = gr[1:] == gr[:-1]
    assert np.all(gs[1:][same_row] <= gs[:-1][same_row])
    assert np.all(np.diff(gr) >= 0)


def test_two_series_and_tilings_agree():
    master = make_names(3000, seed=2)
    dupes = make_names(1500, seed=2)[:1000] + make_names(500, seed=3)
    m, d, ref, got = _run(master, dupes, 20, 0.7)
    cut = row_cutoffs(ref.indptr, ref.data, 20, len(master))
    compare_triples(csr_triples(ref), got.host_triples(), len(dupes), 0.7, cutoff_row=cut, label="two-series")
    # block invariance (reference tests test_n_blocks_*): any tile shape gives the same answer
    for tile_w, warps in [(128, 4), (256, 8), (1024, 16), (3072, 16), (1536, 32)]:
        _, _, _, g2 = _run(master, dupes, 20, 0.7, tile_w=tile_w, warps=warps, kernel="row")
        a, b = got.host_triples(), g2.host_triples()
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


@pytest.mark.parametrize("thr", [0.8, 0.5, 0.3])
def test_pruning_and_accumulator_variants_agree(thr):
    """Exact threshold pruning (csrc/sg_prune.cu) and the fixed-point accumulator tile only change which candidates
    are generated, never the result: every variant returns the same triples, bit for bit, as the unpruned
    fp32 traversal, and those equal the oracle."""
    names = make_names(12000, seed=11)
    st0 = {"count_macs": True}
    m, d, ref, base = _run(names, None, 20, thr, prune=0.0, acc="f32", stats=st0, kernel="row")
    cut = row_cutoffs(ref.indptr, ref.data, 20, len(names))
    compare_triples(csr_triples(ref), base.host_triples(), len(names), thr, cutoff_row=cut, label="unpruned")
    b = base.host_triples()
    walked = {}
    for prune, acc, tile_w, kernel in [(0.0, "u16", None, "row"), (0.5, "f32", None, "row"), (0.7, "u16", None, "row"),
                                       (0.9, "f32", 256, "row"), (0.95, "u16", 512, "row"), (0.7, "u16", 3072, "row"),
                                       (0.0, "u16", None, "tiles"), (0.5, "u16", None, "tiles"),
                                       (0.9, "u16", None, "tiles"), (0.97, "u16", None, "tiles")]:
        st = {"count_macs": True}
        _, _, _, got = _run(names, None, 20, thr, prune=prune, acc=acc, tile_w=tile_w, stats=st, kernel=kernel)
        g = got.host_triples()
        assert got.nnz == base.nnz, (prune, acc, kernel, got.nnz, base.nnz)
        for x, y in zip(b, g):
            assert np.array_equal(x, y), (prune, acc, tile_w, kernel)
        if kernel == "row":
            walked[(prune, acc)] = st.get("macs_walked")
        else:
            assert st["kernel"] == "tiles" or thr - 1e-3 < 0.05
    full = walked[(0.0, "u16")]
    assert walked[(0.7, "u16")] < 0.6 * full and walked[(0.95, "u16")] <= walked[(0.7, "u16")]


def test_pruning_two_series_unnormalised_rows():
    """user-supplied scipy matrices (rows not L2-normalised, a few negative weights): the bound uses the right
    matrix' largest row norm, the accumulator falls back to fp32."""
    from string_grouper_b200 import _device as D
    from oracle.sdt import sp_matmul_topn
    P = _oracle()
    master = make_names(4000, seed=21)
    dupes = make_names(3000, seed=22) + master[:500]
    m, d, _ = P.tf_idf_matrices(master, dupes)
    rng = np.random.default_rng(0)
    m = m.copy(); d = d.copy()
    m.data *= rng.uniform(0.5, 1.5, size=m.nnz)
    d.data *= rng.uniform(0.5, 2.0, size=d.nnz)
    d.data[rng.choice(d.nnz, size=50, replace=False)] *= -1.0
    ref = sp_matmul_topn(m, d.T.tocsr(), top_n=10, threshold=0.6, sort=True, n_threads=4)
    A, B = D.DeviceCSR.from_scipy(m), D.DeviceCSR.from_scipy(d)
    cut = row_cutoffs(ref.indptr, ref.data, 10, len(master))
    for prune in (0.0, 0.7):
        got = D.cossim_topn(A, B, 10, 0.6, prune=prune)
        compare_triples(csr_triples(ref), got.host_triples(), len(dupes), 0.6, cutoff_row=cut, label="unnormalised")


def test_row_chunks_and_adaptive_pruning_level(monkeypatch):
    """Left rows are processed in chunks when the candidate estimate exceeds CAND_CHUNK, and the pruning level is
    lowered when the sample pass reports too many candidates per pair; neither changes the result."""
    from string_grouper_b200 import _device as D
    P = _oracle()
    names = make_names(70000, seed=13)
    m, _, _ = P.tf_idf_matrices(names)
    A = D.DeviceCSR.from_scipy(m)
    base = D.cossim_topn(A, A, 20, 0.8, prune=0.0, acc="f32")
    b = base.host_triples()
    monkeypatch.setattr(D, "CAND_CHUNK", 1 << 19)
    for kernel in ("tiles", "row"):
        st = {}
        got = D.cossim_topn(A, A, 20, 0.8, stats=st, kernel=kernel)
        assert st["n_row_chunks"] > 1 and st["kernel"] == kernel
        for x, y in zip(b, got.host_triples()):
            assert np.array_equal(x, y)
    # a bucket directory that would exceed MAX_BUCKETS entries makes the tiles of the row kernel wider
    st3 = {}
    monkeypatch.setattr(D, "MAX_BUCKETS", 2_000_000)
    got3 = D.cossim_topn(D.DeviceCSR.from_scipy(m), D.DeviceCSR.from_scipy(m), 20, 0.8, stats=st3, kernel="row")
    assert st3["tile_w"] > st["tile_w"]
    for x, y in zip(b, got3.host_triples()):
        assert np.array_equal(x, y)
    st2 = {}
    monkeypatch.setattr(D, "MAX_CAND_DENSITY", 1e-7)
    got2 = D.cossim_topn(A, A, 20, 0.8, stats=st2)
    assert st2["prune"] < st["prune"]
    for x, y in zip(b, got2.host_triples()):
        assert np.array_equal(x, y)


def test_row_selection_paths_agree(monkeypatch):
    """per-row ranking (warp network for <= 32 survivors, one CTA for <= sg_topn_rows_cap) vs the three global sorts:
    identical triples, including clusters of identical names far beyond top_n and a row count beyond the CTA path."""
    from string_grouper_b200 import _device as D
    P = _oracle()
    base = make_names(9000, seed=17)
    for big in (700, 5000):        # 700: CTA path; 5000 > sg_topn_rows_cap(): the caller falls back to the sorts
        names = base + ["ACME HOLDINGS LLC"] * big + ["ACME HOLDINGS LLC %d" % (i % 7) for i in range(300)]
        m, _, _ = P.tf_idf_matrices(names)
        A = D.DeviceCSR.from_scipy(m)
        out = {}
        for mode in ("rows", "sort"):
            monkeypatch.setattr(D, "SELECT_MODE", mode)
            st = {}
            for top_n in (20, 1, 3000):
                got = D.cossim_topn(A, A, top_n, 0.8, stats=st)
                out[(mode, top_n)] = got.host_triples() + (got.max_row,)
                # rows longer than one CTA's shared memory are ranked in pieces as long as top_n <= cap / 2
                want = "sort" if (mode == "sort" or (big > 4096 and top_n > 2048)) else "rows"
                assert st["select"] == want, (big, top_n, st["select"])
        for top_n in (20, 1, 3000):
            a, b = out[("rows", top_n)], out[("sort", top_n)]
            assert a[3] == b[3]
            for x, y in zip(a[:3], b[:3]):
                assert np.array_equal(x, y), (big, top_n)
        ref = P.build_matches(m, m, None, 20, 0.8, n_threads=4)
        cut = row_cutoffs(ref.indptr, ref.data, 20, len(names))
        compare_triples(csr_triples(ref), out[("rows", 20)][:3], len(names), 0.8, cutoff_row=cut, label="clusters")


def test_long_rows():
    """strings of several hundred characters (more than 32 features per row: several lane batches)."""
    from string_grouper_b200 import _device as D
    P = _oracle()
    rng = np.random.default_rng(5)
    base = make_names(300, seed=9)
    longs = [" ".join(rng.choice(base, size=12)) for _ in range(200)]
    names = base + longs + longs[:50]
    m, d, _ = P.tf_idf_matrices(names)
    ref = P.build_matches(m, d, None, 10, 0.5)
    A = D.DeviceCSR.from_scipy(m)
    got = D.cossim_topn(A, A, 10, 0.5)
    cut = row_cutoffs(ref.indptr, ref.data, 10, len(names))
    compare_triples(csr_triples(ref), got.host_triples(), len(names), 0.5, cutoff_row=cut, label="long rows")


def test_top_n_larger_than_right_and_empty_rows():
    from string_grouper_b200 import _device as D
    P = _oracle()
    master = ["ab", "foo inc", "foo inc.", "", "bar llc", "x", "foo incorporated", "bar l.l.c"]
    m, d, _ = P.tf_idf_matrices(master)
    ref = P.build_matches(m, d, None, 50, 0.1)
    A = D.DeviceCSR.from_scipy(m)
    got = D.cossim_topn(A, A, 50, 0.1)
    compare_triples(csr_triples(ref), got.host_triples(), len(master), 0.1, label="tiny")
    np.testing.assert_allclose(got.toarray(), ref.toarray(), atol=1e-12)


def test_reference_fixture_build_matches():
    """test_build_matches (reference test_string_grouper.py:546-556): exact dense answer."""
    from string_grouper_b200 import _device as D
    P = _oracle()
    m, d, _ = P.tf_idf_matrices(['foo', 'bar', 'baz'], ['foo', 'bar', 'bop'])
    got = D.cossim_topn(D.DeviceCSR.from_scipy(m), D.DeviceCSR.from_scipy(d), 20, 0.8)
    np.testing.assert_array_equal(got.toarray(), np.array([[1., 0., 0.], [0., 1., 0.], [0., 0., 0.]]))


def test_symmetrize_matches_lil_restatement():
    from string_grouper_b200 import _device as D
    P = _oracle()
    names = make_names(4000, seed=5) + ["zz", ""]
    m, d, ref, got = _run(names, None, 3, 0.75)
    ref_sym = P.fix_diagonal_and_symmetrize(ref)
    sym = D.symmetrize(got)
    r, c, s = sym.host_triples()
    n = len(names)
    cut = row_cutoffs(ref.indptr, ref.data, 3, n)
    compare_triples(csr_triples(ref_sym), (r, c, s), n, 0.75, cutoff_row=cut, cutoff_col=cut, label="symm")
    key = r.astype(np.int64) * n + c
    assert np.all(np.diff(key) > 0)                      # (row, col) ascending, no duplicates
    assert np.all(s[r == c] == 1.0) and (r == c).sum() == n


def _rowwise_dot_exact(dtype):
    """bit-equal to the reference's dot() (scipy's p0 + numpy pairwise order, tests/exact_pipeline.py)"""
    from string_grouper_b200 import _device as D
    P = _oracle()
    a = make_names(1000, seed=7)
    b = make_names(1000, seed=7)[:500] + make_names(500, seed=8)
    m, d, _ = P.tf_idf_matrices(a, b, dtype=dtype)
    ref = np.asarray(m.multiply(d).sum(axis=1)).squeeze(axis=1)
    got = D.rowwise_dot(D.DeviceCSR.from_scipy(m), D.DeviceCSR.from_scipy(d))
    assert got.dtype == ref.dtype == dtype
    assert np.array_equal(got, ref), "%d rows differ" % (got != ref).sum()


def test_rowwise_dot():
    _rowwise_dot_exact(np.float64)


def test_rowwise_dot_float32():
    _rowwise_dot_exact(np.float32)


def test_nearest_master_matches_host_rule():
    """sg_nearest_master: per right row the left row with the highest score, smallest index among equals."""
    import torch
    from string_grouper_b200 import _device as D
    rng = np.random.default_rng(3)
    n_left, n_right, nnz = 5000, 3000, 40000
    r = rng.integers(0, n_left, nnz).astype(np.int32)
    c = rng.integers(0, n_right - 100, nnz).astype(np.int32)          # the last 100 right rows stay unmatched
    s = np.round(rng.random(nnz), 2)                                   # many exact ties
    dev = torch.device("cuda", torch.cuda.current_device())
    M = D.DeviceMatches((n_left, n_right), torch.from_numpy(r).to(dev), torch.from_numpy(c).to(dev),
                        torch.from_numpy(s).to(dev), nnz, 0)
    got = D.nearest_master(M, n_right)
    order = np.lexsort((r, -s, c))
    first = np.ones(nnz, dtype=bool)
    first[1:] = c[order][1:] != c[order][:-1]
    want = np.full(n_right, -1, dtype=np.int64)
    want[c[order][first]] = r[order][first]
    assert np.array_equal(got, want)
    assert np.all(got[-100:] == -1)


@pytest.mark.parametrize("thr,two", [(0.8, False), (0.6, False), (0.7, True)])
def test_grouped_bound_refinement_changes_nothing_but_the_work(monkeypatch, thr, two):
    """sg_rescore_refined drops candidates whose partial score plus the grouped Cauchy-Schwarz bound of the pruned part
    cannot reach the row's threshold: same triples as the plain re-score of every candidate, fewer rows read."""
    from string_grouper_b200 import _device as D
    names = make_names(30000, seed=21)
    master, dupes = (names[:20000], names[20000:]) if two else (names, None)
    out = {}
    for on in (False, True):
        monkeypatch.setattr(D, "REFINE", on)
        st = {}
        _, _, ref, got = _run(master, dupes, 20, thr, stats=st, kernel="row")
        out[on] = (got.host_triples(), st)
    (a, st_off), (b, st_on) = out[False], out[True]
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    assert "n_refined" not in st_off and st_on["n_candidates"] == st_off["n_candidates"]
    assert st_on["n_above_threshold"] == st_off["n_above_threshold"] <= st_on["n_refined"] < 0.7 * st_on["n_candidates"]
    cut = row_cutoffs(ref.indptr, ref.data, 20, len(master))
    compare_triples(csr_triples(ref), b, len(master) if dupes is None else len(dupes), thr, cutoff_row=cut,
                    label="refined")


def test_group_norms_bound_the_heavy_part():
    """fp16 group norms of sg_heavy_norms / sg_prune_rows: never below the fp64 norm of the group, within 0.2 % of it;
    pruned features are heavy features and the 16 groups partition them (ranks 0..13 alone, 14..38, 39..63)."""
    from string_grouper_b200 import _device as D
    P = _oracle()
    names = make_names(6000, seed=3)
    m, _, _ = P.tf_idf_matrices(names, None, dtype=np.float64)
    A = D.DeviceCSR.from_scipy(m)
    hrank, perm, rank = D.right_order(A)
    hr = hrank.cpu().numpy().astype(np.int64)
    grp = np.where(hr < 14, hr, np.where(hr < 39, 14, 15))
    yg = A._heavy_groups.float().cpu().numpy().reshape(-1, 16)
    yh = A._heavy_norm.cpu().numpy()
    csr = m.tocsr()
    sq = csr.multiply(csr).tocsr()
    for g in range(16):
        cols = np.flatnonzero((hr >= 0) & (grp == g))
        true = np.sqrt(np.asarray(sq[:, cols].sum(axis=1)).ravel())
        assert np.all(yg[:, g] >= true) and np.all(yg[:, g] <= true * 1.002 + 2e-6), g
    assert np.all(np.sqrt((yg.astype(np.float64) ** 2).sum(1)) >= yh * (1 - 1e-4))
    p_idx, p_val, p_len, p_thr, p_xp, p_xg = D.prune_left(A, A, hrank, 0, A.shape[0], 0.8, D.CAND_MARGIN,
                                                        D.U16_MARGIN_PER_FEATURE, 0.9)
    xg = p_xg.float().cpu().numpy().reshape(-1, 16).astype(np.float64)
    xp = p_xp.cpu().numpy()
    kept_len = p_len.cpu().numpy()
    kept_idx = p_idx.cpu().numpy()
    indptr = m.indptr
    assert (xp > 0).sum() > 1000
    for r in np.flatnonzero(xp > 0)[:500]:
        kept = set(kept_idx[indptr[r]:indptr[r] + kept_len[r]].tolist())
        pruned = [(f, v) for f, v in zip(m.indices[indptr[r]:indptr[r + 1]], m.data[indptr[r]:indptr[r + 1]])
                  if f not in kept]
        assert pruned and all(hr[f] >= 0 for f, _ in pruned)
        for g in range(16):
            true = np.sqrt(sum(v * v for f, v in pruned if grp[f] == g))
            assert true <= xg[r, g] <= true * 1.002 + 2e-6, (r, g)

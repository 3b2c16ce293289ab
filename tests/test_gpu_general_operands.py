"""-m gpu: the top-n product on general sparse operands bit for bit against the exact reference (tests/exact_topn.py,
tests/exact_nearest.py): rows of any norm, raw counts, signed weights, weights far below fp16's range, unbalanced
norms, non-canonical CSR.  The special rows are embedded in a few thousand TF-IDF rows (the right side spans many
column tiles, and their features are light).  Every case asserts from `stats` which path ran; the rules these
operands meet are restated in numpy in tests/test_general_bounds_math.py."""
import numpy as np
import pytest
import scipy.sparse as sp

from exact_nearest import exact_nearest
from exact_topn import RankedPairs, assert_same, exact_pairs
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

TOP_N = 20
N_BASE = 2500


def _D():
    from string_grouper_b200 import _device as D
    return D


def _base(seed=31):
    from oracle import pipeline as P
    m, _, _ = P.tf_idf_matrices(make_names(N_BASE, seed=seed))
    return m.tocsr()


def _rows(rows, n_cols):
    ind = [np.asarray(c, dtype=np.int64) for c, _ in rows]
    val = [np.asarray(v, dtype=np.float64) for _, v in rows]
    return sp.csr_matrix((np.concatenate(val), np.concatenate(ind), np.cumsum([0] + [len(c) for c in ind])),
                         shape=(len(rows), n_cols))


def _embed(m, rows, extra_cols):
    """m's rows, then `rows` (features of m and extra_cols new ones after them)"""
    V = m.shape[1] + extra_cols
    m = sp.hstack([m, sp.csr_matrix((m.shape[0], extra_cols))]).tocsr()
    return sp.vstack([m, _rows(rows, V)]).tocsr() if rows else m


def _shapes(rng, V0, col):
    """empty rows, single-feature rows, rows of more than 32 and more than 64 features (new features)"""
    rows = [([], []), ([col], [0.7]), ([col], [0.7]), ([col + 1], [2.5])]
    for nf in (33, 40, 65, 90):
        f = np.concatenate([[col + 2 + k for k in range(4)], rng.choice(V0, size=nf - 4, replace=False)])
        rows += [(np.sort(f), rng.uniform(0.05, 1.0, size=nf))] * 2
    return rows, 6


def family(name):
    """(A, B) scipy CSR; A is B for one matrix"""
    rng = np.random.default_rng(sum(map(ord, name)))
    m = _base()
    V0 = m.shape[1]
    extra, n_extra = _shapes(rng, V0, V0)
    col = V0 + n_extra
    if name in ("scaled", "scaled_f32"):
        m = (sp.diags(10.0 ** rng.uniform(-3, 3, size=m.shape[0])) @ m).tocsr()
    elif name == "uniform":
        for norm in (3.0, 10.0, 100.0):
            for n in (16, 29, 40):
                extra += [(np.arange(col, col + n), np.full(n, norm / np.sqrt(n)))] * 2
                col += n
    elif name == "counts":
        for k in range(40):
            nf = int(rng.choice([1, 3, 12, 40, 80]))
            extra.append((np.sort(rng.choice(np.arange(V0, V0 + n_extra), size=min(nf, n_extra), replace=False))
                          if nf <= n_extra else np.sort(rng.choice(V0, size=nf, replace=False)),
                          rng.integers(1, 501, size=min(nf, n_extra) if nf <= n_extra else nf)))
        extra += [([col], [300]), ([col, col + 1], [300, 1]), ([col + 1], [1])]
        col += 2
    elif name == "signed":
        m = m.copy()
        m.data[rng.random(m.nnz) < 0.2] *= -1
        extra += [([col, col + 1], [1, 1]), ([col, col + 1], [1, -0.9999]), ([col, col + 1], [1, -1.0001])]
        col += 2
    elif name == "tiny":
        for k in range(0, 300, 3):                  # next to unit rows of the same features
            r = m[k]
            extra.append((r.indices, 10.0 ** rng.uniform(-12, -9, size=r.nnz)))
        for k in range(20):                         # and on features of their own: only tiny scores in their rows
            f = np.arange(col, col + 3)
            extra += [(f, 10.0 ** rng.uniform(-12, -9, size=3)), (f, 10.0 ** rng.uniform(-12, -9, size=3))]
            col += 3
    elif name != "unbalanced":
        raise KeyError(name)
    M = _embed(m, extra, col - V0)
    if name == "scaled_f32":
        M = M.astype(np.float32)
    if name == "unbalanced":
        return (4.0 * M).tocsr(), (0.25 * M).tocsr()
    return M, M


FAMILIES = ["scaled", "scaled_f32", "uniform", "counts", "signed", "tiny", "unbalanced"]


@pytest.fixture(scope="module")
def fam():
    """name -> (A, B device, host canonical copies, RankedPairs of every nonzero pair, margin)"""
    D = _D()
    cache = {}

    def get(name):
        if name not in cache:
            Ah, Bh = family(name)
            A = D.DeviceCSR.from_scipy(Ah)
            B = A if Ah is Bh else D.DeviceCSR.from_scipy(Bh)
            a, b = A.to_scipy(), B.to_scipy()
            margin = D.CAND_MARGIN * max(A.norm_bound * B.norm_bound, 1.0)
            cache[name] = (A, B, a, b, RankedPairs(*exact_pairs(a, b, -np.inf)), margin)
        return cache[name]
    return get


def _run(A, B, thr, expect, top_n=TOP_N, **kw):
    st = {}
    got = _D().cossim_topn(A, B, top_n, thr, stats=st, **kw)
    for k, v in expect.items():
        assert st.get(k) == v, "path: %s is %r, expected %r (%r)" % (k, st.get(k), v, kw)
    return got.host_triples() + (got.max_row,)


def _pick(table, a, margin):
    """pair scores where kernels go wrong: quantiles of the visible scores, the largest, pairs of long rows"""
    vis = (table.rank < TOP_N) & (table.score > margin * 1.01)
    s = table.score[vis]
    nnz = np.diff(a.indptr)
    picks = [s.max()] + [np.quantile(s, q, method="nearest") for q in (0.1, 0.5, 0.9)]
    long_ = vis & (nnz[table.row] > 32)
    if long_.any():
        picks.append(table.score[long_].max())
    return sorted(set(float(x) for x in picks))


def _thresholds(table, a, margin):
    return [t for s in _pick(table, a, margin) for t in (s, float(np.nextafter(s, -np.inf)))]


# ---------------------------------------------------------------------------------------------------------------
# thresholds on the pair scores, one matrix (the triangle) and two
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", FAMILIES)
def test_thresholds_on_pair_scores(fam, name):
    A, B, a, b, table, margin = fam(name)
    self_match = A is B
    for thr in _thresholds(table, a, margin):
        want = table.topn(TOP_N, thr)
        got = _run(A, B, thr, {"kernel": "row", "acc": "f32", "triangle": self_match, "topn_floor": False})
        assert_same(got, want, "%s thr=%r" % (name, thr))


@pytest.mark.parametrize("name", ["scaled", "uniform", "counts", "tiny"])
def test_two_matrices_and_row_ranges(fam, name):
    """left = every other row (two matrices, the full product), then a shard of rows of the self-match"""
    D = _D()
    A, B, a, b, table, margin = fam(name)
    thr = _pick(table, a, margin)[1]
    left = a[::2]
    Al = D.DeviceCSR.from_scipy(left)
    want = RankedPairs(*exact_pairs(left, b, thr)).topn(TOP_N, thr)
    assert_same(_run(Al, B, thr, {"kernel": "row", "triangle": False}), want, name + " two matrices")
    lo, hi = 700, 1900
    st = {}
    got = D.cossim_topn(A, B, TOP_N, thr, row_begin=lo, row_end=hi, stats=st)
    assert st["triangle"] is False
    assert_same(got.host_triples() + (got.max_row,), table.topn(TOP_N, thr, rows=(lo, hi)), name + " shard")


@pytest.mark.parametrize("name", ["scaled", "counts", "tiny", "uniform", "scaled_f32"])
@pytest.mark.parametrize("thr", ["zero", "-inf", "below_margin"])
def test_thresholds_below_the_margin(fam, name, thr):
    """every pair with a positive score counts: weights down to 1e-12 included (non-negative operands)"""
    A, B, a, b, table, margin = fam(name)
    t = {"zero": 0.0, "-inf": -np.inf, "below_margin": 0.5 * margin}[thr]
    want = table.topn(TOP_N, max(t, 0.0) if t > -np.inf else -np.inf)
    for prune in (None, 0.0):
        got = _run(A, B, t, {"kernel": "row", "acc": "f32", "dedup": False, "blocks": False}, prune=prune, dedup=False)
        assert_same(got, want, "%s thr=%r prune=%r" % (name, t, prune))


def test_tiny_weights_are_found(fam):
    A, B, a, b, table, margin = fam("tiny")
    small = table.score < 1e-15
    assert small.sum() > 1000 and (table.rank[small] < TOP_N).sum() >= 60


@pytest.mark.parametrize("name", ["scaled", "counts", "tiny"])
def test_floor_dedup_chunks_blocks_and_nearest(fam, monkeypatch, name):
    D = _D()
    A, B, a, b, table, margin = fam(name)
    thr = 0.0
    want = table.topn(TOP_N, thr)
    # the top-n floor (non-negative operands)
    assert_same(_run(A, B, thr, {"topn_floor": True}, floor=True), want, name + " floor")
    # identical rows: the product over the distinct rows
    assert_same(_run(A, B, thr, {"dedup": True, "topn_floor": False}, floor=False, dedup=True), want, name + " dedup")
    # row chunks
    monkeypatch.setattr(D, "CAND_CHUNK", 1 << 15)
    st = {}
    got = D.cossim_topn(A, B, TOP_N, thr, stats=st, floor=False, dedup=False)
    assert st["n_row_chunks"] > 1
    assert_same(got.host_triples() + (got.max_row,), want, name + " chunks")
    monkeypatch.undo()
    # blocks: pairs whose rows share a block id
    ids = (np.arange(a.shape[0]) % 7).astype(np.int32)
    d_ids = D.block_id_tensors(ids, a.shape[0], True)
    keep = ids[table.row] == ids[table.col]
    bt = RankedPairs(table.row[keep], table.col[keep], table.score[keep])
    assert_same(_run(A, B, thr, {"blocks": True}, block_ids=d_ids), bt.topn(TOP_N, thr), name + " blocks")
    # nearest
    st = {}
    best, score = D.cossim_nearest(A, B, thr, stats=st)
    wb, ws = exact_nearest(a, b, thr)
    assert np.array_equal(best, wb) and np.array_equal(score, ws), name + " nearest"


def test_unbalanced_norms_leave_the_fixed_point_paths(fam):
    """A scaled by 4 and B by 0.25: scores as before, but u16 and the tile kernel take products of weights <= 1"""
    A, B, a, b, table, margin = fam("unbalanced")
    for thr in _thresholds(table, a, margin)[:4]:
        want = table.topn(TOP_N, thr)
        for kw in ({"acc": "u16"}, {"kernel": "tiles"}):
            assert_same(_run(A, B, thr, {"kernel": "row", "acc": "f32"}, **kw), want, "unbalanced %r" % kw)


def test_signed_operands(fam):
    """signed weights above the margin are exact; below it the call is refused before any launch"""
    D = _D()
    A, B, a, b, table, margin = fam("signed")
    for thr in _thresholds(table, a, margin)[:4] + [margin]:
        assert_same(_run(A, B, thr, {"kernel": "row", "acc": "f32"}, prune=0.0), table.topn(TOP_N, thr),
                    "signed thr=%r" % thr)
    launches = dict(D.LAUNCH_COUNTS)
    for thr in (0.0, -np.inf, -0.5, 0.5 * margin):
        with pytest.raises(ValueError, match="threshold of at least"):
            D.cossim_topn(A, B, TOP_N, thr)
    with pytest.raises(ValueError, match="threshold of at least"):
        D.cossim_nearest(A, B, 0.0)
    assert D.LAUNCH_COUNTS == launches


# ---------------------------------------------------------------------------------------------------------------
# the public operator
# ---------------------------------------------------------------------------------------------------------------
def _compat_triples(C):
    C = C.tocsr()
    r = np.repeat(np.arange(C.shape[0]), np.diff(C.indptr))
    return r, C.indices.astype(np.int64), C.data.astype(np.float64)


@pytest.mark.parametrize("name", ["scaled", "counts", "tiny", "signed"])
def test_sp_matmul_topn(fam, name):
    from string_grouper_b200.sparse_dot_topn_compat import sp_matmul_topn
    A, B, a, b, table, margin = fam(name)
    thrs = [_pick(table, a, margin)[1]] + ([None, 0.0] if name != "signed" else [])
    a64, bt64 = a.copy(), b.T.tocsr()
    for x in (a64, bt64):                               # int64 index arrays
        x.indices, x.indptr = x.indices.astype(np.int64), x.indptr.astype(np.int64)
        assert x.indices.dtype == np.int64
    for thr in thrs:
        want = table.topn(TOP_N, -np.inf if thr is None else thr)
        for sort, (x, y) in ((True, (a, b.T)), (False, (a64, bt64))):
            got = _compat_triples(sp_matmul_topn(x, y, top_n=TOP_N, threshold=thr, sort=sort))
            assert_same(got, want[:3], "%s thr=%r sort=%r" % (name, thr, sort))


def test_sp_matmul_topn_non_canonical_input(fam):
    """duplicate entries are summed, unsorted indices sorted, explicit zeros dropped: the product of the canonical
    matrix, as scipy's"""
    from string_grouper_b200.sparse_dot_topn_compat import sp_matmul_topn
    A, B, a, b, table, margin = fam("counts")
    rng = np.random.default_rng(3)
    coo = a.tocoo()
    k = rng.choice(coo.nnz, size=coo.nnz // 3, replace=False)
    part = rng.uniform(0.2, 0.8, size=len(k))
    zero = rng.choice(coo.nnz, size=200, replace=False)
    rows = np.concatenate([coo.row, coo.row[k], coo.row[zero]])
    cols = np.concatenate([coo.col, coo.col[k], coo.col[zero]])
    vals = np.concatenate([coo.data, np.zeros(len(k)), np.zeros(200)])
    vals[k] *= part                                     # the duplicates add up to the original value ...
    vals[coo.nnz + np.arange(len(k))] = coo.data[k] * (1 - part)
    o = rng.permutation(len(rows))                      # ... in no particular order inside a row
    o = o[np.argsort(rows[o], kind="stable")]
    indptr = np.r_[0, np.cumsum(np.bincount(rows, minlength=a.shape[0]))]
    raw = sp.csr_matrix((vals[o], cols[o], indptr), shape=a.shape)
    assert not raw.has_canonical_format
    canon = raw.copy()
    canon.sum_duplicates()
    canon.eliminate_zeros()
    thr = _pick(table, a, margin)[1]
    want = RankedPairs(*exact_pairs(canon, canon, thr)).topn(TOP_N, thr)
    got = _compat_triples(sp_matmul_topn(raw, raw.T.tocsr(), top_n=TOP_N, threshold=thr, sort=True))
    assert_same(got, want[:3], "non-canonical")


def test_refused_inputs_raise_before_any_launch():
    from string_grouper_b200.sparse_dot_topn_compat import sp_matmul_topn
    D = _D()
    m = _base()[:200].tocsr()
    launches = dict(D.LAUNCH_COUNTS)
    for bad, match in ((np.nan, "NaN or infinite"), (np.inf, "NaN or infinite"), (1e-300, "2\\^-50 and 2\\^50"),
                       (1e300, "2\\^-50 and 2\\^50")):
        x = m.copy()
        x.data[5] = bad
        with pytest.raises(ValueError, match=match):
            sp_matmul_topn(x, m.T, top_n=5, threshold=0.5)
    s = m.copy()
    s.data[::4] *= -1
    with pytest.raises(NotImplementedError):
        sp_matmul_topn(s, s.T, top_n=5, threshold=None)
    with pytest.raises(ValueError, match="threshold of at least"):
        sp_matmul_topn(s, s.T, top_n=5, threshold=0.0)
    assert D.LAUNCH_COUNTS == launches

"""-m gpu: K2, K3 and K4 against the exact reference (tests/exact_topn.py).  Every test compares the WHOLE output with
np.array_equal: rows, columns, scores bit for bit, the output order and max_row, with no exemption for scores near
the threshold or ties at the cut.  Every case also asserts from `stats` which path ran, because cossim_topn silently
changes path (fp32 accumulator for low thresholds or unnormalised input, row kernel when the tiles do not apply, the
global sorts for long rows with a large top_n)."""
import numpy as np
import pytest
from scipy.sparse import csr_matrix, hstack, vstack

from exact_topn import RankedPairs, assert_same, exact_pairs, exact_topn, exact_zip, to_csr
from synth_corpus import make_names

pytestmark = pytest.mark.gpu

TOP_N = 20
FLOOR = 0.3           # every threshold of the score tests lies above this
# features of the uniform-weight rows (see _uniform_rows)
UNIFORM = (116, 134, 660)


def _D():
    from string_grouper_b200 import _device as D
    return D


def _P():
    from oracle import pipeline as P
    return P


def _run(A, B, top_n, thr, expect, **kw):
    """cossim_topn -> ((row, col, score, max_row), stats); asserts every stats entry of `expect` ("n_refined": True
    means the grouped-bound re-score ran, False that it did not)"""
    st = {}
    got = _D().cossim_topn(A, B, top_n, thr, stats=st, **kw)
    for k, v in expect.items():
        have = ("n_refined" in st) if k == "n_refined" else st.get(k)
        assert have == v, "path: %s is %r, expected %r (%r)" % (k, have, v, kw)
    return got.host_triples() + (got.max_row,), st


# ---------------------------------------------------------------------------------------------------------------
# corpus for thresholds set on the scores
# ---------------------------------------------------------------------------------------------------------------
def _uniform_rows(first_col):
    """Two identical rows per n in UNIFORM: n features nobody else holds, every weight 1/sqrt(n).  Every product
    rounds the same way, so the fixed-point errors add up instead of cancelling: at n = 134 the 16-bit accumulator
    of the row kernel ends 22/32768 below the threshold minus CAND_MARGIN (only the per-feature margin keeps the
    pair), at n = 116 and 660 the 2^-15 products of the tile kernel end 2.8e-4 and 7.7e-4 below the exact score
    (far beyond TILE_MARGIN)."""
    rows, col = [], first_col
    for n in UNIFORM:
        for _ in range(2):
            rows.append((np.arange(col, col + n), np.full(n, 1.0 / np.sqrt(n))))
        col += n
    return rows, col


def _names():
    rng = np.random.default_rng(5)
    names = make_names(10000, seed=23)
    base = names[:400]
    longs = [" ".join(rng.choice(base, size=12)) for _ in range(120)]      # > 64 features
    mids = [" ".join(rng.choice(base, size=3)) for _ in range(120)]        # 33 .. 64 features
    near = [s[:-len(s.split()[-1]) - 1] for s in longs[:60]] + [s.replace("A", "E", 1) for s in mids[:60]]
    singles = ["llc", "LLC", "L.L.C.", "inc", "Inc.", "ltd", "LTD", "org"]   # one trigram: weight exactly 1
    return names + longs + mids + near + longs[:20] + mids[:20] + singles


def _matrix(dtype):
    P = _P()
    m, _, _ = P.tf_idf_matrices(_names(), dtype=dtype)
    rows, n_cols = _uniform_rows(m.shape[1])
    u = csr_matrix((np.concatenate([v for _, v in rows]).astype(dtype), np.concatenate([c for c, _ in rows]),
                    np.cumsum([0] + [len(c) for c, _ in rows])), shape=(len(rows), n_cols))
    m = vstack([hstack([m, csr_matrix((m.shape[0], n_cols - m.shape[1]), dtype=dtype)]), u]).tocsr().astype(dtype)
    m.sort_indices()
    return m


def _fp16_shortfall(m, r, c):
    """exact score - the score the fp32 accumulator of the row kernel adds up (fp32 left weights times fp16 right
    weights) for the pairs (r, c)"""
    a = m[r].astype(np.float32).astype(np.float64)
    w = m[c].copy()
    w.data = w.data.astype(np.float32).astype(np.float16).astype(np.float64)
    approx = np.asarray(a.multiply(w.astype(np.float64)).sum(axis=1)).ravel()
    exact = np.asarray(m[r].astype(np.float64).multiply(m[c].astype(np.float64)).sum(axis=1)).ravel()
    return exact - approx


def _pick_scores(m, table):
    """a few dozen distinct pair scores in (FLOOR, 1] where kernels go wrong; every chosen pair is within the top
    TOP_N of its row, so it shows in the output as soon as the threshold lets it in"""
    vis = (table.rank < TOP_N) & (table.row != table.col) & (table.score > FLOOR + 0.01)
    r, c, s = table.row[vis], table.col[vis], table.score[vis]
    nnz = np.diff(m.indptr)
    picks = []
    if np.any(s == 1.0):
        picks.append(1.0)                                              # single-feature rows
    picks.append(s[s < 1.0].max())                                     # the largest score below 1
    u = np.unique(s[(s > 0.5) & (s < 0.99)])
    k = int(np.argmin(np.diff(u)))
    picks += [u[k], u[k + 1]]                                          # the two nearest distinct scores
    for sel in ((nnz[r] > 64) & (nnz[c] > 64) & (s < 0.99), (nnz[r] > 32) & (nnz[r] <= 64) & (s < 0.99),
                (nnz[r] == 1) & (s < 1.0)):
        if sel.any():
            picks.append(np.sort(s[sel])[sel.sum() // 2])
    for q in (0.35, 0.5, 0.65, 0.8, 0.9):
        picks.append(s[np.argmin(np.abs(s - q))])
    # the pairs the fp16 posting weights underestimate most: lost first when a candidate margin is too small
    sample = np.random.default_rng(2).choice(len(r), size=min(len(r), 40000), replace=False)
    short = _fp16_shortfall(m, r[sample], c[sample])
    picks += list(s[sample[np.argsort(-short)[:3]]])
    # the uniform-weight rows: their pair score
    first = m.shape[0] - 2 * len(UNIFORM)
    for k in range(len(UNIFORM)):
        sel = (r == first + 2 * k) & (c == first + 2 * k + 1)
        assert sel.sum() == 1
        picks.append(s[sel][0])
    return sorted(set(float(x) for x in picks))


@pytest.fixture(scope="module")
def scored():
    """dtype -> (device matrix, RankedPairs of all pairs above FLOOR, chosen scores)"""
    D = _D()
    out = {}
    for dtype in (np.float64, np.float32):
        m = _matrix(dtype)
        A = D.DeviceCSR.from_scipy(m)
        host = A.to_scipy()
        table = RankedPairs(*exact_pairs(host, host, FLOOR))
        scores = _pick_scores(host, table)
        assert len(scores) >= 12
        for s in scores:           # the chosen pair is out at threshold s and in just below it
            assert len(table.topn(TOP_N, s)[0]) < len(table.topn(TOP_N, np.nextafter(s, -np.inf))[0])
        out[dtype] = (A, table, scores)
    return out


def _thresholds(scores):
    return [t for s in scores for t in (s, float(np.nextafter(s, -np.inf)))]


# kernel, acc, prune (None = the default level), REFINE, tile_w (None = automatic), SELECT_MODE
DEFAULT = ("row", "u16", None, True, None, "rows")
CONFIGS = [
    DEFAULT,
    ("row", "u16", 0.0, True, None, "rows"),
    ("row", "u16", 0.5, True, 128, "rows"),
    ("row", "u16", 0.97, True, 3072, "rows"),
    ("row", "u16", 0.9, False, None, "rows"),
    ("row", "u16", 0.9, True, 256, "sort"),
    ("row", "f32", 0.0, True, None, "rows"),
    ("row", "f32", 0.9, True, 256, "sort"),
    ("row", "f32", 0.97, False, 3072, "rows"),
    ("tiles", "u16", None, True, None, "rows"),
    ("tiles", "u16", 0.0, True, None, "sort"),
    ("tiles", "u16", 0.5, True, None, "rows"),
    ("tiles", "u16", 0.97, True, None, "rows"),
]
CONFIGS_F32 = [DEFAULT, ("row", "f32", 0.0, True, None, "rows"), ("tiles", "u16", 0.9, True, None, "sort")]


def _config(monkeypatch, cfg):
    """apply a configuration: (keyword arguments of cossim_topn, expected stats)"""
    D = _D()
    kernel, acc, prune, refine, tile_w, select = cfg
    monkeypatch.setattr(D, "REFINE", refine)
    monkeypatch.setattr(D, "SELECT_MODE", select)
    kw = {"kernel": kernel, "acc": acc, "prune": prune, "tile_w": tile_w}
    expect = {"kernel": kernel, "acc": acc, "prune": D.PRUNE_FRAC if prune is None else prune, "n_row_chunks": 1,
              "n_refined": refine and kernel == "row" and acc == "u16"}
    if kernel == "row":
        expect["tile_w"] = tile_w or (256 if acc == "u16" else 128)
    return kw, expect


def _cfg_id(cfg):
    return "-".join(str(x) for x in cfg)


@pytest.mark.parametrize("dtype,cfg", [(np.float64, c) for c in CONFIGS] + [(np.float32, c) for c in CONFIGS_F32],
                         ids=["f64-" + _cfg_id(c) for c in CONFIGS] + ["f32-" + _cfg_id(c) for c in CONFIGS_F32])
def test_thresholds_on_pair_scores(scored, monkeypatch, dtype, cfg):
    """threshold = a pair's exact score (the pair must be out) and the next double below it (the pair must be in),
    for a few dozen scores chosen where margins run out: nearly equal scores, the largest score below 1, exactly 1
    (single-feature rows, 32768 in a 16-bit word), long rows (more than 32 and 64 kept features), the pairs the fp16
    weights underestimate most, and rows whose fixed-point roundings all go the same way."""
    A, table, scores = scored[dtype]
    kw, expect = _config(monkeypatch, cfg)
    for thr in _thresholds(scores):
        want = table.topn(TOP_N, thr)
        got, st = _run(A, A, TOP_N, thr, dict(expect, select=cfg[5]), **kw)
        assert_same(got, want, "%s thr=%r" % (_cfg_id(cfg), thr))


# ---------------------------------------------------------------------------------------------------------------
# scores exactly on the threshold
# ---------------------------------------------------------------------------------------------------------------
def _dyadic(dtype):
    """L2-normalised non-negative rows with dyadic weights: 4 features of 0.5 or 16 features of 0.25 out of 60, so
    every score is a multiple of 1/16 (0.25, 0.5, 0.75, 1 ...) and exact in fp16, in 1/32768 units and in 2^-15
    units; some rows repeated (score exactly 1)."""
    rng = np.random.default_rng(12)
    rows = [(np.sort(rng.choice(60, 4, replace=False)), 0.5) for _ in range(3000)]
    rows += [(np.sort(rng.choice(60, 16, replace=False)), 0.25) for _ in range(500)]
    rows += rows[:200:7]
    rows = [rows[i] for i in rng.permutation(len(rows))]
    idx = np.concatenate([f for f, _ in rows])
    val = np.concatenate([np.full(len(f), w) for f, w in rows]).astype(dtype)
    return csr_matrix((val, idx, np.cumsum([0] + [len(f) for f, _ in rows])), shape=(len(rows), 60))


@pytest.mark.parametrize("dtype,cfg", [(np.float64, c) for c in CONFIGS] + [(np.float32, c) for c in CONFIGS_F32],
                         ids=["f64-" + _cfg_id(c) for c in CONFIGS] + ["f32-" + _cfg_id(c) for c in CONFIGS_F32])
def test_scores_exactly_on_the_threshold(monkeypatch, dtype, cfg):
    """scores equal to the threshold are out (strict >) on every path: the re-score, floorf(thr * 32768) of the
    16-bit tiles, the crossing test of the tile kernel, the selection; the next double below lets them in"""
    D = _D()
    m = _dyadic(dtype)
    A = D.DeviceCSR.from_scipy(m)
    table = RankedPairs(*exact_pairs(m, m, 0.2))
    kw, expect = _config(monkeypatch, cfg)
    expect.pop("tile_w", None)
    for s in (0.25, 0.5, 0.75, 1.0):
        for thr in (s, float(np.nextafter(s, -np.inf))):
            got, _ = _run(A, A, 10, thr, dict(expect, select=cfg[5]), **kw)
            assert_same(got, table.topn(10, thr), "%s thr=%r" % (_cfg_id(cfg), thr))
    assert len(table.topn(10, 0.75)[0]) < len(table.topn(10, np.nextafter(0.75, 0))[0])


# ---------------------------------------------------------------------------------------------------------------
# selection paths and ties
# ---------------------------------------------------------------------------------------------------------------
SIZES = (1, 31, 32, 33, 512, 513, 4096, 4097, 9000)
SEL_THR = 0.5


@pytest.fixture(scope="module")
def clusters():
    """Left: one base string per size m (and its three variants); right: per m, m rows that all score above SEL_THR
    with the base — half of them identical copies of it (exact ties), the rest three near-duplicates in turn (ties
    among their copies) — shuffled, so that tied columns interleave."""
    rng = np.random.default_rng(7)
    letters = np.array(list("ABCDEFGHIJKLMNOPQRSTUVWXYZ"))
    left, right = [], []
    for m in SIZES:
        base = "".join(rng.choice(letters, 30))
        variants = [base[:k] + "Z" + base[k + 1:] for k in (5, 15, 25)]
        left += [base] + variants
        n_id = (m + 1) // 2
        right += [base] * n_id + [variants[i % 3] for i in range(m - n_id)]
    right = [right[i] for i in rng.permutation(len(right))]
    m_left, m_right, _ = _P().tf_idf_matrices(left, right)
    table = RankedPairs(*exact_pairs(m_left, m_right, SEL_THR))
    counts = np.bincount(table.row, minlength=len(left))
    assert np.array_equal(counts[::4], SIZES), counts[::4]          # the base rows have exactly m survivors
    D = _D()
    return D.DeviceCSR.from_scipy(m_left), D.DeviceCSR.from_scipy(m_right), table, int(counts.max())


@pytest.mark.parametrize("mode", ["rows", "sort"])
def test_selection_paths_and_ties(clusters, monkeypatch, mode):
    """rows with 1 .. 9000 survivors against top_n on both sides of every path boundary: streaming warp (<= 32),
    warp network / one warp in shared memory (<= 512), one CTA (<= 4096) and in pieces of 4096 with the best top_n
    carried along (33 <= top_n <= 2048 with longer rows), and the three global sorts"""
    D = _D()
    A, B, table, longest = clusters
    monkeypatch.setattr(D, "SELECT_MODE", mode)
    for top_n in (1, 20, 31, 32, 33, 100, 512, 513, 2048, 2049, 4096):
        want_sel = "sort" if mode == "sort" or (top_n > 32 and longest > 4096 and top_n > 2048) else "rows"
        got, _ = _run(A, B, top_n, SEL_THR, {"select": want_sel, "kernel": "row", "acc": "u16"})
        assert_same(got, table.topn(top_n, SEL_THR), "select %s top_n=%d" % (mode, top_n))


# ---------------------------------------------------------------------------------------------------------------
# chunks, shards, odd shapes
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["row", "tiles"])
def test_row_chunks(scored, monkeypatch, kernel):
    D = _D()
    A, table, scores = scored[np.float64]
    monkeypatch.setattr(D, "CAND_CHUNK", 1 << 14)
    for thr in _thresholds(scores[::4]):
        got, st = _run(A, A, TOP_N, thr, {"kernel": kernel}, kernel=kernel)
        assert st["n_row_chunks"] > 1
        assert_same(got, table.topn(TOP_N, thr), "chunks %s thr=%r" % (kernel, thr))


@pytest.mark.parametrize("kernel", ["row", "tiles"])
def test_row_range_shards(scored, kernel):
    """row_begin / row_end (one rank's block of left rows): the exact result of those rows, absolute row ids"""
    A, table, scores = scored[np.float64]
    n = A.shape[0]
    for rb, re_ in ((0, 3001), (3001, 7777), (7777, n), (n - 5, n)):
        for thr in _thresholds(scores[1::5]):
            got, _ = _run(A, A, TOP_N, thr, {"kernel": kernel}, row_begin=rb, row_end=re_, kernel=kernel)
            assert_same(got, table.topn(TOP_N, thr, rows=(rb, re_)), "shard [%d, %d) thr=%r" % (rb, re_, thr))


@pytest.mark.parametrize("n_right", [1000, 100, 7])
@pytest.mark.parametrize("kernel", ["row", "tiles"])
def test_two_series_odd_shapes(kernel, n_right):
    """right sides that are not a multiple of the tile width, smaller than one tile, smaller than top_n"""
    D = _D()
    names = make_names(6000, seed=29)
    left = names[:3000]
    right = [names[i] for i in np.random.default_rng(n_right).choice(6000, n_right, replace=False)]
    m, d, _ = _P().tf_idf_matrices(left, right)
    A, B = D.DeviceCSR.from_scipy(m), D.DeviceCSR.from_scipy(d)
    for thr in (0.4, 0.6, 0.8):
        want = exact_topn(m, d, TOP_N, thr)
        assert len(want[0]) > 0
        got, _ = _run(A, B, TOP_N, thr, {"kernel": kernel}, kernel=kernel)
        assert_same(got, want, "%d right rows, thr=%r" % (n_right, thr))


# ---------------------------------------------------------------------------------------------------------------
# the operators (K2 through sparse_dot_topn_compat, K3) and K4
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("threshold,sort", [(None, True), (None, False), (0.0, True), (0.75, True), (0.75, False)])
def test_sp_matmul_topn_is_exact(dtype, threshold, sort):
    from parity import csr_triples
    from string_grouper_b200 import sparse_dot_topn_compat as C
    left = make_names(700, seed=31)
    right = make_names(400, seed=32) + left[:150]
    m, d, _ = _P().tf_idf_matrices(left, right, dtype=dtype)
    got = C.sp_matmul_topn(m, d.T, top_n=7, threshold=threshold, sort=sort)
    r, c, s = csr_triples(got)
    want = exact_topn(m, d, 7, -np.inf if threshold is None else threshold)
    assert got.dtype == dtype
    assert_same((r, c, s.astype(np.float64)), want[:3], "sp_matmul_topn(%r, sort=%r)" % (threshold, sort))


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_zip_is_exact(dtype):
    from scipy.sparse import random as sprandom
    from parity import csr_triples
    from string_grouper_b200 import sparse_dot_topn_compat as C
    rng = np.random.default_rng(4)
    blocks = []
    for w in (50, 1, 33, 120):
        b = sprandom(200, w, density=0.2, format="csr", random_state=rng, dtype=np.float64)
        b.data = np.round(b.data, 2)              # many exact ties, some exact zeros
        blocks.append(b.astype(dtype))
    for top_n in (1, 4, 300):
        got = C.zip_sp_matmul_topn(top_n, blocks)
        r, c, s = csr_triples(got)
        assert_same((r, c, s.astype(np.float64)), exact_zip(top_n, blocks)[:3], "zip top_n=%d" % top_n)


def test_symmetrize_is_exact():
    D = _D()
    P = _P()
    from parity import csr_triples
    names = make_names(4000, seed=5) + ["zz", ""]
    m, _, _ = P.tf_idf_matrices(names)
    A = D.DeviceCSR.from_scipy(m)
    for top_n, thr in ((3, 0.75), (20, 0.5)):
        M = D.cossim_topn(A, A, top_n, thr)
        want = exact_topn(m, m, top_n, thr)
        assert_same(M.host_triples() + (M.max_row,), want, "K2 before K4")
        ref = P.fix_diagonal_and_symmetrize(to_csr(want, m.shape[:1] * 2))
        assert_same(D.symmetrize(M).host_triples(), csr_triples(ref), "symmetrize top_n=%d" % top_n)

"""not-gpu: what the no-threshold mode of the top-n product rests on (DESIGN.md §4, `cossim_topn` with a threshold
<= 0 and the top-n floor), restated in numpy / scipy on the oracle's TF-IDF matrix.  The CUDA path is checked end to
end by tests/test_gpu_topn_nothreshold.py; this file pins the MATH on CPU.

  (1) every threshold <= 0 means "score > 0" for non-negative operands: exact_topn at 0.0, -0.25 and -inf agree
  (2) initial floor (topn_floor_init): the top_n-th best exact score of any 64 distinct columns, 0 when fewer than
      top_n of them score above the threshold, rounded down to fp32, never exceeds the row's exact top_n-th best
  (3) long rows (SG_FLOOR_LONG_ROWS): the block-max bound over ALL kept features, 32 at a time in fp16 with one
      rounding per feature (hfma2), left weights rounded up, plus 5e-4 per feature + 1e-4, never falls below the
      partial score over those features
"""
import numpy as np
import pytest
import scipy.sparse as sp

from exact_topn import assert_same, exact_topn
from oracle import pipeline as P
from synth_corpus import make_names

WINDOW = 64

LONG = ["international consolidated widget manufacturing holdings of north america incorporated",
        "the first national bank and trust company of greater south western pennsylvania",
        "associated independent wholesale grocers and food distributors cooperative association"]


def _matrix(dtype):
    names = make_names(2500, seed=21) + ["acme global holdings llc"] * 60 + LONG * 3 + [n + " ltd" for n in LONG]
    m, _, _ = P.tf_idf_matrices(names, dtype=dtype)
    m = sp.csr_matrix(m).astype(dtype)
    m.sort_indices()
    return m


@pytest.fixture(scope="module", params=[np.float64, np.float32], ids=["f64", "f32"])
def matrix(request):
    return _matrix(request.param)


def test_thresholds_at_or_below_zero_agree(matrix):
    m = matrix
    for top_n in (1, 20, 32):
        want = exact_topn(m, m, top_n, 0.0)
        assert want[3] == top_n and len(want[0]) >= m.shape[0]
        for thr in (-0.25, -np.inf):
            assert_same(exact_topn(m, m, top_n, thr), want, "top_n=%d thr=%r" % (top_n, thr))
    # two matrices of different widths
    left, right = m[100:1300], m[700:2801]
    assert_same(exact_topn(left, right, 20, -np.inf), exact_topn(left, right, 20, 0.0), "two matrices")


def _round_down_f32(x):
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f).astype(np.float64)


@pytest.mark.parametrize("top_n", [1, 20, 32])
def test_initial_floor_never_exceeds_the_exact_top_n_th_score(matrix, top_n):
    m = matrix
    n = m.shape[0]
    S = (m @ m.T).toarray().astype(np.float64)            # exact scores in the matrix dtype, widened
    nth = np.where((S > 0).sum(1) >= top_n, -np.sort(-S, axis=1)[:, top_n - 1], 0.0)
    rng = np.random.default_rng(top_n)
    checked = 0
    for r in range(0, n, 3):
        # any 64 distinct columns: random ones, the window around the row, and the row's own exact best 64
        for cols in (rng.choice(n, WINDOW, replace=False),
                     np.arange(WINDOW) + min(max(r - WINDOW // 2, 0), n - WINDOW),
                     np.argsort(-S[r], kind="stable")[:WINDOW]):
            s = S[r, cols]
            s = s[s > 0.0]
            kth = -np.sort(-s)[top_n - 1] if len(s) >= top_n else 0.0
            floor = _round_down_f32(np.array([kth]))[0]
            assert 0.0 <= floor <= nth[r], (r, floor, nth[r])
            checked += floor > 0
    assert checked > n // 3                               # most windows give a positive floor


def _fp16_up(x):
    """__float2half_ru as float64"""
    h = np.asarray(x, dtype=np.float64).astype(np.float16)
    return np.where(h.astype(np.float64) < x, np.nextafter(h, np.float16(np.inf)), h).astype(np.float64)


def _fp16_rn(x):
    return np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def _chunked_bound(a_up, f, maxw):
    """ub(t) as the kernel accumulates it for every tile t: ub = fp16(a_up * maxw[t, f] + ub), one rounding per kept
    feature in the stored order (the first 32 from registers, the later chunks of 32 loaded per 64-tile batch: the
    order of the additions is the same)"""
    ub = np.zeros(maxw.shape[0])
    for ak, fk in zip(a_up, f):
        ub = _fp16_rn(ak * maxw[:, fk] + ub)               # fp16 x fp16 + fp16 is exact in float64
    return ub


def _uniform_block(n_feat, n_rows, first_col):
    """n_rows rows of n_feat shared features of weight 1/sqrt(n_feat): every product and every sum rounds the same
    way, so the fp16 roundings add up"""
    w = np.full(n_feat, 1.0 / np.sqrt(n_feat))
    return [(np.arange(first_col, first_col + n_feat), w)] * n_rows


def test_chunked_block_max_bound_of_long_rows_never_falls_below_the_partial():
    m = _matrix(np.float64)
    rows = []
    col = m.shape[1]
    for nf in (33, 64, 65, 130, 400, 1000):
        rows += _uniform_block(nf, 3, col)
        col += nf
    u = sp.csr_matrix((np.concatenate([v for _, v in rows]), np.concatenate([c for c, _ in rows]),
                       np.cumsum([0] + [len(c) for c, _ in rows])), shape=(len(rows), col))
    m = sp.vstack([sp.hstack([m, sp.csr_matrix((m.shape[0], col - m.shape[1]))]), u]).tocsr()
    m.sort_indices()
    n = m.shape[0]
    nf = np.diff(m.indptr)
    long_rows = np.flatnonzero(nf > 32)
    assert len(long_rows) >= 30 and nf.max() == 1000
    # right rows in some processing order, 128-column tiles; the fp16 block maxima of the fp16 posting weights
    W = 128
    tile_of = np.empty(n, np.int64)
    tile_of[np.random.default_rng(4).permutation(n)] = np.arange(n) // W
    T = int(tile_of.max()) + 1
    coo = m.tocoo()
    w32 = coo.data.astype(np.float32).astype(np.float64)
    maxw = np.zeros((T, m.shape[1]))
    np.maximum.at(maxw, (tile_of[coo.row], coo.col), _fp16_rn(w32))
    Mt = m.T.tocsr()
    M16 = sp.csr_matrix((_fp16_rn(w32), coo.col, m.indptr), shape=m.shape).T.tocsr()
    shortfall = 0.0
    for r in long_rows:
        lo, hi = m.indptr[r], m.indptr[r + 1]
        f, a = m.indices[lo:hi], m.data[lo:hi]
        a32 = a.astype(np.float32).astype(np.float64)
        ub = _chunked_bound(_fp16_up(a32), f, maxw)[tile_of]
        row = sp.csr_matrix((a, f, [0, len(f)]), shape=(1, m.shape[1]))
        exact = np.asarray((row @ Mt).todense()).ravel()            # x_S . y over all kept features
        fp16w = np.asarray((row @ M16).todense()).ravel()           # the same with the fp16 posting weights
        need = np.maximum(exact, fp16w)
        assert np.all(ub + 5e-4 * len(f) + 1e-4 >= need), (r, len(f), (need - ub).max())
        shortfall = max(shortfall, (need - ub).max())
    # the slack is needed: on the uniform rows of 400 and 1000 features the fp16 sum alone falls 0.02 short
    assert shortfall > 0.01, shortfall

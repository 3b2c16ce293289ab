"""not-gpu: the inequality the top-n floor of K2 rests on (csrc/sg_cossim.cu, cossim_candidates_floor_kernel), restated
in numpy on the oracle's TF-IDF matrix.  The CUDA path is checked end to end by tests/test_gpu_topn_floor.py; this file
pins the MATH, so that a change of the margins that breaks exactness fails on CPU already.

  (1) lower bound:  p^(r, c) - E_r <= exact(r, c)   for every pair, E_r = CAND_MARGIN + margin_pf * (kept features)
      p^ = the partial score over the kept features as the kernel accumulates it: fp32 left weights times fp16
      posting weights, each product rounded to 1/32768 (u16 tiles, margin_pf = U16_MARGIN_PER_FEATURE) or added in
      fp32 (f32 tiles, margin_pf = 0)
  (2) the floor (top_n-th best of p^ - E_r, rounded down) never exceeds the exact top_n-th best score, and every pair
      of the exact top n passes the candidate test  p^ + |x_P| |y_H| > floor - E_r - FLOOR_EPS
"""
import numpy as np
import scipy.sparse as sp

from oracle import pipeline as P
from synth_corpus import make_names
from test_bounds_math import N_HEAVY, _prune

CAND_MARGIN, U16_PF, FLOOR_EPS, TOP_N = 1.5e-3, 2e-5, 1e-6, 20
UNIFORM = (116, 134, 300, 660, 1000)


def _uniform_rows(first_col):
    """two identical rows per n: n private features of weight 1/sqrt(n).  Every product rounds the same way (the fp16
    weight and the fixed-point product), so the roundings add up instead of cancelling"""
    rows, col = [], first_col
    for n in UNIFORM:
        for _ in range(2):
            rows.append((np.arange(col, col + n), np.full(n, 1.0 / np.sqrt(n))))
        col += n
    return rows, col


def _matrix():
    names = make_names(3000, seed=13) + ["acme global holdings llc"] * 40
    m, _, _ = P.tf_idf_matrices(names)
    m = m.tocsr()
    rows, n_cols = _uniform_rows(m.shape[1])
    u = sp.csr_matrix((np.concatenate([v for _, v in rows]), np.concatenate([c for c, _ in rows]),
                       np.cumsum([0] + [len(c) for c, _ in rows])), shape=(len(rows), n_cols))
    m = sp.vstack([sp.hstack([m, sp.csr_matrix((m.shape[0], n_cols - m.shape[1]))]), u]).tocsr()
    m.sort_indices()
    return m


def _setup():
    A = _matrix()
    df = np.bincount(A.indices, minlength=A.shape[1])
    heavy = np.zeros(A.shape[1], bool)
    heavy[np.argsort(-df, kind="stable")[:N_HEAVY]] = True
    S, xp = _prune(A, df, heavy)
    AH = sp.csr_matrix((A.data * heavy[A.indices], A.indices.copy(), A.indptr.copy()), shape=A.shape)
    y_heavy = np.sqrt(np.asarray(AH.multiply(AH).sum(axis=1)).ravel())
    return A, S, xp, y_heavy


def _partials(S, A, rows):
    """(u16 p^, f32 p^) of rows x all columns as the kernel accumulates them, dense [len(rows), n]"""
    W16 = A.astype(np.float32).tocsr()
    W16.data = W16.data.astype(np.float16).astype(np.float32)            # fp16 posting weights
    Wt = W16.T.tocsr()
    out_u16 = np.zeros((len(rows), A.shape[0]))
    out_f32 = np.zeros((len(rows), A.shape[0]), dtype=np.float32)
    for k, r in enumerate(rows):
        lo, hi = S.indptr[r], S.indptr[r + 1]
        f, a = S.indices[lo:hi], S.data[lo:hi].astype(np.float32)
        for fk, ak in zip(f, a):
            lo2, hi2 = Wt.indptr[fk], Wt.indptr[fk + 1]
            cols, w = Wt.indices[lo2:hi2], Wt.data[lo2:hi2]
            out_u16[k, cols] += np.rint((ak * np.float32(32768.0)) * w)          # fp32 product, rounded to an integer
            out_f32[k, cols] += ak * w                                            # fp32 products and sums
    return out_u16 / 32768.0, out_f32.astype(np.float64)


def test_partial_minus_margin_is_a_lower_bound_of_the_exact_score():
    A, S, xp, _ = _setup()
    n = A.shape[0]
    rng = np.random.default_rng(3)
    rows = np.r_[rng.choice(n - 2 * len(UNIFORM), 300, replace=False), np.arange(n - 2 * len(UNIFORM), n)]
    exact = (A[rows] @ A.T).toarray()
    kept = np.diff(S.indptr)[rows]
    p16, p32 = _partials(S, A, rows)
    for p, pf in ((p16, U16_PF), (p32, 0.0)):
        lb = p - (CAND_MARGIN + pf * kept)[:, None]
        assert np.all(lb <= exact), (lb - exact).max()
    # the uniform rows: every rounding goes up, so p^ exceeds the exact score (the bound is needed in this direction)
    u0 = n - 2 * len(UNIFORM)
    over = []
    for k in range(len(rows) - 2 * len(UNIFORM), len(rows)):
        partner = u0 + ((rows[k] - u0) ^ 1)
        over.append(p16[k, partner] - exact[k, partner])
    assert max(over) > 2e-4, over                                  # far more than the rounding of a single product


def test_floor_never_drops_a_pair_of_the_exact_top_n():
    A, S, xp, y_heavy = _setup()
    n = A.shape[0]
    rows = np.r_[np.arange(0, n, 11), np.arange(n - 2 * len(UNIFORM) - 40, n)]
    rows = np.unique(rows)
    exact = (A[rows] @ A.T).toarray()
    kept = np.diff(S.indptr)[rows]
    p16, p32 = _partials(S, A, rows)
    threshold = 0.05
    for p, pf in ((p16, U16_PF), (p32, 0.0)):
        e = (CAND_MARGIN + pf * kept).astype(np.float32)
        reported = p > 0
        lb = np.where(reported, np.maximum((p.astype(np.float32) - e[:, None]).astype(np.float64), 0.0), 0.0)
        floor = -np.sort(-lb, axis=1)[:, TOP_N - 1]
        floor = np.nextafter(floor.astype(np.float32), np.float32(-np.inf)).astype(np.float64)   # rounded down
        floor = np.maximum(floor, 0.0)
        nth = -np.sort(-exact, axis=1)[:, TOP_N - 1]
        assert np.all(floor <= nth)
        assert (floor > threshold).mean() > 0.3                     # the floor has teeth: most rows rise above 0.05
        # every pair of the exact top n (score > threshold, rank < TOP_N by score desc, column desc) stays a candidate
        thr_floor = floor - e - FLOOR_EPS
        for k in range(len(rows)):
            s = exact[k]
            order = np.lexsort((-np.arange(n), -s))[:TOP_N]
            top = order[s[order] > threshold]
            assert np.all(p[k, top] + xp[rows[k]] * y_heavy[top] > thr_floor[k]), rows[k]

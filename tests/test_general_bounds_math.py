"""not-gpu: the candidate stage's approximations on general operands (rows of any norm, signed weights, weights below
fp16's range, unbalanced norms), restated in numpy as the kernels compute them (csrc/sg_cossim.cu, csrc/sg_tiles.cu):

  * posting weight  fp16 rn of fp32(v) * w_scale; a nonzero weight below fp16's range becomes +-2^-24
  * block maxima    the largest |posting| of a (feature, tile), fp16
  * left weight     fp16 ru of |fp32(a) * a_scale * b_scale| for the bound, fp32(a) * a_scale for the partial
  * bound           one hfma2 rounding per kept feature, tested as ub + (5e-4 nf + 1e-4) > thr_c * b_scale
  * thr_c           max(threshold - CAND_MARGIN * max(1, scale), 0)
  * u16 / tiles     products rounded to 2^-15 units, admitted by _device.fixed_point_ok

The scales and the admission rule are the library's own (_device.candidate_scales, _device.fixed_point_ok), so a change
of those rules that breaks exactness fails here, without a GPU.  Exactness rests on:

  (a) for a pair of score s and a threshold just below s, the block-max bound of its tile passes the test;
  (b) with non-negative operands every pair of positive score has a positive partial score (what thr_c = 0 needs);
  (c) the partial score is within the candidate margin of s (fp32 accumulator), or within the margin plus the
      per-feature margin (fixed-point accumulators).

PARENT states the rules these replaced; test_parent_rules_lose_pairs shows that the properties catch them.
"""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp

from exact_topn import exact_pairs
from string_grouper_b200 import _device as D

F16_TINY = 2.0 ** -24


def _fixed_scales(norm_a, norm_b):
    return D.candidate_scales(norm_a, norm_b)


def _fixed_admit(A, B):
    return D.fixed_point_ok(A, B)


FIXED = {"scales": _fixed_scales, "admit": _fixed_admit, "round_up": True}
PARENT = {"scales": lambda na, nb: (1.0 / max(nb, 1.0), max(nb, 1.0), 1.0),
          "admit": lambda A, B: A.nonneg and B.nonneg and A.norm_bound * B.norm_bound <= 1.0 + 1e-6,
          "round_up": False}


# ---------------------------------------------------------------------------------------------------------------
# the kernels' arithmetic
# ---------------------------------------------------------------------------------------------------------------
def _half_up(x):
    """fp16 rounded towards +inf (__float2half_ru) of non-negative x, as float64"""
    x = np.asarray(x, dtype=np.float64)
    with np.errstate(over="ignore"):
        h = x.astype(np.float16)
    low = h.astype(np.float64) < x
    return np.where(low, np.nextafter(h, np.float16(np.inf)), h).astype(np.float64)


def _postings(v32, w_scale, round_up):
    x = (v32 * np.float32(w_scale)).astype(np.float32)
    with np.errstate(over="ignore", under="ignore"):
        h = x.astype(np.float16)
    if round_up:
        h = np.where((x != 0) & (np.abs(x) < F16_TINY), np.copysign(np.float16(F16_TINY), x), h).astype(np.float16)
    return h


def _side(m):
    """what DeviceCSR.from_scipy keeps on the host: the fp32 copy, the norm bound and the sign flag"""
    m = sp.csr_matrix(m)
    m.sum_duplicates()
    nb = float(np.sqrt(m.multiply(m).sum(axis=1).max())) if m.nnz else 1.0
    return SimpleNamespace(m=m, m32=m.astype(np.float32), norm_bound=max(nb, 1e-30),
                           nonneg=bool(m.nnz == 0 or m.data.min() >= 0))


class Model:
    """candidate-stage quantities of every pair (i, j) with a nonzero exact score, each right row its own column tile
    (the tightest block maxima: any real tile's are at least as large)"""

    def __init__(self, Am, Bm, rules):
        self.A, self.B = _side(Am), _side(Bm)
        A, B = self.A, self.B
        self.scale = A.norm_bound * B.norm_bound
        self.margin = D.CAND_MARGIN * max(self.scale, 1.0)
        w_scale, a_scale, b_scale = rules["scales"](A.norm_bound, B.norm_bound)
        self.w_scale, self.a_scale, self.b_scale = (np.float32(x) for x in (w_scale, a_scale, b_scale))
        self.post = sp.csr_matrix((_postings(B.m32.data, w_scale, rules["round_up"]).astype(np.float64),
                                   B.m.indices, B.m.indptr), shape=B.m.shape)
        self.admit = rules["admit"](A, B)
        r, c, s = exact_pairs(A.m, B.m, -np.inf)
        self.row, self.col, self.score = r, c, s

    def left(self, i):
        lo, hi = self.A.m.indptr[i], self.A.m.indptr[i + 1]
        f = self.A.m.indices[lo:hi]
        a = (self.A.m32.data[lo:hi] * self.a_scale).astype(np.float32)
        return f, a

    def dense_right(self, cols, f):
        """posting weights (fp16 values as float64) of right rows `cols` on features f, 0 where absent"""
        return np.asarray(self.post[cols][:, f].todense())

    def bound(self, i, cols):
        """ub + slack (fp32) of row i against the single-row tiles `cols`, and the slack"""
        f, a = self.left(i)
        an = _half_up(np.abs((a * self.b_scale).astype(np.float32)))
        W = np.abs(self.dense_right(cols, f))
        ub = np.zeros(len(cols), dtype=np.float16)
        with np.errstate(over="ignore", invalid="ignore"):
            for k in range(len(f)):
                ub = (an[k] * W[:, k] + ub.astype(np.float64)).astype(np.float16)
        slack = np.float32(5e-4) * np.float32(len(f)) + np.float32(1e-4)
        return ub.astype(np.float32) + slack

    def partial(self, i, cols):
        """fp32 accumulator: every product rounded to fp32, then added"""
        f, a = self.left(i)
        W = self.dense_right(cols, f)
        acc = np.zeros(len(cols), dtype=np.float32)
        for k in range(len(f)):
            acc = (acc + (a[k] * W[:, k].astype(np.float32)).astype(np.float32)).astype(np.float32)
        return acc

    def partial_u16(self, i, cols):
        """16-bit fixed point: every product rounded once to 2^-15 units (Ops::atomic_add)"""
        f, a = self.left(i)
        a_fix = (a * np.float32(32768)).astype(np.float32)
        W = self.dense_right(cols, f).astype(np.float32)
        return np.rint((a_fix[None, :] * W).astype(np.float32)).sum(axis=1) / 32768.0

    def partial_tiles(self, i, cols):
        """tile kernel: both weights rounded to 2^-15 units (pack_left, tile build), products in 2^-30 units"""
        f, _ = self.left(i)
        lo, hi = self.A.m.indptr[i], self.A.m.indptr[i + 1]
        a = np.maximum(self.A.m32.data[lo:hi] * np.float32(max(self.B.norm_bound, 1.0)), 0).astype(np.float32)
        aq = np.rint((a * np.float32(32768)).astype(np.float32))
        Bw = np.asarray(self.B.m32[cols][:, f].todense()).astype(np.float32)
        wq = np.rint((Bw * np.float32(1.0 / max(self.B.norm_bound, 1.0)) * np.float32(32768)).astype(np.float32))
        return (aq[None, :] * wq).sum(axis=1) / 2.0 ** 30

    def by_row(self):
        for i in np.unique(self.row):
            sel = np.flatnonzero(self.row == i)
            yield i, sel


def violations(model, prop):
    """pairs (i, j) of the model that break property `prop` ("a", "b", "c", "u16", "tiles")"""
    bad = []
    for i, sel in model.by_row():
        cols, s = model.col[sel], model.score[sel]
        if prop == "a":
            thr = np.nextafter(s, -np.inf)
            thr_c = np.maximum(thr - model.margin, 0.0).astype(np.float32)
            ok = model.bound(i, cols) > (thr_c * model.b_scale).astype(np.float32)
            ok |= s <= 0
        elif prop == "b":
            ok = (s <= 0) | (model.partial(i, cols) > 0)
        elif prop == "c":
            ok = model.partial(i, cols).astype(np.float64) > s - model.margin
        else:
            nf = model.A.m.indptr[i + 1] - model.A.m.indptr[i]
            if prop == "u16":
                got, room = model.partial_u16(i, cols), model.margin + nf * D.U16_MARGIN_PER_FEATURE
            else:
                got = model.partial_tiles(i, cols)
                room = D.TILE_MARGIN * max(model.scale, 1.0) + nf * D.TILE_MARGIN_PER_FEATURE
            ok = np.abs(got - s) <= room
        bad += [(int(i), int(c)) for c in cols[~ok]]
    return bad


# ---------------------------------------------------------------------------------------------------------------
# operand families (seeded)
# ---------------------------------------------------------------------------------------------------------------
def _tfidf(n=400, seed=3):
    from oracle import pipeline as P
    from synth_corpus import make_names
    m, _, _ = P.tf_idf_matrices(make_names(n, seed=seed))
    return m.tocsr()


def _rows(rows, n_cols, dtype=np.float64):
    """CSR from [(indices, values), ...]"""
    ind = [np.asarray(c, dtype=np.int64) for c, _ in rows]
    val = [np.asarray(v, dtype=np.float64) for _, v in rows]
    return sp.csr_matrix((np.concatenate(val).astype(dtype), np.concatenate(ind), np.cumsum([0] + [len(c) for c in ind])),
                         shape=(len(rows), n_cols))


def _uniform(norm, n, col=0):
    """two identical rows of n equal weights at the given norm: every rounding goes the same way"""
    row = (np.arange(col, col + n), np.full(n, norm / math.sqrt(n)))
    return [row, row]


def family(name):
    """(A, B) of a family; A is B for self-products"""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name in ("scaled", "scaled_f32"):
        m = _tfidf()
        m = sp.diags(10.0 ** rng.uniform(-3, 3, size=m.shape[0])) @ m
        m = m.tocsr().astype(np.float32 if name == "scaled_f32" else np.float64)
        return m, m
    if name.startswith("uniform_"):
        rows = []
        col = 0
        for n in (16, 29, 40):
            rows += _uniform(float(name[8:]), n, col)
            col += n
        m = _rows(rows, col)
        return m, m
    if name == "counts":
        V = 400
        rows = []
        for k in range(160):
            nf = int(rng.choice([1, 2, 5, 12, 40, 80, 200]))
            rows.append((np.sort(rng.choice(V, size=nf, replace=False)), rng.integers(1, 501, size=nf)))
        rows.append(([7], [300]))                                     # one entry of 300 against a right side of norm 300
        rows.append(([7, 8], [300, 1]))
        m = _rows(rows, V)
        return m, m
    if name == "tiny":
        m = _tfidf(300)
        V = m.shape[1]
        tiny = []
        for k in range(60):
            r = m[k]
            v = 10.0 ** rng.uniform(-12, -9, size=r.nnz)
            tiny.append((r.indices, v))
        t = _rows(tiny, V)
        m = sp.vstack([m, t]).tocsr()
        return m, m
    if name == "unbalanced":
        # plus one pair of single-feature rows whose 2^-15 roundings both go up by nearly 2^-16: 6.5e-5 at |a| = 4
        m = _tfidf(300)
        V = m.shape[1]
        m = sp.hstack([m, sp.csr_matrix((m.shape[0], 1))]).tocsr()
        a = _rows([([V], [131071.5001 / 32768])], V + 1)
        w = _rows([([V], [8191.5001 / 32768])], V + 1)
        return sp.vstack([4.0 * m, a]).tocsr(), sp.vstack([0.25 * m, w]).tocsr()
    if name == "unbalanced_far":
        m = _tfidf(300)
        rows = _uniform(1.0, 24, m.shape[1])
        u = _rows(rows, m.shape[1] + 24)
        m = sp.vstack([sp.hstack([m, sp.csr_matrix((m.shape[0], 24))]), u]).tocsr()
        return (1e5 * m).tocsr(), (1e-5 * m).tocsr()
    if name == "signed":
        m = _tfidf(300).copy()
        m.data[rng.random(m.nnz) < 0.2] *= -1
        return m, m
    if name == "long":
        V = 600
        rows = [(np.sort(rng.choice(V, size=nf, replace=False)), rng.uniform(0.1, 1.0, size=nf))
                for nf in (33, 64, 65, 120, 200, 200, 1)]
        m = _rows(rows, V)
        m = sp.diags(1.0 / np.sqrt(m.multiply(m).sum(axis=1).A.ravel())) @ m
        return m.tocsr(), m.tocsr()
    raise KeyError(name)


FAMILIES = ["scaled", "scaled_f32", "uniform_3", "uniform_10", "uniform_100", "uniform_1e4", "uniform_1e-6", "counts", "tiny", "unbalanced", "unbalanced_far", "signed", "long"]
NONNEG = [f for f in FAMILIES if f != "signed"]


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(name, rules=FIXED):
        key = (name, id(rules))
        if key not in cache:
            cache[key] = Model(*family(name), rules)
        return cache[key]
    return get


@pytest.mark.parametrize("name", FAMILIES)
def test_block_max_bound_passes_every_pair_at_its_own_score(models, name):
    """(a): norms 1e-6 .. 1e4, 1 .. 200 features, uniform rows, raw counts of up to 500"""
    m = models(name)
    assert len(m.score) > 10
    assert violations(m, "a") == []


@pytest.mark.parametrize("name", NONNEG)
def test_positive_scores_have_positive_partials(models, name):
    """(b): what a candidate threshold of 0 (thresholds below the margin) needs, weights down to 1e-12 included"""
    assert violations(models(name), "b") == []


@pytest.mark.parametrize("name", FAMILIES)
def test_partial_score_within_the_candidate_margin(models, name):
    """(c) for the fp32 accumulator"""
    assert violations(models(name), "c") == []


@pytest.mark.parametrize("name", FAMILIES)
def test_fixed_point_paths_only_where_their_margins_hold(models, name):
    """(c) for the u16 accumulator and the tile kernel, on the operands fixed_point_ok admits"""
    m = models(name)
    if not m.admit:
        return
    assert violations(m, "u16") == []
    assert violations(m, "tiles") == []


def test_fixed_point_admission():
    A, B = _side(family("unbalanced")[0]), _side(family("unbalanced")[1])
    assert not D.fixed_point_ok(A, B)
    n = _side(_tfidf())
    assert D.fixed_point_ok(n, n)
    # L2-normalised rows: the kernels receive exactly 1 (fp32) for every scale
    assert all(np.float32(x) == 1 for x in D.candidate_scales(n.norm_bound, n.norm_bound))
    assert D.candidate_scales(1.0, 1.0) == (1.0, 1.0, 1.0)


@pytest.mark.parametrize("item,name,prop", [
    ("NaN bound of large weights", "counts", "a"),
    ("absolute slack", "uniform_10", "a"),
    ("posting weights underflow", "tiny", "b"),
    ("posting scale of unbalanced norms", "unbalanced_far", "c"),
    ("tile margin of unbalanced norms", "unbalanced", "tiles"),
])
def test_parent_rules_lose_pairs(models, item, name, prop):
    """the rules these replaced break the properties above on the families that exercise them"""
    m = models(name, PARENT)
    if prop == "tiles":
        assert m.admit
    assert violations(m, prop), item


# ---------------------------------------------------------------------------------------------------------------
# the reference: scipy's product is the ascending-feature sum without FMA, for general values too
# ---------------------------------------------------------------------------------------------------------------
def _sequential(a_idx, a_val, b_idx, b_val, dtype):
    common, ia, ib = np.intersect1d(a_idx, b_idx, assume_unique=True, return_indices=True)
    acc = dtype(0)
    for i, j in zip(ia, ib):
        acc = dtype(acc + dtype(a_val[i] * b_val[j]))
    return acc


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["scaled", "counts", "tiny", "signed", "unbalanced_far"])
def test_reference_is_the_ascending_sum_without_fma(name, dtype):
    A, B = family(name)
    A, B = A.astype(dtype).tocsr(), B.astype(dtype).tocsr()
    r, c, s = exact_pairs(A, B, -np.inf)
    assert len(r) > 50
    pick = np.random.default_rng(4).choice(len(r), size=min(len(r), 1500), replace=False)
    for k in pick:
        a, b = A[r[k]], B[c[k]]
        assert float(_sequential(a.indices, a.data, b.indices, b.data, dtype)) == s[k], (name, k)

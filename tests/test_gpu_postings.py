"""-m gpu: the right matrix's bucketed postings (sg_postings_build) against the same directory stated in numpy, for
every (feature, tile) bucket: its length, the multiset of {column in tile, fp16 weight} in its posting range, the fp16
maximum in the directory and in the block-maxima rows, and zeros for the empty buckets and the padding tiles."""
import numpy as np
import pytest
import scipy.sparse as sp

from synth_corpus import make_names

pytestmark = pytest.mark.gpu

SMEM_CAP = 8192     # postings of a tile sorted in shared memory (PB_CAP in csrc/sg_cossim.cu); larger tiles spill


def _expected(m, perm, W, w_scale):
    """(bucket id f*T + t, posting u32) of every stored value, in the processing order perm (position -> row)."""
    m = m.tocsr()
    n = m.shape[0]
    T = max(-(-n // W), 1)
    pos = np.empty(n, dtype=np.int64)
    pos[perm] = np.arange(n)
    lens = np.diff(m.indptr)
    p = np.repeat(pos, lens)
    t = p // W
    x = m.data.astype(np.float32) * np.float32(w_scale)
    w = x.astype(np.float16)                                                     # fp32 product, RN to fp16
    # a nonzero weight that rounds to zero keeps its sign and becomes the smallest subnormal
    w = np.where((w == 0) & (x != 0), np.copysign(np.float16(2.0 ** -24), x), w).astype(np.float16)
    post = (w.view(np.uint16).astype(np.uint32) << 16) | (p - t * W).astype(np.uint32)
    return m.indices.astype(np.int64) * T + t, post, T


def _check(m, W, perm=None):
    import torch
    from string_grouper_b200 import _device as D
    B = D.DeviceCSR.from_scipy(m)
    D.right_order(B)                        # the heavy norms the tile bounds need
    n, V = m.shape
    perm = np.random.default_rng(W).permutation(n).astype(np.int32) if perm is None else perm
    spilled = torch.zeros(1, dtype=torch.int32, device=B.device)
    bdir, bmaxw, post, T, _ = D._build_postings(B, torch.from_numpy(perm).to(B.device), W, spilled)
    V1, Tp = V + 1, bmaxw.numel() // (V + 1)
    assert Tp % 64 == 0 and Tp >= T
    d = bdir.cpu().numpy().reshape(V1 * T, 2)
    maxw = bmaxw.cpu().numpy().view(np.uint16).reshape(V1, Tp)
    gpost = post.cpu().numpy().view(np.uint32)[:m.nnz]

    b, epost, T_np = _expected(m, perm, W, D.candidate_scales(1.0, B.norm_bound)[0])
    assert T == T_np
    elen = np.bincount(b, minlength=V1 * T)
    emax = np.zeros(V1 * T, dtype=np.uint32)
    np.maximum.at(emax, b, (epost >> 16) & 0x7fff)
    start, glen, gmax = d[:, 0].astype(np.int64), d[:, 1] & 0xffff, (d[:, 1].view(np.uint32) >> 16)
    assert np.array_equal(glen, elen)
    assert np.array_equal(gmax, emax)
    assert np.array_equal(maxw[:, :T].reshape(-1), emax.astype(np.uint16))
    assert not maxw[:, T:].any()                                  # padding tiles
    assert not start[elen == 0].any() and not d[elen == 0].any()  # empty buckets: all zero
    # the posting ranges of the buckets tile [0, nnz) without overlap and hold exactly the bucket's postings
    ne = np.flatnonzero(elen)
    order = ne[np.argsort(start[ne], kind="stable")]
    assert start[order[0]] == 0 and np.array_equal(start[order[1:]], (start + elen)[order[:-1]])
    assert start[order[-1]] + elen[order[-1]] == m.nnz
    gb = np.repeat(ne, elen[ne])
    gp = gpost[np.repeat(start[ne], elen[ne]) + np.arange(m.nnz) - np.repeat(np.cumsum(elen[ne]) - elen[ne], elen[ne])]
    g = np.lexsort((gp, gb))
    e = np.lexsort((epost, b))
    assert np.array_equal(gb[g], b[e]) and np.array_equal(gp[g], epost[e])
    tile_nnz = np.bincount(b % T, minlength=T)
    assert int(spilled.item()) == int((tile_nnz > SMEM_CAP).sum())
    return int(spilled.item())


@pytest.mark.parametrize("W", [128, 256])
def test_corpus_in_processing_order(W):
    from oracle import pipeline as P
    from string_grouper_b200 import _device as D
    m, _, _ = P.tf_idf_matrices(make_names(3000, seed=5))       # 24 / 12 tiles: T is not a multiple of 64
    B = D.DeviceCSR.from_scipy(m)
    perm = D.right_order(B)[1].cpu().numpy()
    assert _check(m, W, perm) == 0


@pytest.mark.parametrize("W", [128, 256])
def test_empty_rows_and_a_feature_in_every_tile(W):
    rng = np.random.default_rng(7)
    m = sp.random(1000, 300, density=0.04, format="lil", random_state=rng, dtype=np.float64)
    m[::3] = 0                                  # empty rows
    m[::5, 17] = 0.25                           # a feature in every tile ...
    m[W:2 * W] = 0                              # ... but the second, which holds no posting at all
    m = m.tocsr()
    m.eliminate_zeros()
    assert _check(m, W, np.arange(1000, dtype=np.int32)) == 0


def test_fp16_subnormal_weights_and_weights_below_fp16():
    """weights in fp16's subnormal range, and below it: those keep their sign as the smallest subnormal (2^-24)"""
    rng = np.random.default_rng(8)
    m = sp.random(700, 200, density=0.05, format="csr", random_state=rng, dtype=np.float64)
    m.data *= 10.0 ** rng.integers(-9, 0, size=m.nnz)           # below 6.1e-5 is subnormal, below 3e-8 zero in fp16
    m.data[::7] *= -1
    assert (np.abs(m.data) < 6.1e-5).sum() > 100 and (np.abs(m.data) * 4 < 2.0 ** -25).sum() > 100
    assert _check(m, 128) == 0


def test_tiles_too_large_for_shared_memory():
    rng = np.random.default_rng(9)
    # long rows: 256-row tiles of ~45 postings per row (> SMEM_CAP in most tiles) next to short ones
    n, V = 3000, 2000
    lens = np.where(np.arange(n) < 2000, 45, 6)
    cols = [np.sort(rng.choice(V, size=k, replace=False)) for k in lens]
    m = sp.csr_matrix((rng.random(lens.sum()) + 1e-3, np.concatenate(cols), np.r_[0, np.cumsum(lens)]), shape=(n, V))
    assert _check(m, 256, np.arange(n, dtype=np.int32)) >= 7
    assert _check(m, 256) > 0                                   # spilled and in-memory tiles mixed by a permutation
    # one feature in every row of a 16384-row tile: a bucket of 16384 postings
    n = 18000
    m2 = sp.random(n, 500, density=0.004, format="lil", random_state=rng, dtype=np.float64)
    m2[:, 3] = 0.5
    assert _check(m2.tocsr(), 16384) == 1

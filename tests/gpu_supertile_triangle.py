"""Ad-hoc (GPU box): what super-tile block maxima would save the candidates kernel on the benchmark's dedup triangle.

    python tests/gpu_supertile_triangle.py [N] [--sample ROWS]

The benchmark's self-match runs on U = unique_rows(A) of make_names(N, 0), over the triangle: a row tests the 64-tile
batches from the one holding its own position on.  For a sample of U's rows (spread over the processing order) and
S = 8 and 16, this states in torch what the block-max test does, with every kept feature (rows of more than 32 too):
  * the share of the triangle's super-tiles whose coarse bound (max of the S block maxima, max of the S tile bounds)
    can reach the row's threshold, and the share of tiles that survive the fine test;
  * the block-maxima bytes per row and kept feature of the test as it is (one 128-byte row per 64-tile batch) and of a
    coarse pass (the group's super-tiles, 64 per warp load, whole 32-byte sectors) followed by the fine test of only
    the sectors of surviving super-tiles, in batches that hold one;
  * the rows that keep more than 32 features.
Sums over fp32 instead of the kernel's fp16: close enough for shares, and the coarse bound still covers the fine one."""
import argparse
import os
import sys

import numpy as np
import pandas as pd
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE)]

from synth_corpus import make_names  # noqa: E402
from string_grouper_b200 import _device as D, _ingest  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("n", nargs="?", type=int, default=663_000)
ap.add_argument("--sample", type=int, default=16384)
ap.add_argument("--thr", type=float, default=0.8)
args = ap.parse_args()

names = make_names(args.n, 0)
data, offsets, flags, _ = _ingest.pack_strings([pd.Series(names)])
A, _, _ = D.tfidf(data, offsets, args.n, 3, flags, np.float64)
U = D.unique_rows(A)
m = U.shape[0]
tile_w, _ = D.pick_tile(m, None, None, 2, n_left=m)
hrank, perm, rank, bdir, maxw, post, T, tile_bound = D.right_side(U, tile_w)
W = tile_w
V1 = U.shape[1] + 1
Tp = maxw.numel() // V1
maxw = maxw.view(V1, Tp)[:, :T].float()
tpg = max(64, int(D.GROUP_BYTES // max(4 * U.nnz / T, 1)) // 64 * 64)
l_idx, l_val, l_len, l_thr, l_xp, _ = D.prune_left(U, U, hrank, 0, m, args.thr, D.CAND_MARGIN,
                                                   D.U16_MARGIN_PER_FEATURE, D.PRUNE_FRAC)
scale = 1.0 / max(U.norm_bound, 1.0)
dev = maxw.device
tb = tile_bound[:T]
nf_all = l_len.long()
print("U: %d rows, V = %d, nnz = %d; W = %d, T = %d, tiles per group = %d" % (m, U.shape[1], U.nnz, W, T, tpg))
print("rows of U keeping more than 32 features: %d (mean kept %.2f)" % (int((nf_all > 32).sum()), nf_all.float().mean()))

SS = (8, 16)
acc = {"rows": 0, "feat": 0, "tiles": 0, "tiles_live": 0, "bytes_now": 0.0}
for S in SS:
    acc[S] = {"st": 0, "st_live": 0, "bytes": 0.0}
R = 256
positions = torch.linspace(0, m - 1, args.sample, device=dev).long()
tiles = torch.arange(T, device=dev)
for b0 in range(0, positions.numel(), R):
    pos = positions[b0:b0 + R]
    rows = perm[pos].long()
    nf = nf_all[rows]
    K = int(nf.max())
    if K == 0:
        continue
    p0 = U.d_indptr[rows]
    kk = torch.arange(K, device=dev)
    ok = kk[None, :] < nf[:, None]
    idx = torch.where(ok, p0[:, None] + kk[None, :], torch.zeros_like(p0[:, None]))
    f = torch.where(ok, l_idx[idx].long(), torch.full_like(idx, V1 - 1))
    w = torch.where(ok, (l_val[idx] * scale).abs(), torch.zeros_like(idx, dtype=torch.float32))
    thr_r, xp = l_thr[rows], l_xp[rows]
    slack = 5e-4 * nf.float() + 1e-4
    # the triangle: tiles from the 64-tile batch holding the row's own position on
    t_first = (pos // W) & ~63
    in_tri = tiles[None, :] >= t_first[:, None]

    def survive(mw, bound):
        ub = torch.zeros(pos.numel(), mw.shape[1], device=dev)
        for k in range(K):
            ub += w[:, k:k + 1] * mw[f[:, k]]
        thr_t = (thr_r[:, None] - xp[:, None] * bound[None, :]).clamp(min=0)
        thr_t = torch.where(xp[:, None] > 0, thr_t, thr_r[:, None].expand_as(thr_t))
        return ub + slack[:, None] > thr_t

    fine = survive(maxw, tb) & in_tri & (nf[:, None] > 0)
    live_rows = nf > 0
    nfl = nf.float()
    acc["rows"] += int(live_rows.sum())
    acc["feat"] += float(nfl.sum())
    acc["tiles"] += int(in_tri[live_rows].sum())
    acc["tiles_live"] += int(fine.sum())
    # now: one 128-byte row of block maxima per kept feature and 64-tile batch of the triangle
    n_batches = (T - t_first + 63) // 64
    acc["bytes_now"] += float((n_batches.float() * 128 * nfl)[live_rows].sum())
    for S in SS:
        Ts = -(-T // S)
        pad = Ts * S - T
        mws = torch.nn.functional.pad(maxw, (0, pad)).view(V1, Ts, S).amax(2)
        bds = torch.nn.functional.pad(tb, (0, pad)).view(Ts, S).amax(1)
        st = torch.arange(Ts, device=dev)
        st_tri = (st[None, :] * S + S) > t_first[:, None]
        coarse = survive(mws, bds) & st_tri & (nf[:, None] > 0)
        truth = torch.nn.functional.pad(fine, (0, pad)).view(-1, Ts, S).any(2)
        assert bool((coarse | ~truth).all()), "a coarse bound fell below a fine one"
        e = acc[S]
        e["st"] += int(st_tri[live_rows].sum())
        e["st_live"] += int(coarse.sum())
        # coarse pass: per group, the super-tiles from the row's first batch, 2 bytes each, whole sectors, per 1024 tiles
        coarse_bytes = torch.zeros(pos.numel(), device=dev)
        for g0 in range(0, T, tpg):
            g1 = min(g0 + tpg, T)
            for s0 in range(g0, g1, 1024):
                s1 = min(s0 + 1024, g1)
                lo = torch.clamp(t_first, min=s0)
                n_st = ((s1 - lo).clamp(min=0) + S - 1) // S
                coarse_bytes += ((n_st * 2 + 31) // 32 * 32).float()
        # fine pass: the 32-byte sectors (16 tiles) of the batches that hold a surviving super-tile, only those that
        # hold one
        per_sector = 16 // S if S < 16 else 1
        sec_live = torch.nn.functional.pad(coarse, (0, (-Ts) % per_sector)).view(pos.numel(), -1, per_sector).any(2)
        if S > 16:
            sec_live = sec_live.repeat_interleave(S // 16, 1)
        fine_bytes = sec_live.sum(1).float() * 32
        e["bytes"] += float(((coarse_bytes + fine_bytes) * nfl)[live_rows].sum())

rows = acc["rows"]
print("sampled rows %d, kept features %.2f per row" % (rows, acc["feat"] / rows))
print("tiles of the triangle surviving the fine test: %.4f (%.1f per row)" % (
    acc["tiles_live"] / acc["tiles"], acc["tiles_live"] / rows))
print("block-maxima bytes per row now: %.0f" % (acc["bytes_now"] / rows))
for S in SS:
    e = acc[S]
    print("S=%2d: super-tiles surviving %.4f (%.1f per row); block-maxima bytes per row %.0f -> %.0f (%.1fx less)" % (
        S, e["st_live"] / e["st"], e["st_live"] / rows, acc["bytes_now"] / rows, e["bytes"] / rows,
        acc["bytes_now"] / max(e["bytes"], 1.0)))

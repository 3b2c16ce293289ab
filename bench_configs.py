#!/usr/bin/env python
"""The other BASELINE.json configurations (2, 4, 5; config 3 is bench.py) through the public API — absolute numbers beside
bench.py's line.

    python bench_configs.py --config 2                      # 100k self-match @0.8, 1 GPU
    torchrun --nproc-per-node 8 ... bench_configs.py --config 4   # master 5M x duplicates 1M @0.7, row blocks over 8 GPUs
    torchrun --nproc-per-node 8 ... bench_configs.py --config 5   # group_similar_strings 1M @0.85 end to end

Prints one JSON line on rank 0: wall time of the API call (max over ranks, best of --repeat after one warm-up), result rows,
MACs / kernel time / algorithmic GB/s of the K2 candidates kernel on rank 0.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def cpu_port(master, dupes, kw, fn, config):
    """The reference's CPU path (oracle port) for the same call, timed phase by phase on this box's usable cores."""
    import bench_cpu as C
    from oracle import pipeline as P
    from oracle import sdt
    from sklearn.feature_extraction.text import TfidfVectorizer
    sdt.build()
    cores = min(C.usable_cores(), 16)
    thr = kw["min_similarity"]
    scale_prod = scale_lin = 1.0
    m_names, d_names = master.tolist(), (dupes.tolist() if dupes is not None else None)
    if config == 4:                       # 1/10 of both sides: the product scales with rows_left x rows_right
        m_names, d_names = m_names[:len(m_names) // 10], d_names[:len(d_names) // 10]
        scale_prod, scale_lin = 100.0, 10.0
    ph = {}
    t0 = time.perf_counter()
    TfidfVectorizer(min_df=1, analyzer=P.n_grams, dtype=np.float64).fit(m_names + (d_names or []))   # __init__ :267
    m, d, _ = P.tf_idf_matrices(m_names, d_names)
    ph["vectorise_s"] = (time.perf_counter() - t0) * scale_lin
    t0 = time.perf_counter()
    Cm = P.build_matches(m, d, P.guess_blocks(m.shape[0], d.shape[0]), 20, thr, cores)
    ph["product_s"] = (time.perf_counter() - t0) * scale_prod
    t0 = time.perf_counter()
    if dupes is None:
        Cm = P.fix_diagonal_and_symmetrize(Cm)
    ml = P.matches_list(Cm)
    ph["post_s"] = (time.perf_counter() - t0) * scale_lin
    t0 = time.perf_counter()
    if fn == "group":
        P.deduplicate(ml, m.shape[0], "centroid")
    ph["result_s"] = (time.perf_counter() - t0) * scale_lin
    total = sum(ph.values())
    return {"wall_s": total, "phases": {k: round(v, 2) for k, v in ph.items()}, "threads": cores,
            "matches": int(len(ml) * scale_lin), "measured": "whole job" if config != 4 else
            "1/10 x 1/10 slice, product x100, other phases x10 (extrapolated)"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, required=True, choices=[2, 3, 4, 5])
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0, help="shrink the row counts (smoke runs)")
    ap.add_argument("--cpu", action="store_true",
                    help="rank 0 also times the CPU port (oracle) of the same call on this box's usable cores: the whole "
                         "job for configs 2, 3 and 5; config 4 from a 1/10 x 1/10 slice, extrapolated (x100 for the "
                         "product, x10 for the per-string and per-match parts) as SURVEY.md §8d allows")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))

    import pandas as pd
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("SG_B200_DISTRIBUTED", "1")
        dist.init_process_group("nccl", device_id=dev)
    import string_grouper_b200 as api
    from string_grouper_b200 import _device as D
    from synth_corpus import make_names

    sc = args.scale
    if args.config == 2:
        master, dupes, kw, fn = pd.Series(make_names(int(100_000 * sc), 0)), None, {"min_similarity": 0.8}, "match"
    elif args.config == 3:
        master, dupes, kw, fn = pd.Series(make_names(int(663_000 * sc), 0)), None, {"min_similarity": 0.8}, "match"
    elif args.config == 4:
        n_m, n_d = int(5_000_000 * sc), int(1_000_000 * sc)
        names = make_names(n_m + int(0.6 * n_d), 0)
        master = pd.Series(names[:n_m])
        dupes = pd.Series(names[n_m - (n_d - int(0.6 * n_d)):])          # 40 % of the duplicates are master rows
        kw, fn = {"min_similarity": 0.7}, "match"
    else:
        master, dupes, kw, fn = pd.Series(make_names(int(1_000_000 * sc), 0)), None, {"min_similarity": 0.85}, "group"

    def run():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sg = api.StringGrouper(master, dupes, **kw)
        sg._last_stats = {}
        sg.fit()
        out = sg.get_groups() if fn == "group" else sg.get_matches()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        t = torch.tensor([dt], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item()), sg, out

    run()                                                   # warm-up (CUDA context, allocator, NCCL)
    best, sg, out = min((run() for _ in range(args.repeat)), key=lambda r: r[0])

    # K2 kernel timing + MACs on this rank (one extra product with event timing)
    A, B = sg._get_tf_idf_matrices()
    stats = {"time_kernels": True, "count_macs": True}
    lo, hi = (0, A.shape[0])
    if world > 1 and getattr(A, "row_offset", None) is None:
        from string_grouper_b200 import _dist
        lo, hi = _dist.shard_range(A.shape[0], rank, world)
    D.cossim_topn(A, B, 20, kw["min_similarity"], row_begin=lo, row_end=hi, stats=stats)
    torch.cuda.synchronize()
    k_ms = sum(a.elapsed_time(b) for a, b in stats["candidate_events"])
    dfb = torch.bincount(B.d_indices[B.base:B.base + B.nnz].long(), minlength=B.shape[1])
    ip = A.d_indptr
    macs = int(dfb[A.d_indices[int(ip[lo].item()):int(ip[hi].item())].long()].sum().item())
    cpu = None
    if rank == 0 and args.cpu:
        cpu = cpu_port(master, dupes, kw, fn, args.config)
    if rank == 0:
        print(json.dumps({
            "cpu_port": cpu,
            "config": args.config, "n_gpus": world, "rows_left": len(master), "rows_right": len(dupes) if dupes is not None else len(master),
            "api": "group_similar_strings" if fn == "group" else "match_strings", "kwargs": kw,
            "e2e_wall_s": best, "result_rows": int(len(out)),
            "pairs_per_s": (len(sg._matches_list) / best),
            "matches": int(len(sg._matches_list)), "k2_macs_rank0": macs, "k2_kernel_ms_rank0": k_ms,
            "k2_algorithmic_GBps_rank0": 8 * macs / (k_ms / 1e3) / 1e9,
            "k2_frac_of_h100_datasheet_hbm": 8 * macs / (k_ms / 1e3) / 1e9 / 3350.0,
            "k2_walked_macs_rank0": stats.get("macs_walked"), "prune": stats.get("prune"), "kernel": stats.get("kernel"),
            "select": stats.get("select"),
            "accumulator": stats.get("acc"), "tile_w": stats.get("tile_w"), "warps": stats.get("warps"),
            "n_candidates_rank0": stats.get("n_candidates"),
            "n_refined_rank0": stats.get("n_refined"),
            "n_above_threshold_rank0": stats.get("n_above_threshold")}), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

"""Measure match_records against match_strings on one field and on the concatenated fields, in one process.

    python tests/gpu_records_measure.py [--out FILE]

Self-match: the 663 000 benchmark names (make_names(663_000, seed=0)) with seeded addresses, min_similarity 0.8, top
20: match_records (name 0.6, address 0.4), match_strings on the name, match_strings on name + " " + address.  Two
frames: 100 000 perturbed records against the 663 000.  The calls alternate; each is warmed up once and then timed
three times (fit + get_matches, ended by a device synchronisation).  Reported per call: wall-time range, peak device
memory above the baseline, candidates and the K2 path, rows of the left matrix with more than 32 stored features
(an upper bound of the rows that keep more than 32 after pruning), K1 per field and the stacking time, and the card's
name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

from synth_corpus import make_names  # noqa: E402
from synth_records import make_addresses, perturb  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--n", type=int, default=663_000)
    ap.add_argument("--n-dup", type=int, default=100_000)
    args = ap.parse_args()
    import torch
    from string_grouper_b200 import StringGrouper, _device as D
    from string_grouper_b200.records import _RecordsGrouper
    assert torch.cuda.is_available(), "needs a CUDA device"

    df = pd.DataFrame({"name": make_names(args.n, seed=0), "address": make_addresses(args.n, seed=1)})
    rng = np.random.default_rng(5)
    dup = perturb(df.iloc[rng.choice(args.n, args.n_dup, replace=False)].reset_index(drop=True), seed=6)
    concat = lambda f: f["name"] + " " + f["address"].fillna("")      # noqa: E731  today's workaround
    W = {"name": 0.6, "address": 0.4}
    calls = {
        "self/records": lambda: _RecordsGrouper(df, None, W),
        "self/name": lambda: StringGrouper(df["name"]),
        "self/concat": lambda: StringGrouper(concat(df)),
        "two/records": lambda: _RecordsGrouper(df, dup, W),
        "two/name": lambda: StringGrouper(df["name"], dup["name"]),
        "two/concat": lambda: StringGrouper(concat(df), concat(dup)),
    }
    res = {k: {"ms": []} for k in calls}

    def run(name):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        sg = calls[name]().fit()
        out = sg.get_matches()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        st = sg._last_stats
        r = res[name]
        r["ms"].append(round(ms, 1))
        r["peak_mib_above_baseline"] = round((torch.cuda.max_memory_allocated() - base) / 2**20, 1)
        r["n_matches"] = len(out)
        r["n_candidates"] = st.get("n_candidates")
        r["path"] = {k: st.get(k) for k in ("triangle", "dedup", "topn_floor", "kernel", "prune")}
        if "k1_ms" in st:
            r["k1_ms"] = {f: round(v, 2) for f, v in st["k1_ms"].items()}
            r["stack_ms"] = round(st["stack_ms"], 3)
        A, _ = sg._get_tf_idf_matrices() if "rows_over_32" not in r else (None, None)
        if A is not None:
            lens = (A.d_indptr[1:A.shape[0] + 1] - A.d_indptr[:A.shape[0]])
            r["rows_over_32_stored"] = int((lens > 32).sum().item())
            r["rows_over_32"] = True
        del sg, out

    for name in calls:          # warm-up of every shape
        run(name)
        res[name]["ms"].clear()
    for _ in range(3):
        for name in calls:
            run(name)
    for r in res.values():
        r["ms_range"] = [min(r["ms"]), max(r["ms"])]
        r.pop("rows_over_32", None)
    line = {"card": card(), "n": args.n, "n_dup": args.n_dup, "results": res}
    text = json.dumps(line, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()

"""Ad-hoc (not a test, not the bench): match_strings with blocking keys, next to the unkeyed call and the pandas loop
over the keys that users write without them.

Corpus: make_names(663_000, seed=0) (the benchmark corpus), self-match at min_similarity 0.8, top 20, with seeded
keys of 50 and of 5 000 distinct values.  One process per configuration (python tests/gpu_blocks_measure.py with no
arguments runs them all in turn):

    keyed     match_strings(names, master_keys=keys)
    unkeyed   match_strings(names)
    loop      for key, part in frame.groupby("key"): match_strings(part["name"])   (refits per key: other scores)

Each process makes one warm-up call, then times REPS calls (one for the loop), the device synchronised around each,
and prints one JSON line with the wall times, the path of the product and the card's name and power limit.

    python tests/gpu_blocks_measure.py [out.jsonl] [reps]
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CONFIGS = [("keyed", 50), ("unkeyed", 0), ("loop", 50), ("keyed", 5000), ("loop", 5000)]


def run_one(what, n_keys, reps):
    import numpy as np
    import pandas as pd
    import torch
    import string_grouper_b200 as api
    from gpu_corpus_measure import card
    from synth_corpus import make_names

    torch.cuda.set_device(0)
    names = pd.Series(make_names(663_000, seed=0))
    keys = pd.Series(np.random.default_rng(n_keys).integers(0, max(n_keys, 1), size=len(names)).astype(str))
    path = {}

    if what == "keyed":
        def call():
            sg = api.StringGrouper(names, master_keys=keys).fit()
            path.update({k: sg._last_stats.get(k) for k in ("blocks", "n_blocks_used", "triangle", "n_candidates",
                                                            "n_row_chunks", "topn_floor", "dedup")})
            return len(sg.get_matches())
    elif what == "unkeyed":
        def call():
            sg = api.StringGrouper(names).fit()
            path.update({k: sg._last_stats.get(k) for k in ("blocks", "triangle", "n_candidates", "n_row_chunks",
                                                            "topn_floor", "dedup")})
            return len(sg.get_matches())
    else:
        frame = pd.DataFrame({"name": names, "key": keys})

        def call():
            return sum(len(api.match_strings(part["name"])) for _, part in frame.groupby("key"))
        reps = 1

    n_out = call()                                   # warm-up
    times = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n_out = call()
        torch.cuda.synchronize()
        times.append(round(time.perf_counter() - t0, 4))
    rec = {"what": what, "n_keys": n_keys, "rows": len(names), "min_similarity": 0.8, "top_n": 20, "s": times,
           "n_matches": n_out, "path": path}
    rec.update(card())
    return rec


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--one":
        print(json.dumps(run_one(sys.argv[2], int(sys.argv[3]), int(sys.argv[4]))), flush=True)
        return
    out = sys.argv[1] if len(sys.argv) > 1 else None
    reps = sys.argv[2] if len(sys.argv) > 2 else "3"
    lines = []
    for what, n_keys in CONFIGS:
        res = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", what, str(n_keys), reps],
                             capture_output=True, text=True)
        line = res.stdout.strip().splitlines()[-1] if res.returncode == 0 and res.stdout.strip() else json.dumps(
            {"what": what, "n_keys": n_keys, "error": res.stderr[-2000:]})
        print(line, flush=True)
        lines.append(line)
    if out:
        with open(out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

"""Ad-hoc (not a test, not the bench): the top-n product without a threshold (min_similarity 0: every pair with a
positive score counts) with and without the top-n floor (DESIGN.md §4, "No threshold") on the benchmark shapes.  Each
run is a child process with a time limit, so a run that does not finish is recorded as such.  One JSON line per run on
stdout (and in `out.jsonl` when given): outcome, wall time, candidates (init / seed / main), survivors, peak memory.

    python tests/gpu_nothreshold_measure.py [out.jsonl] [time limit s] [modes,...]

`modes` keeps only the runs in those modes ("auto", "usual"); "usual" is the path without the floor.
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

THRESHOLD = 0.0


def child(kind, mode):
    import pandas as pd
    import torch
    from string_grouper_b200 import StringGrouper, _device as D
    from synth_corpus import make_names

    D.TOPN_FLOOR = {"usual": False, "auto": "auto"}[mode]
    gpu = torch.cuda.get_device_name(0)
    if kind == "self":
        sg = StringGrouper(pd.Series(make_names(663_000, seed=0)))
    else:                                   # match_most_similar shape: 150k duplicates against 400k master names
        base = make_names(480_000, seed=3)
        sg = StringGrouper(pd.Series(base[:400_000]), duplicates=pd.Series(base[330_000:480_000]), max_n_matches=1)
    A, B = sg._get_tf_idf_matrices()
    top_n = 20 if kind == "self" else 1
    D.cossim_topn(A, B, top_n, 0.8)                                         # warm-up: modules, right-side caches
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    st = {}
    t0 = time.time()
    try:
        out = D.cossim_topn(A, B, top_n, THRESHOLD, stats=st)
        torch.cuda.synchronize()
        outcome, nnz = "ok", out.nnz
    except Exception as e:                                                  # the usual path does not fit
        outcome, nnz = "%s: %s" % (type(e).__name__, str(e)[:160]), None
    wall = time.time() - t0
    keys = ("topn_floor", "floor_init", "n_candidates", "n_candidates_init", "n_candidates_seed", "n_candidates_main",
            "n_floor_init_positive", "n_rows_long", "n_survivors", "n_floor_dropped", "triangle", "n_row_chunks")
    rec = {"case": kind, "top_n": top_n, "threshold": THRESHOLD, "mode": mode, "outcome": outcome,
           "wall_s": round(wall, 3)}
    rec.update({k: st.get(k) for k in keys})
    rec.update({"nnz": nnz, "max_memory_allocated_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2),
                "gpu": gpu})
    print(json.dumps(rec), flush=True)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    limit = float(sys.argv[2]) if len(sys.argv) > 2 else 240.0
    modes = sys.argv[3].split(",") if len(sys.argv) > 3 else ["auto", "usual"]
    runs = [(kind, mode) for kind in ("self", "most_similar") for mode in ("auto", "usual") if mode in modes]
    lines = []
    for kind, mode in runs:
        cmd = [sys.executable, os.path.abspath(__file__), "--child", kind, mode]
        try:
            p = subprocess.run(cmd, capture_output=True, text=True, timeout=limit, cwd=ROOT)
            line = p.stdout.strip().splitlines()[-1] if p.stdout.strip() else json.dumps(
                {"case": kind, "mode": mode, "outcome": "exit %d: %s" % (p.returncode, p.stderr.strip()[-300:])})
        except subprocess.TimeoutExpired:
            line = json.dumps({"case": kind, "mode": mode,
                               "outcome": "not finished within %d s (process stopped)" % limit})
        print(line, flush=True)
        lines.append(line)
    if out:
        with open(out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        child(sys.argv[2], sys.argv[3])
    else:
        main()

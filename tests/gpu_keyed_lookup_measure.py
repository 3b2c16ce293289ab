"""Ad-hoc (not a test, not the bench): keyed register lookups, the four calls a record-linkage user would compare.

Register: make_names(663_000, seed=0) (the benchmark corpus) with seeded blocking keys in three layouts: 50 keys,
5 000 keys, and one key holding 70 % of the rows (the other 30 % over 49 keys).  Batches of 10k and 100k names (half
new names, half perturbed copies of register rows, as tests/gpu_corpus_measure.py) with keys drawn the same way.  For
each layout, batch and min_similarity in (0.8, 0.3, 0), after one warm-up call of every variant, the variants are
alternated REPS times, the device synchronised around each call:

    keyed corpus.match_nearest      StringGrouperCorpus(register, keys=...).match_nearest(register, batch, duplicates_keys=...)
    keyed match_nearest             the module function (refits the vectoriser on register ++ batch)
    keyed match_most_similar        the reference's function, keyed
    unkeyed corpus.match_nearest    StringGrouperCorpus(register).match_nearest(register, batch)

One JSON line per measurement on stdout (and in `out.jsonl` when given): wall times, peak device memory of the call,
the path the product took (top-n floor or not, candidates), or the error where the call ran out of memory, with the
card's name and power limit.

    python tests/gpu_keyed_lookup_measure.py [out.jsonl] [reps] [layouts]

`layouts`: comma-separated indices into LAYOUTS (default all), so that the layouts can be measured in separate runs.
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


LAYOUTS = ("50 keys", "5000 keys", "one key 70%")


def layout_keys(kind, n, seed):
    import numpy as np
    import pandas as pd
    rng = np.random.default_rng(seed)
    if kind == "50 keys":
        k = rng.integers(0, 50, size=n)
    elif kind == "5000 keys":
        k = rng.integers(0, 5000, size=n)
    else:                                   # one key holds 70 % of the rows
        k = np.where(rng.random(n) < 0.7, 0, rng.integers(1, 50, size=n))
    return pd.Series(["key%d" % v for v in k], dtype=object)


def main():
    import pandas as pd
    import torch
    import string_grouper_b200 as api
    from gpu_corpus_measure import card, make_batch
    from string_grouper_b200 import StringGrouper
    from synth_corpus import make_names

    out = sys.argv[1] if len(sys.argv) > 1 else None
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
    chosen = [int(i) for i in sys.argv[3].split(",")] if len(sys.argv) > 3 else range(len(LAYOUTS))
    torch.cuda.set_device(0)
    info = card()
    lines = []

    def emit(rec):
        rec.update(info)
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)

    def timed(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        try:
            fn()
            err = None
        except (torch.cuda.OutOfMemoryError, OverflowError, MemoryError) as e:
            err = "%s: %s" % (type(e).__name__, str(e).splitlines()[0][:160])
        torch.cuda.synchronize()
        return time.perf_counter() - t0, (torch.cuda.max_memory_allocated() - base) / 2**30, err

    names = make_names(663_000, seed=0)
    s = pd.Series(names)
    plain = api.StringGrouperCorpus(s)
    stats = {}
    real_nearest, real_fit = StringGrouper._match_nearest, StringGrouper.fit

    def keep(self):
        stats.clear()
        stats.update({k: v for k, v in self._last_stats.items() if isinstance(v, (int, float, bool, str))})

    def spy_nearest(self):              # the path of the last product
        try:
            return real_nearest(self)
        finally:
            keep(self)

    def spy_fit(self):
        try:
            return real_fit(self)
        finally:
            keep(self)

    StringGrouper._match_nearest, StringGrouper.fit = spy_nearest, spy_fit
    for li in chosen:
        kind = LAYOUTS[li]
        rkeys = layout_keys(kind, len(s), 10 + li)
        corpus = api.StringGrouperCorpus(s, keys=rkeys)
        for n, seed in ((10_000, 101), (100_000, 102)):
            b = pd.Series(make_batch(names, n, seed))
            bkeys = layout_keys(kind, n, 20 + li)
            for thr in (0.8, 0.3, 0.0):
                variants = {
                    "keyed corpus.match_nearest": lambda: corpus.match_nearest(
                        s, b, duplicates_keys=bkeys, min_similarity=thr),
                    "keyed match_nearest": lambda: api.match_nearest(
                        s, b, master_keys=rkeys, duplicates_keys=bkeys, min_similarity=thr),
                    "keyed match_most_similar": lambda: api.match_most_similar(
                        s, b, master_keys=rkeys, duplicates_keys=bkeys, min_similarity=thr),
                    "unkeyed corpus.match_nearest": lambda: plain.match_nearest(s, b, min_similarity=thr),
                }
                paths, errors = {}, {}
                for what, fn in variants.items():       # warm-up: modules, the register's right side
                    _, _, errors[what] = timed(fn)
                    paths[what] = dict(stats)
                times = {what: [] for what in variants}
                peaks = {what: 0.0 for what in variants}
                for _ in range(reps):
                    for what, fn in variants.items():
                        if errors[what]:
                            continue
                        dt, peak, err = timed(fn)
                        errors[what] = err
                        times[what].append(round(dt, 4))
                        peaks[what] = max(peaks[what], round(peak, 3))
                for what in variants:
                    p = paths[what]
                    rec = {"what": what, "layout": kind, "batch": n, "min_similarity": thr, "reps": reps,
                           "s": times[what], "peak_gib": peaks[what], "error": errors[what],
                           "path": {k: p.get(k) for k in ("blocks", "n_blocks_used", "nearest", "topn_floor",
                                                          "floor_init", "n_row_chunks", "n_candidates",
                                                          "n_candidates_estimate_usual")}}
                    emit(rec)
    if out:
        with open(out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

"""Ad-hoc (not a test, not the bench): match_nearest as a register lookup, next to match_most_similar on the same
inputs.

Corpus: make_names(663_000, seed=0) (the benchmark corpus).  Batches of 10k and 100k names: half new names, half
perturbed copies of corpus rows (as tests/gpu_corpus_measure.py).  For each batch and min_similarity in (0.8, 0.3, 0),
after one warm-up call of every variant, the variants are alternated REPS times, the device synchronised around each
call:

    corpus.match_nearest(corpus_series, batch)     StringGrouperCorpus, the corpus matrix as the right operand
    match_nearest(corpus_series, batch)            the module function (refits the vectoriser on corpus ++ batch)
    match_most_similar(corpus_series, batch)       the reference's function (one duplicate kept per master)

One JSON line per measurement on stdout (and in `out.jsonl` when given): wall times, peak device memory of the call,
the path the product took, and how many duplicates the module match_nearest maps to another master than
match_most_similar (both fit corpus ++ batch, so they score alike), with the card's name and power limit.

    python tests/gpu_nearest_measure.py [out.jsonl] [reps]
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import pandas as pd
    import torch
    import string_grouper_b200 as api
    from gpu_corpus_measure import card, make_batch
    from string_grouper_b200 import StringGrouper
    from synth_corpus import make_names

    out = sys.argv[1] if len(sys.argv) > 1 else None
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
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
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, (torch.cuda.max_memory_allocated() - base) / 2**30, r

    names = make_names(663_000, seed=0)
    s = pd.Series(names)
    corpus = api.StringGrouperCorpus(s)
    stats = {}
    real = StringGrouper._match_nearest

    def spy(self):                      # the path of the last match_nearest call
        out_ = real(self)
        stats.clear()
        stats.update({k: v for k, v in self._last_stats.items() if isinstance(v, (int, float, bool, str))})
        return out_

    StringGrouper._match_nearest = spy
    for n, seed in ((10_000, 101), (100_000, 102)):
        b = pd.Series(make_batch(names, n, seed))
        for thr in (0.8, 0.3, 0.0):
            variants = {
                "corpus.match_nearest(corpus, batch)": lambda: corpus.match_nearest(s, b, min_similarity=thr),
                "match_nearest(corpus, batch)": lambda: api.match_nearest(s, b, min_similarity=thr),
                "match_most_similar(corpus, batch)": lambda: api.match_most_similar(s, b, min_similarity=thr),
            }
            results, paths = {}, {}
            for what, fn in variants.items():       # warm-up: modules, the corpus's right side
                results[what] = fn()
                paths[what] = dict(stats)
            times = {what: [] for what in variants}
            peaks = {what: 0.0 for what in variants}
            for _ in range(reps):
                for what, fn in variants.items():
                    dt, peak, _ = timed(fn)
                    times[what].append(round(dt, 4))
                    peaks[what] = max(peaks[what], round(peak, 3))
            # the module functions fit the same vectoriser (corpus ++ batch), so their scores are the same; the corpus's
            # idf is the corpus's own, so its answers can differ from both
            col = "most_similar_master"
            near, mms = results["match_nearest(corpus, batch)"][col], results["match_most_similar(corpus, batch)"][col]
            differ = int((near.to_numpy() != mms.to_numpy()).sum())
            for what in variants:
                rec = {"what": what, "batch": n, "min_similarity": thr, "reps": reps, "s": times[what],
                       "peak_gib": peaks[what]}
                if "nearest" in what:
                    p = paths[what]
                    rec["path"] = {k: p.get(k) for k in ("topn_floor", "floor_init", "kernel", "acc", "prune",
                                                         "n_row_chunks", "n_candidates", "n_nearest_written")}
                else:
                    rec["differ_from_match_nearest"] = differ
                emit(rec)
    if out:
        with open(out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

"""Ad-hoc (not a test, not the bench): new batches against a fitted corpus (StringGrouperCorpus) next to the
module-level functions on the same inputs, which refit the vectoriser on batch ++ corpus and rebuild the corpus's
right side on every call.

Corpus: make_names(663_000, seed=0) (the benchmark corpus).  Batches of 10k and 100k names: half new names (another
seed), half perturbed copies of corpus rows.  For each batch, after one warm-up call of every variant, the two
implementations are alternated REPS times, the device synchronised around each call:

    corpus.match_strings(batch, corpus_series)          vs  match_strings(batch, corpus_series)
    corpus.match_most_similar(corpus_series, batch)     vs  match_most_similar(corpus_series, batch)

and the batch's K1 alone: the corpus transform (pack, upload, kernels) vs the refit of batch ++ corpus.  One JSON line
per measurement on stdout (and in `out.jsonl` when given), with the card's name and power limit.

    python tests/gpu_corpus_measure.py [out.jsonl] [reps]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = ""
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def make_batch(names, n, seed):
    from synth_corpus import make_names
    from test_gpu_corpus import perturb
    rng = np.random.default_rng(seed)
    fresh = make_names(n // 2, seed=seed)
    copies = [perturb(names[i], rng) for i in rng.integers(0, len(names), n - n // 2)]
    return fresh + copies


def main():
    import pandas as pd
    import torch
    import string_grouper_b200 as api
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
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    names = make_names(663_000, seed=0)
    s = pd.Series(names)
    t_fit, corpus = timed(lambda: api.StringGrouperCorpus(s))
    emit({"what": "corpus fit (K1 of 663k names)", "s": round(t_fit, 4)})
    for n, seed in ((10_000, 101), (100_000, 102)):
        b = pd.Series(make_batch(names, n, seed))
        variants = {
            "match_strings(batch, corpus)": (lambda: corpus.match_strings(b, s), lambda: api.match_strings(b, s)),
            "match_most_similar(corpus, batch)": (lambda: corpus.match_most_similar(s, b),
                                                  lambda: api.match_most_similar(s, b)),
            "K1 of the batch": (lambda: corpus._matrices(b, None, {}),
                                lambda: StringGrouper(b, s)._get_tf_idf_matrices(shard=False)),
        }
        for what, (on_corpus, module) in variants.items():
            on_corpus(), module()                                   # warm-up: modules, the corpus's right side
            tc, tm = [], []
            for _ in range(reps):
                tc.append(timed(on_corpus)[0])
                tm.append(timed(module)[0])
            rec = {"what": what, "batch": n, "reps": reps, "corpus_s": [round(x, 4) for x in tc],
                   "module_s": [round(x, 4) for x in tm]}
            if what != "K1 of the batch":
                rec["rows_corpus"], rec["rows_module"] = len(on_corpus()), len(module())
            emit(rec)
    if out:
        with open(out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

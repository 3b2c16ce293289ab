"""Ad-hoc (not a test, not the bench): group_similar_strings with linkage='single' and linkage='star' on the benchmark
names, make_names(663_000, seed=0), at min_similarity 0.8, top 20, group_rep 'centroid'.

After one warm-up call of each, the two linkages are alternated REPS times (the device synchronised around each call):
the end-to-end call, then the grouping step alone on one fitted match list (_device.group_reps against
_device.group_star).  Then, once per linkage: the number of groups of two or more strings, the largest group, the
strings whose representative is another string, and how many of those are not listed with their representative (no
direct match).  The round count comes from the numpy rounds of string_grouper.star_representatives on the same list,
which must give the device's groups.  Last, a path of 20 000 strings whose ranks increase along it (20 000 rounds).

One JSON line per measurement on stdout (and in `out.jsonl` when given), with the card's name and power limit.

    python tests/gpu_star_measure.py [out.jsonl] [reps]
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import numpy as np
    import pandas as pd
    import torch
    import string_grouper_b200 as api
    from gpu_corpus_measure import card
    from string_grouper_b200 import StringGrouper, _device
    from string_grouper_b200.string_grouper import _centroid_weight, star_representatives
    from scipy.sparse import csr_matrix
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
        return 1e3 * (time.perf_counter() - t0), r

    s = pd.Series(make_names(663_000, seed=0))
    n = len(s)
    for linkage in ("single", "star"):
        api.group_similar_strings(s, linkage=linkage)          # warm-up
    for rep_i in range(reps):
        for linkage in ("single", "star"):
            ms, _ = timed(lambda: api.group_similar_strings(s, linkage=linkage))
            emit({"what": "group_similar_strings", "linkage": linkage, "rep": rep_i, "ms": round(ms, 1)})

    sg = StringGrouper(s).fit()
    M = _device.as_device_matches(sg._matches_device)
    steps = {"single": lambda: _device.group_reps(M, n, True), "star": lambda: _device.group_star(M, n, True)}
    for fn in steps.values():
        fn()
    for rep_i in range(reps):
        for linkage, fn in steps.items():
            ms, _ = timed(fn)
            emit({"what": "grouping step", "linkage": linkage, "rep": rep_i, "ms": round(ms, 2), "pairs": M.nnz})

    r, c, w = M.host_triples()
    listed = np.unique(np.concatenate([r * n + c, c * n + r]))
    for linkage, fn in steps.items():
        rep = fn()
        size = np.bincount(rep, minlength=n)
        moved = np.nonzero(rep != np.arange(n))[0]
        direct = np.isin(moved * n + rep[moved], listed)
        rec = {"what": "groups", "linkage": linkage, "pairs": M.nnz, "groups_2plus": int((size >= 2).sum()),
               "largest_group": int(size.max()), "rep_is_another_string": int(len(moved)),
               "rep_not_a_direct_match": int((~direct).sum())}
        if linkage == "star":
            weight = _centroid_weight(csr_matrix((np.full(len(r), 1), (r, c)), shape=(n, n)), sg._matches_list)
            host, rounds = star_representatives(n, r, c, weight)
            rec.update(rounds=rounds, host_rule_equal=bool(np.array_equal(host, rep)))
        emit(rec)

    m = 20_000
    path = _device.DeviceMatches((m, m), torch.arange(m - 1, dtype=torch.int32, device="cuda"),
                                 torch.arange(1, m, dtype=torch.int32, device="cuda"),
                                 torch.ones(m - 1, dtype=torch.float64, device="cuda"), m - 1, 1)
    _device.group_star(path, m, False)
    for rep_i in range(reps):
        ms, rep = timed(lambda: _device.group_star(path, m, False))
        emit({"what": "path of increasing ranks", "strings": m, "rounds": m, "rep": rep_i, "ms": round(ms, 1),
              "exact": bool(np.array_equal(rep, np.arange(m) - np.arange(m) % 2))})

    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()

"""Seeded synthetic records (name + address) for the tests and measurements of match_records.

Names come from synth_corpus.make_names; addresses look like "<number> <pseudo-word> <ST|AVE|RD|...>, <city>", and a
share of them is missing (None).  Duplicates copy a record and perturb its name, its address or both by one character
edit, or copy it unchanged.  numpy / pandas only.
"""
import numpy as np
import pandas as pd

from synth_corpus import make_names

_STREET = ["ST", "AVE", "RD", "BLVD", "LN", "DR", "CT", "WAY", "PL", "PKWY"]
_LETTERS = np.array(list("ABCDEFGHIJKLMNOPQRSTUVWXYZ"))


def _words(rng, n, lo=4, hi=10):
    lens = rng.integers(lo, hi, size=n)
    flat = "".join(rng.choice(_LETTERS, size=int(lens.sum())).tolist())
    ends = np.cumsum(lens)
    return [flat[e - k:e] for e, k in zip(ends.tolist(), lens.tolist())]


def make_addresses(n, seed=0, missing=0.1, n_streets=5000, n_cities=300):
    rng = np.random.default_rng(seed)
    streets = _words(rng, n_streets)
    cities = _words(rng, n_cities, 5, 12)
    num = rng.integers(1, 9999, size=n)
    st = rng.integers(0, n_streets, size=n)
    kind = rng.integers(0, len(_STREET), size=n)
    city = rng.integers(0, n_cities, size=n)
    gone = rng.random(n) < missing
    return [None if gone[i] else "%d %s %s, %s" % (num[i], streets[st[i]], _STREET[kind[i]], cities[city[i]])
            for i in range(n)]


def _edit(s, rng):
    """one character replaced, deleted or inserted"""
    if not isinstance(s, str) or not s:
        return s
    p = int(rng.integers(0, len(s)))
    c = str(rng.choice(_LETTERS))
    k = int(rng.integers(0, 3))
    return s[:p] + c + s[p + 1:] if k == 0 else (s[:p] + s[p + 1:] if k == 1 else s[:p] + c + s[p:])


def perturb(records, seed=0, exact=0.1):
    """A copy of every record: unchanged (share `exact`), or its name, its address or both edited."""
    rng = np.random.default_rng(seed)
    names, addrs = records["name"].tolist(), records["address"].tolist()
    what = rng.integers(0, 3, size=len(names))
    same = rng.random(len(names)) < exact
    for i in range(len(names)):
        if same[i]:
            continue
        if what[i] in (0, 2):
            names[i] = _edit(names[i], rng)
        if what[i] in (1, 2):
            addrs[i] = _edit(addrs[i], rng)
    return pd.DataFrame({"name": names, "address": addrs})


def make_records(n, seed=0, missing=0.1, dup_share=0.3):
    """n records: about (1 - dup_share) n originals and dup_share n perturbed copies of them, shuffled."""
    rng = np.random.default_rng(seed + 17)
    n_dup = int(dup_share * n)
    base = pd.DataFrame({"name": make_names(n - n_dup, seed=seed),
                         "address": make_addresses(n - n_dup, seed=seed + 1, missing=missing)})
    copies = perturb(base.iloc[rng.integers(0, n - n_dup, size=n_dup)].reset_index(drop=True), seed=seed + 2)
    out = pd.concat([base, copies], ignore_index=True)
    return out.iloc[rng.permutation(n)].reset_index(drop=True)

"""TEST INFRASTRUCTURE — golden-vector generator.

Runs the UNMODIFIED reference (a checkout of Bergvca/string_grouper) — with the C oracle standing in
for the absent `sparse_dot_topn` wheel (oracle/standin/) — on the reference's own fixtures, the tutorial
data and two seeded synthetic corpora, and writes the answers under tests/golden/.  The tests replay
the committed fixtures, so they do not need the reference checkout.

    python oracle/make_golden.py /path/to/string_grouper_checkout
"""
import json
import os
import sys

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "standin"))
REFERENCE = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else os.environ.get("STRING_GROUPER_SRC", "."))
sys.path.insert(0, REFERENCE)
sys.path.insert(0, ROOT)

from string_grouper import (StringGrouper, compute_pairwise_similarities, group_similar_strings,  # noqa: E402
                            match_most_similar, match_strings)
from synth_corpus import make_names  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def _cell(v):
    if isinstance(v, (np.floating, float)):
        return None if np.isnan(v) else float(v)
    if isinstance(v, (np.integer,)):
        return int(v)
    if isinstance(v, (np.bool_,)):
        return bool(v)
    if v is pd.NA or v is None:
        return None
    return v


def encode(obj):
    """DataFrame / Series -> JSON-able dict (values, labels, index, dtypes kinds)."""
    if isinstance(obj, pd.Series):
        return {"kind": "series", "name": obj.name, "dtype": obj.dtype.kind if hasattr(obj.dtype, "kind") else "O",
                "values": [_cell(v) for v in obj.tolist()],
                "index_names": list(obj.index.names), "index": [list(map(_cell, t)) if isinstance(t, tuple) else _cell(t)
                                                                for t in obj.index.tolist()]}
    assert isinstance(obj, pd.DataFrame)
    return {"kind": "frame", "columns": [str(c) for c in obj.columns],
            "dtypes": [obj[c].dtype.kind if hasattr(obj[c].dtype, "kind") else "O" for c in obj.columns],
            "data": [[_cell(v) for v in row] for row in obj.itertuples(index=False, name=None)],
            "index_names": list(obj.index.names),
            "index": [list(map(_cell, t)) if isinstance(t, tuple) else _cell(t) for t in obj.index.tolist()]}


def customers():
    df = pd.DataFrame(
        [('BB016741P', 'Mega Enterprises Corporation'), ('CC082744L', 'Hyper Startup Incorporated'),
         ('AA098762D', 'Hyper Startup Inc.'), ('BB099931J', 'Hyper-Startup Inc.'),
         ('HH072982K', 'Hyper Hyper Inc.'), ('EE059082Q', 'Mega Enterprises Corp.')],
        columns=('Customer ID', 'Customer Name'))
    df2 = pd.DataFrame(
        [('BB016741P', 'Mega Enterprises Corporation'), ('CC082744L', 'Hyper Startup Incorporated'),
         ('AA098762D', 'Hyper Startup Inc.'), ('BB099931J', 'Hyper-Startup Inc.'),
         ('DD012339M', 'HyperStartup Inc.'), ('HH072982K', 'Hyper Hyper Inc.'),
         ('EE059082Q', 'Mega Enterprises Corp.')],
        columns=('Customer ID', 'Customer Name'))
    return df, df2


UNICODE_TM = ["Acme\u2122 Corp", "ACME TM CORP", "AcmeTM Corp", "\u2116 5 Ltd", "No 5 Ltd", "no 5 ltd",
              "Degree \u2103 Inc", "degree c inc", "plain ascii name"]
UNICODE_RAW = ["Caf\u00e9 M\u00fcller GmbH", "Cafe Muller GmbH", "CAF\u00c9 M\u00dcLLER GMBH", "\u6771\u4eac\u682a\u5f0f\u4f1a\u793e",
               "\u6771\u4eac\u682a\u5f0f\u4f1a\u793e\u30db\u30fc\u30eb\u30c7\u30a3\u30f3\u30b0\u30b9", "\u0130stanbul A.\u015e.", "istanbul a.s.",
               "Stra\u00dfe 7 & S\u00f8n", "strasse 7 & son", "\U0001F600 emoji co", "emoji co"]


def cases():
    """name -> (callable description for the test, result).  Every entry is replayed by
    tests/test_golden_api.py through string_grouper_b200 with the same arguments."""
    out = {}
    acc = pd.read_csv(os.path.join(REFERENCE, "tutorials", "accounts.csv"))
    df, df2 = customers()
    names, ids = df['Customer Name'], df['Customer ID']
    names2, ids2 = df2['Customer Name'], df2['Customer ID']
    multi = names.copy()
    multi.index = pd.MultiIndex.from_tuples([(1, 'a'), (1, 'b'), (2, 'a'), (2, 'b'), (3, 'a'), (3, 'b')],
                                            names=['lvl0', 'lvl1'])
    unnamed = pd.Series(names.tolist())
    shifted = names.copy()
    shifted.index = [10, 11, 12, 13, 14, 15]

    def add(key, fn, series, kwargs, result):
        out[key] = {"fn": fn, "series": series, "kwargs": kwargs, "result": encode(result)}

    # tutorial data (config 1 of BASELINE.json)
    add("accounts_match_0.8", "match_strings", ["acc.name", None, "acc.id", None], {"ignore_index": True},
        match_strings(acc['name'], master_id=acc['id'], ignore_index=True))
    add("accounts_match_0.7", "match_strings", ["acc.name", None, "acc.id", None],
        {"ignore_index": True, "min_similarity": 0.7},
        match_strings(acc['name'], master_id=acc['id'], ignore_index=True, min_similarity=0.7))
    add("accounts_match_default", "match_strings", ["acc.name", None, None, None], {}, match_strings(acc['name']))
    add("accounts_groups", "group_similar_strings", ["acc.name", "acc.id"], {},
        group_similar_strings(acc['name'], acc['id']))
    add("accounts_groups_first", "group_similar_strings", ["acc.name", None], {"group_rep": "first"},
        group_similar_strings(acc['name'], group_rep='first'))

    # reference fixture frames
    S = {"names": names, "ids": ids, "names2": names2, "ids2": ids2, "multi": multi, "unnamed": unnamed,
         "shifted": shifted}
    for key, args, kw in [
        ("cust_self", ["names", None, None, None], {}),
        ("cust_self_ids", ["names", None, "ids", None], {}),
        ("cust_self_0.6", ["names", None, None, None], {"min_similarity": 0.6}),
        ("cust_self_top1", ["names2", None, None, None], {"max_n_matches": 1, "min_similarity": 0.5}),
        ("cust_self_nosym", ["names2", None, None, None], {"force_symmetries": False, "min_similarity": 0.5}),
        ("cust_two", ["names", "names2", None, None], {"min_similarity": 0.5}),
        ("cust_two_ids", ["names", "names2", "ids", "ids2"], {"min_similarity": 0.5}),
        ("cust_two_ignore_index", ["names", "names2", "ids", "ids2"], {"min_similarity": 0.5, "ignore_index": True}),
        ("cust_multi", ["multi", None, None, None], {"min_similarity": 0.5}),
        ("cust_unnamed_two", ["unnamed", "names2", None, None], {"min_similarity": 0.4}),
        ("cust_shifted", ["shifted", "names2", None, None], {"min_similarity": 0.5}),
        ("cust_f32", ["names", "names2", None, None], {"min_similarity": 0.5, "tfidf_matrix_dtype": "float32"}),
        ("cust_ngram2", ["names", "names2", None, None], {"min_similarity": 0.5, "ngram_size": 2}),
        ("cust_ngram4", ["names", "names2", None, None], {"min_similarity": 0.3, "ngram_size": 4}),
        ("cust_case", ["names", "names2", None, None], {"min_similarity": 0.5, "ignore_case": False}),
        ("cust_regex", ["names", "names2", None, None], {"min_similarity": 0.5, "regex": r"[aeiou]"}),
        ("cust_zero", ["names", ["whatever"], None, None], {"min_similarity": 0.0}),
        ("cust_blocks", ["names", "names2", None, None], {"min_similarity": 0.1, "n_blocks": (2, 3)}),
        # keys beyond 32 bits (sort-based vocabulary of the device vectoriser)
        ("cust_ngram5", ["names", "names2", None, None], {"min_similarity": 0.3, "ngram_size": 5}),
        ("cust_ngram9", ["names", "names2", None, None], {"min_similarity": 0.1, "ngram_size": 9}),
        ("cust_ngram12", ["names", "names2", None, None], {"min_similarity": 0.05, "ngram_size": 12}),
        # str.lower() runs BEFORE NFKD, which can put capital ASCII back (ADVICE r1): 'TM', 'No', 'C' stay capital
        ("sym_tm", [UNICODE_TM, None, None, None], {"min_similarity": 0.2}),
        ("sym_tm_two", [UNICODE_TM, ["ACME TM CORP", "acmeTM corp", "no 5 ltd"], None, None], {"min_similarity": 0.2}),
        # normalize_to_ascii=False keeps the non-ASCII code points (code-point n-grams)
        ("raw_unicode", [UNICODE_RAW, None, None, None], {"min_similarity": 0.2, "normalize_to_ascii": False}),
        ("raw_unicode_case", [UNICODE_RAW, UNICODE_RAW[:4], None, None],
         {"min_similarity": 0.2, "normalize_to_ascii": False, "ignore_case": False}),
        ("raw_unicode_ngram2", [UNICODE_RAW, None, None, None],
         {"min_similarity": 0.2, "normalize_to_ascii": False, "ngram_size": 2}),
    ]:
        a = [S[x] if isinstance(x, str) else (pd.Series(x) if isinstance(x, list) else None) for x in args]
        kw2 = dict(kw)
        if kw2.get("tfidf_matrix_dtype") == "float32":
            kw2["tfidf_matrix_dtype"] = np.float32
        add(key, "match_strings", args, kw, match_strings(*a, **kw2))

    for key, args, kw in [
        ("mms_plain", ["names", "names2", None, None], {}),
        ("mms_ids", ["names", "names2", "ids", "ids2"], {}),
        ("mms_ignore_index", ["names", "names2", "ids", "ids2"], {"ignore_index": True}),
        ("mms_replace_na", ["names", ["Hyper Startup Inc", "zzz qqq", "Mega Enterprises"], None, None],
         {"replace_na": True, "min_similarity": 0.6}),
        ("mms_unmatched", ["names", ["Hyper Startup Inc", "zzz qqq", "Mega Enterprises"], None, None],
         {"min_similarity": 0.6}),
        ("mms_unmatched_ids", ["names", ["Hyper Startup Inc", "zzz qqq", "Mega Enterprises"], "ids",
                               ["X1", "X2", "X3"]], {"min_similarity": 0.6}),
        ("mms_multi", ["multi", ["Hyper Startup Inc", "zzz qqq"], None, None], {"min_similarity": 0.6}),
        ("mms_unnamed", ["unnamed", ["Hyper Startup Inc", "zzz qqq"], None, None], {"min_similarity": 0.6}),
    ]:
        a = [S[x] if isinstance(x, str) else (pd.Series(x) if isinstance(x, list) else None) for x in args]
        add(key, "match_most_similar", args, kw, match_most_similar(*a, **kw))

    for key, args, kw in [
        ("grp_centroid", ["names", None], {}),
        ("grp_first", ["names", None], {"group_rep": "first"}),
        ("grp_ids", ["names", "ids"], {"min_similarity": 0.6}),
        ("grp_ignore_index", ["names2", "ids2"], {"ignore_index": True, "min_similarity": 0.6}),
        ("grp_multi", ["multi", None], {"min_similarity": 0.6}),
        ("grp_unnamed", ["unnamed", None], {"min_similarity": 0.6}),
    ]:
        a = [S[x] if isinstance(x, str) else None for x in args]
        add(key, "group_similar_strings", args, kw, group_similar_strings(*a, **kw))

    s1 = pd.Series(['foo', 'bar', 'baz', 'Mega Enterprises Corporation'])
    s2 = pd.Series(['foosball', 'bar', 'bay', 'Mega Enterprises Corp.'])
    add("pairwise", "compute_pairwise_similarities", [s1.tolist(), s2.tolist()], {},
        compute_pairwise_similarities(s1, s2))
    add("pairwise_f32", "compute_pairwise_similarities", [s1.tolist(), s2.tolist()],
        {"tfidf_matrix_dtype": "float32"}, compute_pairwise_similarities(s1, s2, tfidf_matrix_dtype=np.float32))
    return out


def synthetic():
    """Bigger seeded corpora: store the match list (and groups) as arrays."""
    arrays = {}
    names = pd.Series(make_names(3000, seed=11), name="name")
    sg = StringGrouper(names, min_similarity=0.8).fit()
    ml = sg._matches_list
    arrays["self3000_master_side"] = ml.master_side.to_numpy()
    arrays["self3000_dupe_side"] = ml.dupe_side.to_numpy()
    arrays["self3000_similarity"] = ml.similarity.to_numpy()
    arrays["self3000_true_max"] = np.array([sg._true_max_n_matches])
    grp = sg.get_groups()
    arrays["self3000_group_rep_index"] = grp["group_rep_index"].to_numpy()

    master = pd.Series(make_names(2000, seed=12))
    dupes = pd.Series(make_names(1200, seed=12)[:600] + make_names(200, seed=13))
    sg = StringGrouper(master, dupes, min_similarity=0.7, max_n_matches=5).fit()
    ml = sg._matches_list
    arrays["two2000_master_side"] = ml.master_side.to_numpy()
    arrays["two2000_dupe_side"] = ml.dupe_side.to_numpy()
    arrays["two2000_similarity"] = ml.similarity.to_numpy()
    near = sg.get_groups()
    arrays["two2000_nearest"] = np.array(near["most_similar_master"].tolist(), dtype=object)
    arrays["two2000_nearest_index"] = near["most_similar_index"].to_numpy(dtype=np.float64)

    # TF-IDF matrix pin (K1): CSR of a corpus with every analyzer case
    texts = pd.Series(make_names(500, seed=14) + ["", "ab", "abc", "A.B,C-D/E F\tG", "ÀbracâDABRÀ", "ﬁ½① İstanbul",
                                                  "x" * 300 + " inc", "aaa aaa aaa aaaa"])
    sg = StringGrouper(texts)
    m, _ = sg._get_tf_idf_matrices()
    arrays["tfidf_indptr"], arrays["tfidf_indices"], arrays["tfidf_data"] = m.indptr, m.indices, m.data
    vocab = sg._vectorizer.vocabulary_
    arrays["tfidf_vocab"] = np.array(sorted(vocab, key=vocab.get), dtype=object)
    sg32 = StringGrouper(texts, tfidf_matrix_dtype=np.float32)
    m32, _ = sg32._get_tf_idf_matrices()
    arrays["tfidf32_data"] = m32.data
    return arrays


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    c = cases()
    with open(os.path.join(OUT, "api_cases.json"), "w") as f:
        json.dump(c, f, indent=1, sort_keys=True)
    arr = synthetic()
    np.savez_compressed(os.path.join(OUT, "synthetic.npz"), **arr)
    acc = pd.read_csv(os.path.join(REFERENCE, "tutorials", "accounts.csv"))
    acc.to_csv(os.path.join(OUT, "accounts_input.csv"), index=False)   # 14-row tutorial input, data not code
    print("wrote %d api cases, %d arrays" % (len(c), len(arr)))

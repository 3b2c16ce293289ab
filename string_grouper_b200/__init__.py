"""string_grouper_b200 — the string_grouper hot path (n-gram TF-IDF + top-n thresholded sparse cosine
product) on H100 (sm_90a), behind the reference's own API.

    from string_grouper_b200 import match_strings, match_most_similar, group_similar_strings, \
        compute_pairwise_similarities, StringGrouper

mirrors `from string_grouper import ...` (string_grouper/__init__.py:1-2).  `StringGrouperCorpus` fits the
vectoriser once and matches new Series against that corpus (string_grouper_b200/corpus.py).  `match_nearest` returns
what the reference documents for match_most_similar: every duplicate's most similar master.  Blocking keys
(`master_keys` / `duplicates_keys`, `keys`) restrict the matches to strings of equal keys in every function that
matches, `match_nearest` included, and in a `StringGrouperCorpus` built with `keys=` (a keyed register lookup).
`match_records` and `group_similar_records` match DataFrames over several string columns with a weighted similarity
(string_grouper_b200/records.py).
"""
from .corpus import StringGrouperCorpus  # noqa: F401
from .records import group_similar_records, match_records  # noqa: F401
from .string_grouper import (StringGrouper, StringGrouperConfig, StringGrouperNotFitException,  # noqa: F401
                             compute_pairwise_similarities, group_similar_strings, match_most_similar,
                             match_nearest, match_strings)

__all__ = ["StringGrouper", "StringGrouperConfig", "StringGrouperCorpus", "StringGrouperNotFitException",
           "compute_pairwise_similarities", "group_similar_records", "group_similar_strings", "match_most_similar",
           "match_nearest", "match_records", "match_strings"]

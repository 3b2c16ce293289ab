"""string_grouper_b200 — the string_grouper hot path (n-gram TF-IDF + top-n thresholded sparse cosine
product) on H100 (sm_90a), behind the reference's own API.

    from string_grouper_b200 import match_strings, match_most_similar, group_similar_strings, \
        compute_pairwise_similarities, StringGrouper

mirrors `from string_grouper import ...` (string_grouper/__init__.py:1-2).
"""
from .string_grouper import (StringGrouper, StringGrouperConfig, StringGrouperNotFitException,  # noqa: F401
                             compute_pairwise_similarities, group_similar_strings, match_most_similar,
                             match_strings)

__all__ = ["StringGrouper", "StringGrouperConfig", "StringGrouperNotFitException", "compute_pairwise_similarities",
           "group_similar_strings", "match_most_similar", "match_strings"]

"""StringGrouperCorpus: fit the TF-IDF vectoriser once on a corpus, then match new strings against it.

The reference documents this workflow (its `StringGrouper.match_strings` "without rebuilding the corpus", docs
"reuse the same tf-idf corpus") but every one of its methods refits the vectoriser on the new master ++ duplicates;
StringGrouper here does the same.  A corpus instead keeps what K1 fitted in HBM — the vocabulary tables, the idf and
the corpus matrix — and turns every Series a method receives into `vectoriser.transform(series)` (csrc/sg_tfidf.cu,
csrc/sg_tfidf64.cu): n-grams outside the corpus vocabulary are dropped, idf is the corpus's.  What follows the
matrices is StringGrouper's own code.

Because transform(corpus) is fit_transform(corpus) bit for bit, `StringGrouperCorpus(s).match_strings(s)` equals
`match_strings(s)` and `StringGrouperCorpus(pd.concat([m, d])).match_strings(m, d)` equals `match_strings(m, d)`.
"""
from typing import Optional, Union

import pandas as pd

from . import _device, _ingest
from .string_grouper import StringGrouper

# options that define the vectoriser: fixed when the corpus is built
VECTORISER_OPTIONS = ("ngram_size", "regex", "ignore_case", "normalize_to_ascii", "tfidf_matrix_dtype")


class StringGrouperCorpus:
    """A TF-IDF corpus fitted once (K1), resident in HBM, that new Series are matched against.

    `kwargs` are StringGrouperConfig keys.  The vectoriser options among them are fixed here; the others are defaults
    that a method's own kwargs override.  A method argument that IS the corpus Series object (`is`) uses the corpus
    matrix itself: it is not vectorised again, and what K2 builds for it (row order, postings) carries over from call
    to call.
    """

    def __init__(self, strings: pd.Series, **kwargs):
        grouper = StringGrouper(strings, **kwargs)      # validates the Series and the options like StringGrouper
        self._matrix, _ = grouper._get_tf_idf_matrices(shard=False)    # ValueError on an empty vocabulary
        self._series = strings
        self._config = grouper._config
        self._vocabulary = grouper._vocabulary

    @property
    def n_docs(self) -> int:
        """Number of corpus strings (the document count of the idf)."""
        return len(self._series)

    @property
    def idf_(self):
        """idf of every column (TfidfVectorizer.idf_, matrix dtype)."""
        return self._vocabulary.idf_

    def feature_names(self):
        """The corpus vocabulary in column order (TfidfVectorizer.get_feature_names_out)."""
        return self._vocabulary.feature_names()

    # ------------------------------------------------------------------ the reference's functions, on this corpus
    def fit(self, master: pd.Series, duplicates: Optional[pd.Series] = None, master_id: Optional[pd.Series] = None,
            duplicates_id: Optional[pd.Series] = None, **kwargs) -> StringGrouper:
        """A fitted StringGrouper (get_matches, get_groups, add_match ...) whose matrices come from this corpus."""
        return self._grouper(master, duplicates, master_id, duplicates_id, **kwargs).fit()

    def match_strings(self, master: pd.Series, duplicates: Optional[pd.Series] = None,
                      master_id: Optional[pd.Series] = None, duplicates_id: Optional[pd.Series] = None,
                      **kwargs) -> pd.DataFrame:
        return self.fit(master, duplicates, master_id, duplicates_id, **kwargs).get_matches()

    def match_most_similar(self, master: pd.Series, duplicates: pd.Series, master_id: Optional[pd.Series] = None,
                           duplicates_id: Optional[pd.Series] = None, **kwargs) -> Union[pd.DataFrame, pd.Series]:
        kwargs['max_n_matches'] = 1
        return self.fit(master, duplicates, master_id, duplicates_id, **kwargs).get_groups()

    def match_nearest(self, master: pd.Series, duplicates: pd.Series, master_id: Optional[pd.Series] = None,
                      duplicates_id: Optional[pd.Series] = None, **kwargs) -> Union[pd.DataFrame, pd.Series]:
        """match_nearest on this corpus.  With the corpus Series as `master` (a register lookup: which corpus entry
        is each incoming string?) the corpus matrix is the right operand, and its row order and postings carry over
        from call to call."""
        return self._grouper(master, duplicates, master_id, duplicates_id, **kwargs)._match_nearest()

    def group_similar_strings(self, strings_to_group: pd.Series, string_ids: Optional[pd.Series] = None,
                              **kwargs) -> Union[pd.DataFrame, pd.Series]:
        return self.fit(strings_to_group, master_id=string_ids, **kwargs).get_groups()

    def compute_pairwise_similarities(self, string_series_1: pd.Series, string_series_2: pd.Series,
                                      **kwargs) -> pd.Series:
        return self._grouper(string_series_1, string_series_2, **kwargs).dot()

    # ------------------------------------------------------------------ internals
    def _grouper(self, master, duplicates=None, master_id=None, duplicates_id=None, **kwargs):
        options = self._config._asdict()
        options.update(kwargs)
        return _CorpusGrouper(self, master, duplicates, master_id, duplicates_id, **options)

    def _check_options(self, options):
        changed = [k for k in VECTORISER_OPTIONS if k in options and options[k] != getattr(self._config, k)]
        if changed:
            raise ValueError("%s fixed when the corpus was built: %s" % (
                "option is" if len(changed) == 1 else "options are",
                ", ".join("%s=%r (corpus: %r)" % (k, options[k], getattr(self._config, k)) for k in changed)))

    def _matrices(self, master, duplicates, stats):
        """(master matrix, duplicate matrix): the corpus matrix for an argument that is the corpus Series, one K1
        transform for the others."""
        series = [master] if duplicates is None else [master, duplicates]
        fresh = [s for s in series if s is not self._series]
        mats = iter(())
        if fresh:
            cfg = self._config
            data, offsets, flags, _ = _ingest.pack_strings(fresh, cfg.regex, cfg.ignore_case, cfg.normalize_to_ascii)
            mats = iter(_device.tfidf_transform(data, offsets, len(fresh[0]), flags, self._vocabulary, stats=stats))
        out = [self._matrix if s is self._series else next(mats) for s in series]
        return out[0], out[-1]


class _CorpusGrouper(StringGrouper):
    """StringGrouper whose _get_tf_idf_matrices (the reference's seam between vectoriser and product) transforms
    through a corpus instead of refitting."""

    def __init__(self, corpus, *args, **kwargs):
        self._corpus = corpus
        super().__init__(*args, **kwargs)

    def _set_options(self, **kwargs):
        self._corpus._check_options(kwargs)      # also guards update_options() of the returned grouper
        super()._set_options(**kwargs)

    def _get_tf_idf_matrices(self, shard=True):
        stats = {}
        master, dup = self._corpus._matrices(self._master, self._duplicates, stats)
        self._vocabulary = self._corpus._vocabulary
        self._last_stats = stats
        self._raw_device = None
        return master, dup

"""StringGrouperCorpus: fit the TF-IDF vectoriser once on a corpus, then match new strings against it.

The reference documents this workflow (its `StringGrouper.match_strings` "without rebuilding the corpus", docs
"reuse the same tf-idf corpus") but every one of its methods refits the vectoriser on the new master ++ duplicates;
StringGrouper here does the same.  A corpus instead keeps what K1 fitted in HBM — the vocabulary tables, the idf and
the corpus matrix — and turns every Series a method receives into `vectoriser.transform(series)` (csrc/sg_tfidf.cu,
csrc/sg_tfidf64.cu): n-grams outside the corpus vocabulary are dropped, idf is the corpus's.  What follows the
matrices is StringGrouper's own code.

Because transform(corpus) is fit_transform(corpus) bit for bit, `StringGrouperCorpus(s).match_strings(s)` equals
`match_strings(s)` and `StringGrouperCorpus(pd.concat([m, d])).match_strings(m, d)` equals `match_strings(m, d)`.

Blocking keys (see StringGrouper) are fixed with the corpus too: `keys` gives one per corpus string, and every method
argument that is the corpus Series carries them, with its id tensor, row order and postings reused from call to call.
"""
from typing import Optional, Union

import numpy as np
import pandas as pd

from . import _device, _ingest
from .string_grouper import StringGrouper, block_ids_of, check_keys, factorise_keys

# options that define the vectoriser: fixed when the corpus is built
VECTORISER_OPTIONS = ("ngram_size", "regex", "ignore_case", "normalize_to_ascii", "tfidf_matrix_dtype")
IDENTITY_HINT = ("the corpus recognises its own Series by identity (`is`): pass the Series object the corpus was built "
                 "with, not an equal one (a column selected again from its DataFrame, df['name'], is a new object)")


class StringGrouperCorpus:
    """A TF-IDF corpus fitted once (K1), resident in HBM, that new Series are matched against.

    `kwargs` are StringGrouperConfig keys.  The vectoriser options among them are fixed here; the others are defaults
    that a method's own kwargs override.  A method argument that IS the corpus Series object (`is`) uses the corpus
    matrix itself: it is not vectorised again, and what K2 builds for it (row order, postings) carries over from call
    to call.

    `keys` (optional blocking keys of the corpus strings, a Series aligned by position): the corpus Series then
    always carries them, and passing keys of other values for it raises ValueError; the other argument of such a call
    needs keys of its own.  As for the matrix, the corpus Series is the object itself: keep it in a variable, a column
    selected again from a DataFrame is another Series without keys.  Keys of any other Series are mapped onto the corpus keys: equal values share an id with the
    corpus strings, values the corpus lacks share one among themselves, a missing key (None, NaN, pd.NA) matches
    nothing.  On a corpus without keys a keyed call factorises its keys like the module functions.
    """

    def __init__(self, strings: pd.Series, keys: Optional[pd.Series] = None, **kwargs):
        grouper = StringGrouper(strings, **kwargs)      # validates the Series and the options like StringGrouper
        self._keys = self._key_index = self._ids = self._d_ids = None
        if keys is not None:
            check_keys(strings, keys, 'keys')
            self._ids, uniques = factorise_keys(keys)
            self._key_index = pd.Index(uniques, tupleize_cols=False)
            self._n_ids = int(self._ids.max()) + 1 if len(self._ids) else 0
        self._matrix, _ = grouper._get_tf_idf_matrices(shard=False)    # ValueError on an empty vocabulary
        if keys is not None:
            self._keys = keys
            # one device tensor for the corpus rows: the blocked row order and postings are cached under it
            self._d_ids = _device.block_id_tensors(self._ids, len(self._ids), True)[0]
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

    @property
    def keys(self) -> Optional[pd.Series]:
        """The blocking keys the corpus was built with (None: none)."""
        return self._keys

    # ------------------------------------------------------------------ the reference's functions, on this corpus
    def fit(self, master: pd.Series, duplicates: Optional[pd.Series] = None, master_id: Optional[pd.Series] = None,
            duplicates_id: Optional[pd.Series] = None, *, master_keys: Optional[pd.Series] = None,
            duplicates_keys: Optional[pd.Series] = None, **kwargs) -> StringGrouper:
        """A fitted StringGrouper (get_matches, get_groups, add_match ...) whose matrices come from this corpus."""
        return self._grouper(master, duplicates, master_id, duplicates_id, master_keys=master_keys,
                             duplicates_keys=duplicates_keys, **kwargs).fit()

    def match_strings(self, master: pd.Series, duplicates: Optional[pd.Series] = None,
                      master_id: Optional[pd.Series] = None, duplicates_id: Optional[pd.Series] = None, *,
                      master_keys: Optional[pd.Series] = None, duplicates_keys: Optional[pd.Series] = None,
                      **kwargs) -> pd.DataFrame:
        return self.fit(master, duplicates, master_id, duplicates_id, master_keys=master_keys,
                        duplicates_keys=duplicates_keys, **kwargs).get_matches()

    def match_most_similar(self, master: pd.Series, duplicates: pd.Series, master_id: Optional[pd.Series] = None,
                           duplicates_id: Optional[pd.Series] = None, *, master_keys: Optional[pd.Series] = None,
                           duplicates_keys: Optional[pd.Series] = None, **kwargs) -> Union[pd.DataFrame, pd.Series]:
        kwargs['max_n_matches'] = 1
        return self.fit(master, duplicates, master_id, duplicates_id, master_keys=master_keys,
                        duplicates_keys=duplicates_keys, **kwargs).get_groups()

    def match_nearest(self, master: pd.Series, duplicates: pd.Series, master_id: Optional[pd.Series] = None,
                      duplicates_id: Optional[pd.Series] = None, *, master_keys: Optional[pd.Series] = None,
                      duplicates_keys: Optional[pd.Series] = None, **kwargs) -> Union[pd.DataFrame, pd.Series]:
        """match_nearest on this corpus.  With the corpus Series as `master` (a register lookup: which corpus entry
        is each incoming string?) the corpus matrix is the right operand, and its row order and postings carry over
        from call to call; on a keyed corpus so do its blocked order and postings (a keyed lookup needs only
        `duplicates_keys`)."""
        return self._grouper(master, duplicates, master_id, duplicates_id, master_keys=master_keys,
                             duplicates_keys=duplicates_keys, **kwargs)._match_nearest()

    def group_similar_strings(self, strings_to_group: pd.Series, string_ids: Optional[pd.Series] = None, *,
                              keys: Optional[pd.Series] = None, **kwargs) -> Union[pd.DataFrame, pd.Series]:
        return self.fit(strings_to_group, master_id=string_ids, master_keys=keys, **kwargs).get_groups()

    def compute_pairwise_similarities(self, string_series_1: pd.Series, string_series_2: pd.Series,
                                      **kwargs) -> pd.Series:
        return self._grouper(string_series_1, string_series_2, keyed=False, **kwargs).dot()

    # ------------------------------------------------------------------ internals
    def _grouper(self, master, duplicates=None, master_id=None, duplicates_id=None, *, master_keys=None,
                 duplicates_keys=None, keyed=True, **kwargs):
        options = self._config._asdict()
        options.update(kwargs)
        return _CorpusGrouper(self, keyed, master, duplicates, master_id, duplicates_id, master_keys=master_keys,
                              duplicates_keys=duplicates_keys, **options)

    def _block_ids(self, master, duplicates=None, master_keys=None, duplicates_keys=None):
        """int32 block id of every string of master ++ duplicates (None without keys), by the rules of the class
        docstring."""
        if self._keys is None:
            return block_ids_of(master, duplicates, master_keys, duplicates_keys)
        if duplicates_keys is not None and duplicates is None:
            raise ValueError('duplicates_keys needs duplicates')
        sides = [(master, master_keys, 'master')] + ([] if duplicates is None else [(duplicates, duplicates_keys,
                                                                                      'duplicates')])
        own = [s is self._series for s, _, _ in sides]
        for (strings, keys, name), is_corpus in zip(sides, own):
            if is_corpus:
                if keys is not None and not self._same_keys(keys):
                    raise ValueError(f'{name} is the corpus Series: its keys are the corpus keys, got {name}_keys '
                                     f'of other values')
            elif keys is not None:
                check_keys(strings, keys, f'{name}_keys')
        fresh = [(strings, keys, name) for (strings, keys, name), is_corpus in zip(sides, own) if not is_corpus]
        missing = [name for _, keys, name in fresh if keys is None]
        if missing and (any(own) or len(missing) < len(fresh)):
            raise ValueError(f'{missing[0]}_keys needed: the corpus has blocking keys, and {missing[0]} is not the '
                             f'corpus Series, so it carries none; {IDENTITY_HINT}')
        if missing:
            return None
        mapped = iter(self._map_keys([keys for _, keys, _ in fresh]) if fresh else ())
        return np.concatenate([self._ids if is_corpus else next(mapped) for is_corpus in own]).astype(np.int32)

    def _same_keys(self, keys):
        """True when `keys` holds the corpus keys' values by position, whatever its dtype or index: the same corpus id
        for every present value, missing where the corpus keys are missing."""
        if len(keys) != len(self._keys):
            return False
        present = self._ids < len(self._key_index)
        codes = self._key_index.get_indexer(keys)
        return bool(np.array_equal(codes, np.where(present, self._ids, -1))
                    and np.array_equal(keys.isna().to_numpy(), ~present))

    def _map_keys(self, keys_list):
        """The int32 ids of other Series' keys (a list, one array each): the corpus id of every value the corpus
        has; after the corpus ids, the values it lacks factorised among themselves (over all the Series given), then
        one id per missing value."""
        keys = pd.concat(keys_list, ignore_index=True)
        codes = self._key_index.get_indexer(keys).astype(np.int64)
        new = codes < 0
        ids, _ = factorise_keys(keys[new], first_id=self._n_ids)
        codes[new] = ids
        return np.split(codes.astype(np.int32), np.cumsum([len(k) for k in keys_list])[:-1])

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

    def __init__(self, corpus, keyed, *args, **kwargs):
        self._corpus = corpus
        self._keyed = keyed         # compute_pairwise_similarities takes no keys
        super().__init__(*args, **kwargs)

    def _set_data(self, master, duplicates=None, master_id=None, duplicates_id=None, master_keys=None,
                  duplicates_keys=None):
        super()._set_data(master, duplicates, master_id, duplicates_id)
        if self._keyed:
            self._block_ids = self._corpus._block_ids(master, duplicates, master_keys, duplicates_keys)

    def _block_id_tensors(self, n_left, self_match):
        corpus = self._corpus
        if corpus._d_ids is None or not (self._master is corpus._series or self._duplicates is corpus._series):
            return super()._block_id_tensors(n_left, self_match)
        # a side that is the corpus Series takes the corpus tensor itself, under which its blocked order is cached

        def side(strings, ids):
            return corpus._d_ids if strings is corpus._series else _device.block_id_tensors(ids, len(ids), True)[0]
        left = side(self._master, self._block_ids[:n_left])
        return (left, left) if self._duplicates is None else (left, side(self._duplicates, self._block_ids[n_left:]))

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

"""Host-side mirror of the reference interface for the hot path, calling the sm_90a kernels.

Drop-in for `string_grouper.string_grouper` of Bergvca/string_grouper @ 270044e9
(string_grouper/string_grouper.py, cited below as "ref:<line>"):
same public names, keyword arguments, column labels, exceptions and result
ordering.  What differs is where the arithmetic runs:

    ref:365-378 + 685-707   analyzer + TfidfVectorizer      -> K1  (csrc/sg_tfidf.cu)
    ref:709-752             _build_matches / sparse_dot_topn -> K2  (csrc/sg_cossim.cu)
    ref:419-427, 955-964    LIL fix-diagonal + symmetrise    -> K4  (csrc/sg_symm.cu)
    ref:433-440             dot()                            -> sg_rowwise_dot

There is no CPU fallback: without libsg_b200.so and a CUDA device `fit()` raises.
Everything below the kernels (pandas result shaping) is host glue re-written
for vectorised numpy/pandas; its behaviour is pinned by tests/golden/.
"""
import multiprocessing
import re
from functools import wraps
from typing import List, NamedTuple, Optional, Tuple, Union
from unicodedata import normalize

import numpy as np
import pandas as pd
from loguru import logger
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import connected_components

from . import _device, _dist, _ingest

DEFAULT_NGRAM_SIZE: int = 3
DEFAULT_TFIDF_MATRIX_DTYPE: type = np.float64
DEFAULT_REGEX: str = r'[,-./]|\s'
DEFAULT_MAX_N_MATCHES: int = 20
DEFAULT_MIN_SIMILARITY: float = 0.8
DEFAULT_N_PROCESSES: int = multiprocessing.cpu_count() - 1
DEFAULT_IGNORE_CASE: bool = True
DEFAULT_DROP_INDEX: bool = False
DEFAULT_REPLACE_NA: bool = False
DEFAULT_INCLUDE_ZEROES: bool = True
GROUP_REP_CENTROID: str = 'centroid'
GROUP_REP_FIRST: str = 'first'
DEFAULT_GROUP_REP: str = GROUP_REP_CENTROID
DEFAULT_FORCE_SYMMETRIES: bool = True
DEFAULT_N_BLOCKS: Optional[Tuple[int, int]] = None
DEFAULT_NORMALIZE_TO_ASCII: bool = True

DEFAULT_COLUMN_NAME: str = 'side'
DEFAULT_ID_NAME: str = 'id'
LEFT_PREFIX: str = 'left_'
RIGHT_PREFIX: str = 'right_'
MOST_SIMILAR_PREFIX: str = 'most_similar_'
DEFAULT_MASTER_NAME: str = 'master'
DEFAULT_MASTER_ID_NAME: str = f'{DEFAULT_MASTER_NAME}_{DEFAULT_ID_NAME}'
GROUP_REP_PREFIX: str = 'group_rep_'


class StringGrouperConfig(NamedTuple):
    """Keyword options, same names and defaults as ref:156-202.

    `number_of_processes` is accepted for compatibility and ignored (the product runs on the GPU);
    `n_blocks` is validated like the reference, but the result does not depend on it (the kernel picks
    its own column tiles; the reference's own tests pin this invariance, ref test file :191-336).
    """
    ngram_size: int = DEFAULT_NGRAM_SIZE
    tfidf_matrix_dtype: type = DEFAULT_TFIDF_MATRIX_DTYPE
    regex: str = DEFAULT_REGEX
    max_n_matches: Optional[int] = DEFAULT_MAX_N_MATCHES
    min_similarity: float = DEFAULT_MIN_SIMILARITY
    number_of_processes: int = DEFAULT_N_PROCESSES
    ignore_case: bool = DEFAULT_IGNORE_CASE
    ignore_index: bool = DEFAULT_DROP_INDEX
    include_zeroes: bool = DEFAULT_INCLUDE_ZEROES
    replace_na: bool = DEFAULT_REPLACE_NA
    group_rep: str = DEFAULT_GROUP_REP
    force_symmetries: bool = DEFAULT_FORCE_SYMMETRIES
    n_blocks: Optional[Tuple[int, int]] = DEFAULT_N_BLOCKS
    normalize_to_ascii: bool = DEFAULT_NORMALIZE_TO_ASCII


class StringGrouperNotFitException(Exception):
    """A result was requested before fit() (ref:219-221)."""


def validate_is_fit(method):
    @wraps(method)
    def guarded(self, *args, **kwargs):
        if not self.is_build:
            raise StringGrouperNotFitException(
                f'{method.__name__} was called before the "fit" function was called. '
                f'Make sure to run fit the StringGrouper first using StringGrouper.fit()')
        return method(self, *args, **kwargs)
    return guarded


# ------------------------------------------------------------------ module-level entry points (ref:55-153)

def compute_pairwise_similarities(string_series_1: pd.Series, string_series_2: pd.Series, **kwargs) -> pd.Series:
    """Row-wise cosine similarity of two equally long Series (ref:55-67)."""
    return StringGrouper(string_series_1, string_series_2, **kwargs).dot()


def group_similar_strings(strings_to_group: pd.Series, string_ids: Optional[pd.Series] = None,
                          **kwargs) -> Union[pd.DataFrame, pd.Series]:
    """Group representative for every string (ref:70-92)."""
    return StringGrouper(strings_to_group, master_id=string_ids, **kwargs).fit().get_groups()


def match_most_similar(master: pd.Series, duplicates: pd.Series, master_id: Optional[pd.Series] = None,
                       duplicates_id: Optional[pd.Series] = None, **kwargs) -> Union[pd.DataFrame, pd.Series]:
    """Most similar master string for every duplicate; forces max_n_matches=1 like ref:120."""
    kwargs['max_n_matches'] = 1
    return StringGrouper(master, duplicates=duplicates, master_id=master_id, duplicates_id=duplicates_id,
                         **kwargs).fit().get_groups()


def match_strings(master: pd.Series, duplicates: Optional[pd.Series] = None, master_id: Optional[pd.Series] = None,
                  duplicates_id: Optional[pd.Series] = None, **kwargs) -> pd.DataFrame:
    """All pairs with cosine similarity above min_similarity (ref:130-153)."""
    return StringGrouper(master, duplicates=duplicates, master_id=master_id, duplicates_id=duplicates_id,
                         **kwargs).fit().get_matches()


class StringGrouper(object):
    def __init__(self, master: pd.Series, duplicates: Optional[pd.Series] = None,
                 master_id: Optional[pd.Series] = None, duplicates_id: Optional[pd.Series] = None, **kwargs):
        self.is_build = False
        self._master = pd.Series(dtype=object)
        self._duplicates = None
        self._master_id = None
        self._duplicates_id = None
        self._left_Series = self._master
        self._right_Series = self._master
        self._matches_list = pd.DataFrame()
        self._true_max_n_matches = 0
        self._max_n_matches = 0
        self._config = StringGrouperConfig(**kwargs)
        self._n_blocks = self._config.n_blocks
        self._vocabulary = None          # device df / rank tables of the last fit (K1)
        self._matches_device = None      # match list in HBM as long as it equals _matches_list
        self._raw_device = None          # the callers' strings in HBM (packed UTF-8) when ingest left them untouched
        self._last_stats = {}
        self._set_data(master, duplicates, master_id, duplicates_id)
        self._set_options(**kwargs)
        # ref:267 fits a vectoriser here and again in fit() (SURVEY §0 fact 9); the second fit gives the
        # identical vocabulary, so the device vectoriser runs once, inside fit().

    # ------------------------------------------------------------------ data / options (ref:269-363)
    def _set_data(self, master, duplicates=None, master_id=None, duplicates_id=None):
        self.master = master
        self.duplicates = duplicates
        if not StringGrouper._is_input_data_combination_valid(duplicates, master_id, duplicates_id):
            raise Exception('List of data Series options is invalid')
        StringGrouper._validate_id_data(master, duplicates, master_id, duplicates_id)
        self._master_id = master_id
        self._duplicates_id = duplicates_id
        self._left_Series = self._master
        self._right_Series = self._master if self._duplicates is None else self._duplicates
        self.is_build = False

    def _set_options(self, **kwargs):
        self._config = StringGrouperConfig(**kwargs)
        self._max_n_matches = self._config.max_n_matches
        self._validate_group_rep_specs()
        self._validate_tfidf_matrix_dtype()
        self._validate_replace_na_and_drop()
        StringGrouper._validate_n_blocks(self._config.n_blocks)
        self.is_build = False

    def reset_data(self, master, duplicates=None, master_id=None, duplicates_id=None):
        """Replace the input Series, keeping the options (ref:310-323)."""
        self._set_data(master, duplicates, master_id, duplicates_id)

    def clear_data(self):
        self._master = None
        self._duplicates = None
        self._master_id = None
        self._duplicates_id = None
        self._matches_list = None
        self._left_Series = None
        self._right_Series = None
        self.is_build = False

    def update_options(self, **kwargs):
        """Merge new keyword options over the current ones (ref:335-343)."""
        StringGrouperConfig(**kwargs)      # rejects unknown keys exactly like the reference
        merged = self._config._asdict()
        merged.update(kwargs)
        self._set_options(**merged)

    @property
    def master(self):
        return self._master

    @master.setter
    def master(self, master):
        if not StringGrouper._is_series_of_strings(master):
            raise TypeError('Master input does not consist of pandas.Series containing only Strings')
        self._master = master

    @property
    def duplicates(self):
        return self._duplicates

    @duplicates.setter
    def duplicates(self, duplicates):
        if duplicates is not None and not StringGrouper._is_series_of_strings(duplicates):
            raise TypeError('Duplicates input does not consist of pandas.Series containing only Strings')
        self._duplicates = duplicates

    # ------------------------------------------------------------------ analyzer (host copy, ref:365-378)
    def n_grams(self, string: str) -> List[str]:
        """Host statement of the analyzer the device kernel implements; used for inspection and tests."""
        n = self._config.ngram_size
        if self._config.ignore_case and string is not None:
            string = string.lower()
        if self._config.normalize_to_ascii:
            string = normalize('NFKD', string).encode('ASCII', 'ignore').decode()
        string = re.sub(self._config.regex, r'', string)
        return [string[i:i + n] for i in range(len(string) - n + 1)]

    # ------------------------------------------------------------------ the hot path
    def fit(self):
        """Vectorise, match, post-process; fills `_matches_list` (ref:380-431)."""
        master_matrix, duplicate_matrix = self._get_tf_idf_matrices()

        guess = (max(1, round(len(self._left_Series) / 1e6)), max(1, round(len(self._right_Series) / 4e3)))
        if self._n_blocks is None:
            self._n_blocks = guess

        if self._n_blocks == (1, 1):
            try:
                matches = self._build_matches(master_matrix, duplicate_matrix, self._n_blocks)
            except OverflowError:
                # same control flow as ref:397-413 (its tests mock _build_matches to fail for (1, 1) only).  The
                # device path sizes its own tiles and row chunks, so n_blocks cannot shrink its buffers: a second
                # OverflowError from the real kernel path is final (raise min_similarity or split the input).
                logger.warning("An OverflowError occurred; retrying with the reference's block guess n_blocks = ("
                               + str(guess[0]) + "," + str(guess[1]) + ")")
                matches = self._build_matches(master_matrix, duplicate_matrix, guess)
        else:
            matches = self._build_matches(master_matrix, duplicate_matrix, self._n_blocks)

        matches = _device.as_device_matches(matches)
        self._true_max_n_matches = matches.max_row

        rank, world_size = _dist.world()
        if world_size > 1 and rank != 0 and not _dist.result_on_all_ranks():
            # SG_B200_RESULT=rank0: this rank took part in the product; the match list lives on rank 0 only
            matches = _device.as_device_matches(csr_matrix(matches.shape, dtype=np.float64))
        elif self._config.force_symmetries and self._duplicates is None:
            matches = StringGrouper._fix_diagonal(matches)
            matches = StringGrouper._symmetrize_matrix(matches)
            matches = _device.apply_pending(matches)

        self._matches_list = self._get_matches_list(matches)
        self._matches_device = matches if hasattr(matches, "d_row") else None   # HBM copy for get_groups()
        self.is_build = True
        return self

    def dot(self) -> pd.Series:
        """Row-wise similarity of master and duplicates (ref:433-440)."""
        if len(self._master) != len(self._duplicates):
            raise Exception("To perform this function, both input Series must have the same length.")
        master_matrix, duplicate_matrix = self._get_tf_idf_matrices(shard=False)
        sims = _device.rowwise_dot(_device.as_device_csr(master_matrix), _device.as_device_csr(duplicate_matrix))
        return pd.Series(sims, name='similarity', index=self._master.index)

    def _get_tf_idf_matrices(self, shard=True):
        """(master_matrix, duplicate_matrix) as HBM-resident CSR (ref:685-697).

        The vocabulary / idf are fitted on master ++ duplicates (ref:699-707); with no duplicates the second
        matrix IS the first (ref:695).  The returned objects answer `.toarray()`, `.shape`, `.indptr` ...
        like scipy matrices (materialised on demand).
        """
        cfg = self._config
        series = [self._master] if self._duplicates is None else [self._master, self._duplicates]
        rank, world_size = _dist.world()
        if shard and world_size > 1:
            # sharding is opt-in (SG_B200_DISTRIBUTED); every rank must hold the same input Series
            _dist.check_same_inputs(_dist.fingerprint(series) + [int(cfg.ngram_size), int(bool(cfg.ignore_case))])
        approx_bytes = (sum(int(s.str.len().sum()) for s in series)
                        if shard and world_size > 1 and len(series) == 2 else 0)
        stats = {}
        if (shard and world_size > 1 and len(series) == 2 and cfg.ngram_size <= 3 and cfg.normalize_to_ascii
                and _dist.shard_vectorise(approx_bytes)):
            # two Series over several GPUs: every rank vectorises only its blocks of master and duplicates rows;
            # document frequencies are all-reduced (NCCL), the duplicate matrix is all-gathered over NVLink,
            # the master block stays local and is this rank's share of the left rows of _build_matches.
            n_m, n_d = len(self._master), len(self._duplicates)
            mlo, mhi = _dist.shard_range(n_m, rank, world_size)
            dlo, dhi = _dist.shard_range(n_d, rank, world_size)
            local = [self._master.iloc[mlo:mhi], self._duplicates.iloc[dlo:dhi]]
            data, offsets, flags, _ = _dist.guarded(_ingest.pack_strings, local, cfg.regex, cfg.ignore_case,
                                                    cfg.normalize_to_ascii)
            master, dup, vocab = _device.tfidf(data, offsets, mhi - mlo, cfg.ngram_size, flags,
                                               cfg.tfidf_matrix_dtype, stats=stats,
                                               df_allreduce=_dist.allreduce_sum_, n_docs_fit=n_m + n_d)
            if dup is None:      # this rank holds no duplicate rows: an empty block still takes part in the gather
                dup = _device.empty_csr(master, 0)
            dup = _device.allgather_csr(dup, n_d)
            master.row_offset, master.global_rows = mlo, n_m
            stats["sharded_vectorise"] = True
            stats.pop("raw", None)           # only this rank's blocks of the strings are on the device
        else:
            data, offsets, flags, pristine = _ingest.pack_strings(series, cfg.regex, cfg.ignore_case,
                                                                  cfg.normalize_to_ascii)
            master, dup, vocab = _device.tfidf(data, offsets, len(self._master), cfg.ngram_size, flags,
                                               cfg.tfidf_matrix_dtype, stats=stats)
            if not pristine:
                stats.pop("raw", None)       # the device bytes are normalised text, not the callers' strings
        if master.shape[1] == 0:
            # sklearn raises this from TfidfVectorizer.fit (the reference hits it in __init__, ref:267/:305-308)
            raise ValueError("empty vocabulary; perhaps the documents only contain stop words")
        self._vocabulary = vocab
        self._last_stats = stats
        self._raw_device = stats.pop("raw", None)
        return master, (master if dup is None else dup)

    def _build_matches(self, master_matrix, duplicate_matrix, n_blocks=None):
        """top-n thresholded master x duplicates^T (ref:709-752) on the device.

        Accepts the HBM matrices of _get_tf_idf_matrices or any scipy CSR.  `n_blocks` only decides the value
        dtype like the reference (None -> matrix dtype, ref:724-732; otherwise float64, ref:750); the block
        split itself is replaced by the kernel's own column tiles and does not change the result.
        """
        A = _device.as_device_csr(master_matrix)
        B = A if duplicate_matrix is master_matrix else _device.as_device_csr(duplicate_matrix)
        rank, world_size = _dist.world()
        if world_size > 1 and getattr(A, "row_offset", None) is not None:
            # K1 was sharded: A already IS this rank's block of left rows.  The rank-local product runs guarded: a
            # rank that fails (OverflowError ...) tells the others before anybody enters the gather.
            out = _dist.guarded(_device.cossim_topn, A, B, self._max_n_matches, self._config.min_similarity,
                                stats=self._last_stats)
            out = _device.offset_rows(out, A.row_offset, A.global_rows)
            out = _device.gather_shards(out)
        elif world_size > 1:
            # one process per GPU: this rank computes its block of left rows, the blocks are all-gathered
            lo, hi = _dist.shard_range(A.shape[0], rank, world_size)
            out = _dist.guarded(_device.cossim_topn, A, B, self._max_n_matches, self._config.min_similarity,
                                row_begin=lo, row_end=hi, stats=self._last_stats)
            out = _device.gather_shards(out)
        else:
            out = _device.cossim_topn(A, B, self._max_n_matches, self._config.min_similarity,
                                      stats=self._last_stats)
        if n_blocks is not None and A.dtype != np.float64:
            # ref:750 `vstack(Czip, dtype=np.float64)`: scipy's astype() de-duplicates when the dtype changes,
            # which re-orders every row by ascending column — float32 runs of the reference come out that way.
            out = _device.symmetrize(out, fix_diagonal=False, mirror=False)
        out.out_dtype = np.dtype(A.dtype if n_blocks is None else np.float64)
        return out

    def _get_matches_list(self, matches) -> pd.DataFrame:
        """(master_side, dupe_side, similarity) in storage order (ref:755-763)."""
        if isinstance(matches, _device.DeviceMatches):
            r, c, s = matches.host_triples()
        else:
            m = matches.tocsr()
            r, c = m.nonzero()
            s = m.data
        return pd.DataFrame({'master_side': np.asarray(r).astype(np.int64, copy=False),
                             'dupe_side': np.asarray(c).astype(np.int64, copy=False),
                             'similarity': np.asarray(s)}, copy=False)

    @staticmethod
    def _fix_diagonal(m):
        """Diagonal := 1 (ref:955-958); recorded on the device result and applied by the fused K4 launch."""
        m = _device.as_device_matches(m)
        return m.with_pending(fix_diagonal=True)

    @staticmethod
    def _symmetrize_matrix(m):
        """Pattern := pattern U pattern^T (ref:961-964); fused with _fix_diagonal in one K4 launch."""
        m = _device.as_device_matches(m)
        return m.with_pending(mirror=True)

    # ------------------------------------------------------------------ results
    @validate_is_fit
    def get_matches(self, ignore_index: Optional[bool] = None, include_zeroes: Optional[bool] = None) -> pd.DataFrame:
        """Matches as a DataFrame, same columns and order as ref:443-518."""
        if ignore_index is None:
            ignore_index = self._config.ignore_index
        if include_zeroes is None:
            include_zeroes = self._config.include_zeroes
        pairs = self._matches_list
        if not (self._config.min_similarity > 0 or not include_zeroes):
            zeros = self._get_non_matches_list()
            if not zeros.empty:
                pairs = pd.concat([pairs, zeros], axis=0, ignore_index=True)

        lpos = pairs.master_side.to_numpy()
        rpos = pairs.dupe_side.to_numpy()
        right_strings = self._master if self._duplicates is None else self._duplicates
        lvals = rvals = None
        dev, raw = self._matches_device, self._raw_device
        if (dev is not None and raw is not None and pairs is self._matches_list and len(pairs) == dev.nnz
                and _is_arrow_str(self._master) and _is_arrow_str(right_strings)
                and raw.n_master == len(self._master)):
            # strings and match positions are both in HBM: gather there, wrap the result as Arrow arrays
            rbase = 0 if self._duplicates is None else raw.n_master
            lhost, rhost = _device.gather_strings(raw, [(0, dev.d_row, dev.nnz), (rbase, dev.d_col, dev.nnz)])
            lvals = _gathered_array(self._master, *lhost)
            rvals = _gathered_array(right_strings, *rhost)
        sides = [(self._master, lpos, DEFAULT_COLUMN_NAME, ignore_index, LEFT_PREFIX, False, lvals),
                 (right_strings, rpos, DEFAULT_COLUMN_NAME, ignore_index, RIGHT_PREFIX, True, rvals)]
        if self._master_id is not None:
            right_ids = self._master_id if self._duplicates is None else self._duplicates_id
            sides.insert(1, (self._master_id, lpos, DEFAULT_ID_NAME, True, LEFT_PREFIX, False, None))
            sides.insert(2, (right_ids, rpos, DEFAULT_ID_NAME, True, RIGHT_PREFIX, True, None))
        # fast path (millions of matches): every side reduces to plain columns -> ONE DataFrame construction
        cols = [_side_columns(*sd) for sd in sides]
        if all(c is not None for c in cols):
            half = len(cols) // 2
            flat = [kv for c in cols[:half] for kv in c] + [('similarity', pairs.similarity.to_numpy())] + \
                   [kv for c in cols[half:] for kv in c]
            if len({k for k, _ in flat}) == len(flat):
                return pd.DataFrame(dict(flat), copy=False)
        frames = [_take_side(*sd[:6], values=sd[6]) for sd in sides]
        similarity = pairs.similarity.reset_index(drop=True)
        half = len(frames) // 2
        return pd.concat(frames[:half] + [similarity] + frames[half:], axis=1)

    @validate_is_fit
    def get_groups(self, ignore_index: Optional[bool] = None,
                   replace_na: Optional[bool] = None) -> Union[pd.DataFrame, pd.Series]:
        """Group representatives (self-match) or nearest master per duplicate (ref:520-544)."""
        if ignore_index is None:
            ignore_index = self._config.ignore_index
        if self._duplicates is None:
            return self._deduplicate(ignore_index=ignore_index)
        if replace_na is None:
            replace_na = self._config.replace_na
        return self._get_nearest_matches(ignore_index=ignore_index, replace_na=replace_na)

    # corpus-reusing variants (ref:546-644); like the reference they refit on the new data
    def match_strings(self, master, duplicates=None, master_id=None, duplicates_id=None, **kwargs) -> pd.DataFrame:
        self.reset_data(master, duplicates, master_id, duplicates_id)
        self.update_options(**kwargs)
        return self.fit().get_matches()

    def match_most_similar(self, master, duplicates, master_id=None, duplicates_id=None, **kwargs):
        self.reset_data(master, duplicates, master_id, duplicates_id)
        self.update_options(**kwargs)
        return self.fit().get_groups()

    def group_similar_strings(self, strings_to_group, string_ids=None, **kwargs):
        self.reset_data(strings_to_group, master_id=string_ids)
        self.update_options(**kwargs)
        return self.fit().get_groups()

    def compute_pairwise_similarities(self, string_series_1, string_series_2, **kwargs) -> pd.Series:
        self.reset_data(string_series_1, string_series_2)
        self.update_options(**kwargs)
        return self.dot()

    # ------------------------------------------------------------------ manual edits (ref:646-683)
    @validate_is_fit
    def add_match(self, master_side: str, dupe_side: str) -> 'StringGrouper':
        """Force a match between two strings (all their occurrences), keeping self-matches symmetric."""
        master_idx, dupe_idx = self._get_indices_of(master_side, dupe_side)
        prior = self._matches_list.master_side[self._matches_list.dupe_side.isin(dupe_idx)]
        dupe_idx = pd.concat([dupe_idx, prior]).drop_duplicates()
        grid = pd.MultiIndex.from_product([master_idx, dupe_idx, [1]],
                                          names=['master_side', 'dupe_side', 'similarity'])
        new = pd.DataFrame(index=grid).reset_index()
        if self._duplicates is None:
            new = pd.concat([new, new.rename(columns={'master_side': 'dupe_side', 'dupe_side': 'master_side'})[
                ['master_side', 'dupe_side', 'similarity']]])
        self._matches_list = pd.concat([self._matches_list.drop_duplicates(), new], ignore_index=True)
        self._matches_device = None
        return self

    @validate_is_fit
    def remove_match(self, master_side: str, dupe_side: str) -> 'StringGrouper':
        master_idx, dupe_idx = self._get_indices_of(master_side, dupe_side)
        if self._duplicates is None:
            master_idx = pd.concat([master_idx, dupe_idx])
            dupe_idx = master_idx
        hit = self._matches_list.master_side.isin(master_idx) & self._matches_list.dupe_side.isin(dupe_idx)
        self._matches_list = self._matches_list[~hit]
        self._matches_device = None
        return self

    # ------------------------------------------------------------------ result shaping helpers
    def _get_non_matches_list(self) -> pd.DataFrame:
        """Pairs absent from the match list, similarity 0 (ref:765-781); O(n_left*n_right), tiny inputs only."""
        n_left = len(self._master)
        n_right = len(self._master if self._duplicates is None else self._duplicates)
        seen = np.zeros(n_left * n_right, dtype=bool)
        seen[self._matches_list.master_side.to_numpy() * n_right + self._matches_list.dupe_side.to_numpy()] = True
        missing = np.nonzero(~seen)[0]
        if missing.size == 0:
            return pd.DataFrame()
        if self._max_n_matches < self._true_max_n_matches:
            raise Exception(f'\nERROR: Cannot return zero-similarity matches since \n'
                            f'\t\t max_n_matches={self._max_n_matches} is too small!\n'
                            f'\t\t Try setting max_n_matches={self._true_max_n_matches} (the \n'
                            f'\t\t true maximum number of matches over all strings in master)\n'
                            f'\t\t or greater or do not set this kwarg at all.')
        return pd.DataFrame({'master_side': missing // n_right, 'dupe_side': missing % n_right, 'similarity': 0})

    def _get_nearest_matches(self, ignore_index=False, replace_na=False) -> Union[pd.DataFrame, pd.Series]:
        """For each duplicate: the master with the highest similarity, lowest index on ties; the duplicate
        itself when nothing matched (ref:783-849)."""
        prefix = MOST_SIMILAR_PREFIX
        master_label = f'{prefix}{self._master.name if self._master.name else DEFAULT_MASTER_NAME}'
        n_dup = len(self._duplicates)
        pairs = self._matches_list
        best = np.full(n_dup, -1, dtype=np.int64)
        dev = self._matches_device
        if dev is not None and len(pairs) == dev.nnz and n_dup > 0:
            # the match list is still in HBM: arg-max per duplicate there (csrc/sg_groups.cu)
            best = _device.nearest_master(dev, n_dup)
        elif len(pairs):
            d = pairs.dupe_side.to_numpy()
            m = pairs.master_side.to_numpy()
            s = pairs.similarity.to_numpy()
            order = np.lexsort((m, -s, d))          # per duplicate: similarity desc, then master index asc
            first = np.ones(len(order), dtype=bool)
            first[1:] = d[order][1:] != d[order][:-1]
            best[d[order][first]] = m[order][first]
        hit = best >= 0
        pos = np.where(hit, best, 0)
        hit_s = pd.Series(hit)

        def nullable(values):
            # masked extension dtypes (Int64, boolean ...) survive the reference's merges un-widened (ref:812-813)
            return isinstance(values.dtype, pd.api.extensions.ExtensionDtype) and \
                not isinstance(values.dtype, pd.StringDtype)

        def pick(master_series, dupe_series):
            # value of the matched master row, the duplicate's own value where nothing matched (ref:815-820)
            if nullable(master_series):
                taken = pd.Series(master_series.array.take(pos))
                return taken.where(hit_s, pd.Series(dupe_series.array))
            taken = pd.Series(master_series.to_numpy()[pos])
            return taken.where(hit_s, pd.Series(dupe_series.to_numpy()))

        columns = {}
        if not ignore_index:
            m_idx = self._master.index.to_frame(index=False)
            d_idx = self._duplicates.index.to_frame(index=False)
            m_names = self._master.reset_index(drop=False).columns[:-1]
            for k, col in enumerate(m_names):
                level = m_idx.iloc[:, k]
                if nullable(level):
                    vals = pd.Series(level.array.take(pos)).where(hit_s, pd.NA)
                    if replace_na:
                        vals = vals.where(hit_s, pd.Series(d_idx.iloc[:, k].array))
                else:
                    vals = pd.Series(level.to_numpy()[pos]).where(hit_s, np.nan)
                    if replace_na:
                        # ref:834-843; the dtype "restore" there assigns through .loc and therefore keeps the
                        # NaN-widened dtype on current pandas, so none is attempted here either
                        vals = vals.where(hit_s, pd.Series(d_idx.iloc[:, k].to_numpy()))
                columns[f'{prefix}{col}'] = vals
        if self._master_id is not None:
            id_label = f'{prefix}{self._master_id.name if self._master_id.name else DEFAULT_MASTER_ID_NAME}'
            columns[id_label] = pick(self._master_id, self._duplicates_id)
        columns[master_label] = pick(self._master, self._duplicates)
        out = pd.DataFrame(columns)
        out.index = self._duplicates.index
        return out.squeeze(axis=1)

    def _deduplicate(self, ignore_index=False) -> Union[pd.DataFrame, pd.Series]:
        """Connected components of the match graph, one representative per group (ref:851-904)."""
        n = len(self._master)
        centroid = self._config.group_rep == GROUP_REP_CENTROID
        rep_values = None
        if self._matches_device is not None:
            # components, similarity sums and representatives on the device (csrc/sg_groups.cu)
            rep, d_rep = _device.group_reps(self._matches_device, n, centroid, keep_device=True)
            raw = self._raw_device
            if raw is not None and n > 0 and _is_arrow_str(self._master) and raw.n_master == n:
                # the strings are in HBM too: gather the representatives there (the Series.iloc of ref:897)
                (rhost,) = _device.gather_strings(raw, [(0, d_rep, n)])
                rep_values = _gathered_array(self._master, *rhost)
        else:
            # the list was edited by add_match / remove_match: host statement of the same rule
            pairs = self._matches_list
            rows, cols = pairs.master_side.to_numpy(), pairs.dupe_side.to_numpy()
            graph = csr_matrix((np.full(len(pairs), 1), (rows, cols)), shape=(n, n))
            _, group = connected_components(csgraph=graph, directed=True)
            if centroid:
                graph.data = pairs['similarity'].to_numpy()
                weight = np.asarray(graph.sum(axis=1)).squeeze(axis=1)
                order = np.lexsort((np.arange(n), -weight, group))   # per group: weight desc, first index on ties
            else:
                order = np.lexsort((np.arange(n), group))            # per group: first index
            head = np.ones(n, dtype=bool)
            head[1:] = group[order][1:] != group[order][:-1]
            rep_of_group = np.empty(group.max() + 1 if n else 0, dtype=np.int64)
            rep_of_group[group[order][head]] = order[head]
            rep = rep_of_group[group]

        prefix = GROUP_REP_PREFIX
        label = f'{prefix}{self._master.name}' if self._master.name else prefix[:-1]
        index = self._master.index
        if rep_values is not None and (ignore_index or (index.nlevels == 1 and index.name is None and label != 'index')):
            # fast path: the gathered strings become the column directly (same frame as the general path below)
            if ignore_index:
                output = pd.Series(rep_values, name=label, copy=False)
            else:
                if isinstance(index, pd.RangeIndex):
                    labels = rep if (index.start == 0 and index.step == 1) else index.start + index.step * rep
                else:
                    labels = index.to_numpy()[rep]
                output = pd.DataFrame({'index': labels, label: rep_values}, copy=False)
        else:
            output = self._master.iloc[rep].rename(label).reset_index(drop=ignore_index)
        if isinstance(output, pd.DataFrame):
            output.rename(columns={c: f'{prefix}{c}' for c in output.columns if str(c) != label}, inplace=True)
        if self._master_id is not None:
            id_label = f'{prefix}{self._master_id.name if self._master_id.name else DEFAULT_ID_NAME}'
            output = pd.concat([self._master_id.iloc[rep].rename(id_label).reset_index(drop=True), output], axis=1)
        output.index = self._master.index
        return output

    def _get_indices_of(self, master_side: str, dupe_side: str) -> Tuple[pd.Series, pd.Series]:
        master_strings = self._master
        dupe_strings = self._master if self._duplicates is None else self._duplicates
        if not master_strings.isin([master_side]).any():
            raise ValueError(f'{master_side} not found in StringGrouper string series')
        if not dupe_strings.isin([dupe_side]).any():
            raise ValueError(f'{dupe_side} not found in StringGrouper dupe string series')
        master_idx = master_strings[master_strings == master_side].index.to_series().reset_index(drop=True)
        dupe_idx = dupe_strings[dupe_strings == dupe_side].index.to_series().reset_index(drop=True)
        return master_idx, dupe_idx

    # ------------------------------------------------------------------ validators (ref:916-1010)
    def _validate_group_rep_specs(self):
        options = (GROUP_REP_FIRST, GROUP_REP_CENTROID)
        if self._config.group_rep not in options:
            raise Exception(f"Invalid option value for group_rep. The only permitted values are\n {options}")

    def _validate_tfidf_matrix_dtype(self):
        options = (np.float32, np.float64)
        if self._config.tfidf_matrix_dtype not in options:
            raise Exception(f"Invalid option value for tfidf_matrix_dtype. The only permitted values are\n {options}")

    def _validate_replace_na_and_drop(self):
        if self._config.ignore_index and self._config.replace_na:
            raise Exception("replace_na can only be set to True when ignore_index=False.")
        if self._config.replace_na and self._master.index.nlevels != self._duplicates.index.nlevels:
            raise Exception("replace_na=True: Cannot replace NaN values of index-columns with the values of another "
                            "index if the number of index-levels does not equal the number of index-columns.")

    @staticmethod
    def _validate_n_blocks(n_blocks):
        if n_blocks is None:
            return
        ok = (isinstance(n_blocks, tuple) and len(n_blocks) == 2
              and all(isinstance(b, int) for b in n_blocks) and min(n_blocks) >= 1)
        if not ok:
            raise Exception("Invalid option value for parameter n_blocks: n_blocks must be None or a tuple of 2 "
                            "integers greater than 0.")

    @staticmethod
    def _is_series_of_strings(series_to_test) -> bool:
        return _ingest.is_series_of_strings(series_to_test)

    @staticmethod
    def _is_input_data_combination_valid(duplicates, master_id, duplicates_id) -> bool:
        if duplicates is None:
            return duplicates_id is None
        return (master_id is None) == (duplicates_id is None)

    @staticmethod
    def _validate_id_data(master, duplicates, master_id, duplicates_id):
        if master_id is not None and len(master) != len(master_id):
            raise Exception('Both master and master_id must be pandas.Series of the same length.')
        if duplicates is not None and duplicates_id is not None and len(duplicates) != len(duplicates_id):
            raise Exception('Both duplicates and duplicates_id must be pandas.Series of the same length.')


def _is_arrow_str(series):
    return isinstance(series.dtype, pd.StringDtype) and hasattr(series.array, "_pa_array")


def _gathered_array(series, offsets, data):
    """(offsets, bytes) of gathered strings -> an extension array of the Series' own dtype, zero-copy."""
    import pyarrow as pa
    n = len(offsets) - 1
    arr = pa.LargeStringArray.from_buffers(n, pa.py_buffer(offsets), pa.py_buffer(data))
    return type(series.array)(pa.chunked_array([arr]), dtype=series.dtype)


def _side_columns(series, positions, default_name, drop_index, prefix, mirror, values=None):
    """[(column label, values)] of one side of get_matches when it reduces to plain columns (index dropped, or an
    unnamed single-level index), else None.  Same labels / order as _take_side."""
    name = series.name if series.name else default_name
    index = series.index
    if not (drop_index or (index.nlevels == 1 and index.name is None and name != 'index')):
        return None
    taken = series.array.take(positions) if values is None else values
    # keep the Series' own dtype (an object column must stay object: the DataFrame constructor would otherwise infer
    # `str` from it — a different dtype than the reference's `iloc`, and a full conversion pass over the result)
    out = [(f"{prefix}{name}", pd.Series(taken, dtype=series.dtype, copy=False))]
    if drop_index:
        return out
    if isinstance(index, pd.RangeIndex):
        pos64 = np.asarray(positions, dtype=np.int64)
        labels = pos64 if (index.start == 0 and index.step == 1) else index.start + index.step * pos64
    else:
        labels = index.to_numpy()[positions]
    level = (f"{prefix}index", labels)
    return out + [level] if mirror else [level] + out


def _take_side(series, positions, default_name, drop_index, prefix, mirror, values=None):
    """Rows of `series` at `positions` as prefixed column(s); index levels become columns unless dropped.
    `mirror` puts the value column first (right-hand side of get_matches, ref:468).  `values` are the already
    gathered rows (device string gather) when available."""
    name = series.name if series.name else default_name
    index = series.index
    if drop_index or (index.nlevels == 1 and index.name is None and name != 'index'):
        # fast path (millions of matches): one take on the backing array, one on the index values
        taken = series.array.take(positions) if values is None else values
        values = pd.Series(taken, name=f"{prefix}{name}", copy=False)
        if drop_index:
            return values
        if isinstance(index, pd.RangeIndex):
            labels = index.start + index.step * np.asarray(positions, dtype=np.int64)
        else:
            labels = index.to_numpy()[positions]
        level = pd.Series(labels, name=f"{prefix}index", copy=False)
        return pd.concat([values, level] if mirror else [level, values], axis=1)
    named = series if series.name else series.rename(default_name)
    taken = named.iloc[positions].reset_index(drop=False)
    if mirror:
        taken = taken[taken.columns[::-1]]
    return taken.rename(columns={c: f"{prefix}{c}" for c in taken.columns})

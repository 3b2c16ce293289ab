"""match_records / group_similar_records: weighted similarity over several string columns of a DataFrame, in one
product.

Every field (a column named in `weights`) is vectorised on its own, with the options of the call: its vocabulary and
idf are fitted on master ++ duplicates of that column, so a field's matrix is exactly what match_strings builds for
that column alone.  Field k's rows are scaled by sqrt(w_k / sum w) and the fields are stacked side by side into one
CSR (csrc/sg_fields.cu); the cosine of two stacked rows is then sum_k (w_k / sum w) cos_k, the weighted mean of the
per-field similarities.  A stacked row is non-negative with norm <= 1 like a K1 row, so the whole top-n product (the
triangle, identical-row dedup, the top-n floor, blocking keys, K4) runs on it unchanged, exact as ever.  The score of
every reported pair in every field is then the exact per-field cosine (sg_rescore over the final match list).

A missing value (None, NaN, pd.NA) in a field reads as the empty string and contributes nothing to that field.
"""
import numbers
from typing import Dict, Optional

import numpy as np
import pandas as pd

from . import _device, _dist, _ingest, _lib
from .string_grouper import (DEFAULT_ID_NAME, GROUP_REP_PREFIX, LEFT_PREFIX, RIGHT_PREFIX,
                             StringGrouper, _side_columns, validate_is_fit)

SIMILARITY_PREFIX = 'similarity_'


def match_records(master: pd.DataFrame, duplicates: Optional[pd.DataFrame] = None, *, weights: Dict[str, float],
                  master_id: Optional[pd.Series] = None, duplicates_id: Optional[pd.Series] = None,
                  master_keys: Optional[pd.Series] = None, duplicates_keys: Optional[pd.Series] = None,
                  **kwargs) -> pd.DataFrame:
    """All pairs of records whose weighted similarity sum_k (w_k / sum w) cos_k exceeds min_similarity, top
    max_n_matches per left record, like match_strings.

    `weights` maps column names to weights > 0; its key order is the field order.  Other columns are ignored.
    `kwargs` are the StringGrouperConfig options; the vectoriser options apply to every field.  Ids and blocking keys
    behave as in match_strings.  The frame has the layout of match_strings with one column per field on each side:
    left_index, left_<f1> .. left_<fk>, [left_id], similarity, similarity_<f1> .. similarity_<fk>, [right_id],
    right_<f1> .. right_<fk>, right_index.  `similarity` is the combined score, `similarity_<f>` the exact cosine of
    the pair in field f (on a self-match's diagonal `similarity` is 1 and `similarity_<f>` the field's self-score).
    """
    return _RecordsGrouper(master, duplicates, weights, master_id, duplicates_id, master_keys, duplicates_keys,
                           **kwargs).fit().get_matches()


def group_similar_records(records: pd.DataFrame, *, weights: Dict[str, float], string_ids: Optional[pd.Series] = None,
                          keys: Optional[pd.Series] = None, **kwargs) -> pd.DataFrame:
    """Group representative of every record over the weighted similarity (see match_records), like
    group_similar_strings: [group_rep_id], group_rep_index, group_rep_<f1> .. group_rep_<fk>, indexed like
    `records`."""
    return _RecordsGrouper(records, None, weights, string_ids, None, keys, None, **kwargs).fit().get_groups()


def _fields_of(weights, frames):
    """(field names, float64 weights) after the argument checks."""
    if not isinstance(weights, dict) or not weights:
        raise ValueError('weights must be a non-empty dict {column name: weight}')
    if len(weights) > _lib.SG_FIELDS_MAX:
        raise ValueError('%d fields; at most %d are supported' % (len(weights), _lib.SG_FIELDS_MAX))
    for f, w in weights.items():
        if isinstance(w, bool) or not isinstance(w, numbers.Real) or not (np.isfinite(w) and w > 0):
            raise ValueError('the weight of field %r must be a finite number > 0, got %r' % (f, w))
        for name, frame in frames:
            if f not in frame.columns:
                raise ValueError('weights name the column %r, which %s does not have' % (f, name))
            if not isinstance(frame[f], pd.Series):
                raise ValueError('%s has more than one column named %r' % (name, f))
    return list(weights), np.array([float(w) for w in weights.values()], dtype=np.float64)


def _field_column(frame, field, side):
    """The column as a Series of strings, missing values read as ''; anything else raises the reference's TypeError."""
    col = frame[field]
    missing = col.isna()
    if missing.any():
        col = col.fillna('') if isinstance(col.dtype, pd.StringDtype) else col.astype(object).where(~missing, '')
    if not _ingest.is_series_of_strings(col):
        raise TypeError('%s input does not consist of pandas.Series containing only Strings' % side)
    return col


def _index_columns(index, positions, prefix):
    """[(label, values)] of the index levels at `positions`, named as reset_index() names them."""
    names = pd.DataFrame(index=index[:0]).reset_index().columns
    taken = index.take(positions)
    if index.nlevels == 1:
        return [(f'{prefix}{names[0]}', pd.Series(taken, copy=False))]
    return [(f'{prefix}{n}', pd.Series(taken.get_level_values(i), copy=False)) for i, n in enumerate(names)]


def _unique(labels):
    seen = set()
    dup = [x for x in labels if x in seen or seen.add(x)]
    if dup:
        raise ValueError('the result would hold several columns named %s; rename the fields or ids' % dup)


class _RecordsGrouper(StringGrouper):
    """StringGrouper over the stacked fields of DataFrames: _get_tf_idf_matrices builds the stacked matrices,
    fit() and the product are StringGrouper's own; the result frames gain one column per field."""

    def __init__(self, master, duplicates, weights, master_id=None, duplicates_id=None, master_keys=None,
                 duplicates_keys=None, **kwargs):
        if not isinstance(master, pd.DataFrame):
            raise TypeError('master must be a pandas.DataFrame')
        if duplicates is not None and not isinstance(duplicates, pd.DataFrame):
            raise TypeError('duplicates must be a pandas.DataFrame')
        frames = [('master', master)] + ([] if duplicates is None else [('duplicates', duplicates)])
        self._fields, self._weights = _fields_of(weights, frames)
        self._frames = (master, duplicates)
        self._columns = [(_field_column(master, f, 'Master'),
                          None if duplicates is None else _field_column(duplicates, f, 'Duplicates'))
                         for f in self._fields]
        self._field_matrices = []
        self._field_scores = []
        # the first field stands for the strings in StringGrouper's checks (lengths, ids, keys)
        super().__init__(self._columns[0][0], self._columns[0][1], master_id, duplicates_id,
                         master_keys=master_keys, duplicates_keys=duplicates_keys, **kwargs)

    def _get_tf_idf_matrices(self, shard=True):
        cfg = self._config
        n_master = len(self._master)
        stats = {"fields": len(self._fields)}
        marks = {"time_kernels": True}      # the records phases are always timed (CUDA events)
        _device.mark(marks, "start")
        masters, dups = [], []
        for f, (m, d) in zip(self._fields, self._columns):
            data, offsets, flags, _ = _ingest.pack_strings([m] if d is None else [m, d], cfg.regex, cfg.ignore_case,
                                                          cfg.normalize_to_ascii)
            fm, fd, _ = _device.tfidf(data, offsets, n_master, cfg.ngram_size, flags, cfg.tfidf_matrix_dtype)
            if fm.shape[1] == 0:
                raise ValueError('field %r: empty vocabulary; perhaps the documents only contain stop words' % (f,))
            masters.append(fm)
            dups.append(fm if fd is None else fd)
            _device.mark(marks, ("k1", f))
        scales = _device.field_scales(self._weights, cfg.tfidf_matrix_dtype)
        master = _device.stack_fields(masters, scales)
        dup = master if self._duplicates is None else _device.stack_fields(dups, scales)
        _device.mark(marks, "stack")
        if marks.get("marks"):
            marks["marks"][-1][1].synchronize()
            ms = _device.phases_ms(marks)
            stats["k1_ms"] = {f: ms[("k1", f)] for f in self._fields}
            stats["stack_ms"] = ms["stack"]
        stats.update(n_docs=n_master + (0 if self._duplicates is None else len(self._duplicates)), nnz=master.nnz +
                     (0 if dup is master else dup.nnz), vocab=master.shape[1], field_vocab=[m.shape[1] for m in masters])
        self._field_matrices = list(zip(masters, dups))
        self._vocabulary = None
        self._last_stats = stats
        self._raw_device = None
        return master, dup

    def _build_matches(self, master_matrix, duplicate_matrix, n_blocks=None):
        # a records call computes the whole product on every rank, as keyed calls do
        with _dist.local():
            return super()._build_matches(master_matrix, duplicate_matrix, n_blocks)

    def _get_matches_list(self, matches):
        out = super()._get_matches_list(matches)
        self._field_scores = [_device.pair_scores(A, B, matches) for A, B in self._field_matrices]
        return out

    @validate_is_fit
    def get_matches(self, ignore_index: Optional[bool] = None, include_zeroes: Optional[bool] = None) -> pd.DataFrame:
        if ignore_index is None:
            ignore_index = self._config.ignore_index
        if include_zeroes is None:
            include_zeroes = self._config.include_zeroes
        pairs, scores = self._matches_list, self._field_scores
        if not (self._config.min_similarity > 0 or not include_zeroes):
            zeros = self._get_non_matches_list()
            if not zeros.empty:
                pairs = pd.concat([pairs, zeros], axis=0, ignore_index=True)
                scores = [np.concatenate([s, np.zeros(len(zeros))]) for s in scores]
        lpos = pairs.master_side.to_numpy()
        rpos = pairs.dupe_side.to_numpy()
        master, dup = self._frames
        right = master if dup is None else dup

        def values(frame, pos, prefix):
            return [(f'{prefix}{f}', pd.Series(frame[f].array.take(pos), copy=False)) for f in self._fields]

        left = values(master, lpos, LEFT_PREFIX)
        if not ignore_index:
            left = _index_columns(master.index, lpos, LEFT_PREFIX) + left
        rcols = values(right, rpos, RIGHT_PREFIX)
        if not ignore_index:
            rcols += _index_columns(right.index, rpos, RIGHT_PREFIX)[::-1]
        if self._master_id is not None:
            right_ids = self._master_id if self._duplicates is None else self._duplicates_id
            left += _side_columns(self._master_id, lpos, DEFAULT_ID_NAME, True, LEFT_PREFIX, False)
            rcols = _side_columns(right_ids, rpos, DEFAULT_ID_NAME, True, RIGHT_PREFIX, True) + rcols
        sims = [('similarity', pairs.similarity.to_numpy())]
        sims += [(f'{SIMILARITY_PREFIX}{f}', s) for f, s in zip(self._fields, scores)]
        flat = left + sims + rcols
        _unique([k for k, _ in flat])
        return pd.DataFrame(dict(flat), copy=False)

    def _deduplicate(self, ignore_index=False) -> pd.DataFrame:
        rep = self._representatives(len(self._master))
        records = self._frames[0]
        output = records[self._fields].iloc[rep].reset_index(drop=ignore_index)
        output.columns = [f'{GROUP_REP_PREFIX}{c}' for c in output.columns]
        if self._master_id is not None:
            name = self._master_id.name if self._master_id.name else DEFAULT_ID_NAME
            ids = self._master_id.iloc[rep].rename(f'{GROUP_REP_PREFIX}{name}').reset_index(drop=True)
            output = pd.concat([ids, output], axis=1)
        _unique(list(output.columns))
        output.index = records.index
        return output

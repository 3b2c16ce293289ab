"""TEST INFRASTRUCTURE — NOT PRODUCT CODE.

CPU restatement of the reference hot path, function by function, on top of the
real scikit-learn / scipy (both are the reference's own dependencies and are
installed on every box of this image) and the C oracle for `sparse_dot_topn`.

Citations are string_grouper/string_grouper.py:<line>.
"""
import re
from unicodedata import normalize

import numpy as np
import pandas as pd
from scipy.sparse import csr_matrix, vstack
from sklearn.feature_extraction.text import TfidfVectorizer

from .sdt import sp_matmul_topn, zip_sp_matmul_topn

DEFAULT_REGEX = r'[,-./]|\s'   # :19


def n_grams(string, ngram_size=3, regex=DEFAULT_REGEX, ignore_case=True, normalize_to_ascii=True):
    """Analyzer, :365-378 — lower, NFKD→ASCII, regex strip, sliding windows."""
    if ignore_case and string is not None:
        string = string.lower()
    if normalize_to_ascii:
        string = normalize('NFKD', string).encode('ASCII', 'ignore').decode()
    string = re.sub(regex, r'', string)
    return [string[i:i + ngram_size] for i in range(len(string) - ngram_size + 1)]


def tf_idf_matrices(master, duplicates=None, ngram_size=3, regex=DEFAULT_REGEX, ignore_case=True,
                    normalize_to_ascii=True, dtype=np.float64):
    """:305-308 + :685-707 — vectoriser fitted on master ⧺ duplicates, then transform."""
    def analyzer(s):
        return n_grams(s, ngram_size, regex, ignore_case, normalize_to_ascii)
    vec = TfidfVectorizer(min_df=1, analyzer=analyzer, dtype=dtype)
    strings = list(master) + (list(duplicates) if duplicates is not None else [])
    vec.fit(strings)
    m = vec.transform(list(master))
    d = vec.transform(list(duplicates)) if duplicates is not None else m
    return m, d, vec


def define_chunks(length, n_chunks):
    """:714-722 — ceil(length / n_chunks)-sized consecutive ranges."""
    chunk = int(np.ceil(length / n_chunks))
    return [range(i, min(i + chunk, length)) for i in range(0, length, chunk)]


def build_matches(master_matrix, duplicate_matrix, n_blocks, max_n_matches=20, min_similarity=0.8,
                  n_threads=1):
    """:709-752 — block loop, per-pair top-n product, zip over right blocks, vstack."""
    if n_blocks is None:
        return sp_matmul_topn(master_matrix, duplicate_matrix.transpose(), top_n=max_n_matches,
                              threshold=min_similarity, sort=True, n_threads=n_threads)
    As = [master_matrix[list(r)] for r in define_chunks(master_matrix.shape[0], n_blocks[0])]
    Bs = [duplicate_matrix[list(r)] for r in define_chunks(duplicate_matrix.shape[0], n_blocks[1])]
    Cs = [[sp_matmul_topn(Aj, Bi.T, top_n=max_n_matches, threshold=min_similarity, sort=True,
                          n_threads=n_threads) for Bi in Bs] for Aj in As]
    Czip = [zip_sp_matmul_topn(top_n=max_n_matches, C_mats=Cis) for Cis in Cs]
    return vstack(Czip, dtype=np.float64).tocsr()


def guess_blocks(n_left, n_right):
    """:387-389."""
    return (max(1, round(n_left / 1e6)), max(1, round(n_right / 4e3)))


def fix_diagonal_and_symmetrize(matches):
    """:419-427, :955-964 — LIL, diagonal := 1, pattern := pattern ∪ patternᵀ."""
    m = matches.tolil()
    r = np.arange(m.shape[0])
    m[r, r] = 1
    r, c = m.nonzero()
    m[c, r] = m[r, c]
    return m.tocsr()


def matches_list(matches):
    """:755-763."""
    r, c = matches.nonzero()
    return pd.DataFrame({'master_side': r.astype(np.int64), 'dupe_side': c.astype(np.int64),
                         'similarity': matches.data})


def get_matches_frame(master, ml, duplicates=None, ignore_index=False):
    """:443-518 for the id-less case — strings (and index columns) gathered by position, prefixed, concatenated."""
    left = master if master.name else master.rename('side')
    left = left.iloc[ml.master_side].reset_index(drop=ignore_index)
    right = master if duplicates is None else duplicates
    right = right if right.name else right.rename('side')
    right = right.iloc[ml.dupe_side].reset_index(drop=ignore_index)
    right = right if isinstance(right, pd.Series) else right[right.columns[::-1]]

    def prefixed(data, prefix):
        if isinstance(data, pd.DataFrame):
            return data.rename(columns={c: f"{prefix}{c}" for c in data.columns})
        return data.rename(f"{prefix}{data.name}")

    return pd.concat([prefixed(left, 'left_'), ml.similarity.reset_index(drop=True), prefixed(right, 'right_')], axis=1)


def deduplicate(ml, n, group_rep='centroid'):
    """:851-904 — index of every string's group representative: weakly connected components of the match
    graph (:863), weight = row index ('first') or row sum of similarities ('centroid', :875-881), representative =
    groupby(...).transform('first' | 'idxmax') (:885-886)."""
    from scipy.sparse.csgraph import connected_components
    graph = csr_matrix((np.full(len(ml), 1), (ml.master_side.to_numpy(), ml.dupe_side.to_numpy())), shape=(n, n))
    _, groups = connected_components(csgraph=graph, directed=True)
    g = pd.Series(groups, name='raw_group_id').reset_index()
    g.rename(columns={'index': 'weight'}, inplace=True)
    method = 'first'
    if group_rep == 'centroid':
        graph.data = ml['similarity'].to_numpy()
        g['weight'] = pd.Series(np.asarray(graph.sum(axis=1)).squeeze(axis=1))
        method = 'idxmax'
    return g.groupby('raw_group_id', sort=False)['weight'].transform(method).to_numpy().astype(np.int64)


def fit(master, duplicates=None, *, ngram_size=3, regex=DEFAULT_REGEX, ignore_case=True,
        normalize_to_ascii=True, tfidf_matrix_dtype=np.float64, max_n_matches=20,
        min_similarity=0.8, n_blocks=None, force_symmetries=True, n_threads=1,
        fast_symmetrize=False):
    """:380-431 — returns (matches_list DataFrame, true_max_n_matches)."""
    m, d, _ = tf_idf_matrices(master, duplicates, ngram_size, regex, ignore_case, normalize_to_ascii,
                              tfidf_matrix_dtype)
    if n_blocks is None:
        n_blocks = guess_blocks(m.shape[0], d.shape[0])
    C = build_matches(m, d, n_blocks, max_n_matches, min_similarity, n_threads)
    true_max = int(np.diff(C.indptr).max()) if C.shape[0] else 0
    if force_symmetries and duplicates is None:
        C = symmetrize_fast(C) if fast_symmetrize else fix_diagonal_and_symmetrize(C)
    return matches_list(C), true_max


def symmetrize_fast(matches):
    """Vectorised equivalent of fix_diagonal_and_symmetrize for big oracle runs
    (same pattern, diagonal exactly 1, columns ascending).  Checked against the
    LIL restatement in tests/test_oracle.py."""
    C = matches.tocoo()
    n = C.shape[0]
    r = np.concatenate([C.row, C.col, np.arange(n)]).astype(np.int64)
    c = np.concatenate([C.col, C.row, np.arange(n)]).astype(np.int64)
    v = np.concatenate([C.data, C.data, np.ones(n)])
    # later entries win on duplicates: order so that transposed < original < diagonal
    pri = np.concatenate([np.ones(len(C.data)), np.zeros(len(C.data)), np.full(n, 2.0)])
    order = np.lexsort((pri, c, r))
    r, c, v = r[order], c[order], v[order]
    last = np.ones(len(r), dtype=bool)
    last[:-1] = (r[1:] != r[:-1]) | (c[1:] != c[:-1])
    # where both (r,c) and (c,r) were stored the reference swaps the two values (:963)
    return csr_matrix((v[last], (r[last], c[last])), shape=C.shape)


def hot_path_macs(A, B):
    """MACs = Σ_f dfA(f)·dfB(f) of the Gustavson product A·Bᵀ (SURVEY.md §8d)."""
    dfa = np.bincount(A.indices, minlength=A.shape[1]).astype(np.int64)
    dfb = np.bincount(B.indices, minlength=B.shape[1]).astype(np.int64)
    return int((dfa * dfb).sum())

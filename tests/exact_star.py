"""Star groups as a specification: what group_similar_strings(linkage='star') must return, stated serially in plain
Python (the rounds of csrc/sg_star.cu and of string_grouper.star_representatives must give exactly this).

1. Graph: u ~ v (u != v) whenever the pair (u, v) or (v, u) is listed.
2. Rank: by index ('first'), or by the row sum of the similarities descending, then index ('centroid').
3. In rank order, a string not yet assigned becomes a pivot and every unassigned neighbour is assigned to it.

Returns rep (int64 [n]): the pivot of every string's group.
"""
import numpy as np
from scipy.sparse import csr_matrix


def row_weights(n, rows, cols, scores):
    """the 'centroid' weight: scipy's CSR row sum over the listed pairs in storage order (reference :875-881)"""
    graph = csr_matrix((np.full(len(rows), 1), (rows, cols)), shape=(n, n))
    graph.data = np.asarray(scores, dtype=np.float64)
    return np.asarray(graph.sum(axis=1)).squeeze(axis=1)


def serial_star(n, rows, cols, weight=None):
    neighbours = [set() for _ in range(n)]
    for u, v in zip(np.asarray(rows).tolist(), np.asarray(cols).tolist()):
        if u != v:
            neighbours[u].add(v)
            neighbours[v].add(u)
    order = range(n) if weight is None else sorted(range(n), key=lambda i: (-float(weight[i]), i))
    rep = [-1] * n
    for p in order:
        if rep[p] >= 0:
            continue
        rep[p] = p
        for q in neighbours[p]:
            if rep[q] < 0:
                rep[q] = p
    return np.asarray(rep, dtype=np.int64)


def star_of_pairs(n, rows, cols, scores, centroid):
    return serial_star(n, rows, cols, row_weights(n, rows, cols, scores) if centroid else None)


def star_of_grouper(sg):
    """the specification on a fitted StringGrouper's current match list and group_rep"""
    pairs = sg._matches_list
    return star_of_pairs(len(sg._master), pairs.master_side.to_numpy(), pairs.dupe_side.to_numpy(),
                         pairs.similarity.to_numpy(), sg._config.group_rep == "centroid")

"""numpy restatement of path 7 (`b200_rank_topk_list`) and of `PopularModel._recommend_u2i`
(rectools/models/popular.py:229-277), vectorised over rows.

Row r keeps the positions p < min(n_list, k + m_r) (m_r = its viewed count, repeats included) whose list id it has not
viewed, ascending, and of them the first min(k, their count): the reference's window `popularity_list[:k + |viewed|]`
minus the viewed ids, cut to k."""
import numpy as np


def rank_list_np(list_ids, indptr, indices, n_rows, k):
    """`(positions int32 [n_rows, k_out], counts int32 [n_rows])` as the export writes them (k_out = min(k, n_list),
    unfilled slots -1).  `indptr` None: nothing viewed."""
    list_ids = np.asarray(list_ids, dtype=np.int64)
    n_list = len(list_ids)
    k_out = min(k, n_list)
    positions = np.full((n_rows, k_out), -1, dtype=np.int32)
    counts = np.zeros(n_rows, dtype=np.int32)
    if n_rows == 0 or k_out == 0:
        return positions, counts
    if indptr is None:
        indptr, indices = np.zeros(n_rows + 1, np.int64), np.zeros(0, np.int64)
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    m = np.diff(indptr)
    limit = np.minimum(n_list, k + m)
    # every (row, position) pair of the windows
    row = np.repeat(np.arange(n_rows, dtype=np.int64), limit)
    starts = np.cumsum(limit) - limit
    pos = np.arange(len(row), dtype=np.int64) - np.repeat(starts, limit)
    # membership of (row, list id) among the (row, viewed id) pairs, which are sorted: rows in order, ids ascending
    shift = np.int64(1) << np.int64(33)
    viewed_key = np.repeat(np.arange(n_rows, dtype=np.int64), m) * shift + (indices[indptr[0] : indptr[-1]] + (np.int64(1) << 32))
    probe = row * shift + (list_ids[pos] + (np.int64(1) << 32))
    keep = np.ones(len(probe), dtype=bool)
    if len(viewed_key):
        at = np.minimum(np.searchsorted(viewed_key, probe), len(viewed_key) - 1)
        keep = viewed_key[at] != probe
    # rank of a kept pair inside its row
    csum = np.cumsum(keep, dtype=np.int64)
    before_row = np.repeat(np.concatenate(([0], csum))[starts], limit)
    rank = csum - before_row - 1
    take = keep & (rank < k)
    positions[row[take], rank[take]] = pos[take]
    counts[:] = np.bincount(row[take], minlength=n_rows)
    return positions, counts


def recommend_u2i_np(list_items, list_scores, user_ids, viewed_csr, k, filter_viewed):
    """The reference's `_recommend_u2i` triplet as arrays, from the (filtered) popularity list and the viewed CSR."""
    user_ids = np.asarray(user_ids)
    if not filter_viewed:
        k_out = min(k, len(list_items))
        return np.repeat(user_ids, k_out), np.tile(list_items[:k_out], len(user_ids)), np.tile(list_scores[:k_out], len(user_ids))
    rows = viewed_csr[user_ids]
    positions, counts = rank_list_np(list_items, rows.indptr, rows.indices, len(user_ids), k)
    flat = positions[np.arange(positions.shape[1])[None, :] < counts[:, None]]
    return np.repeat(user_ids, counts), np.asarray(list_items)[flat], np.asarray(list_scores)[flat]

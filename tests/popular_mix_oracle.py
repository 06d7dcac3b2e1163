"""numpy restatement of path 8 (`b200_rank_topk_list_mix`) and of `PopularInCategoryModel._recommend_u2i`
(rectools/models/popular_in_category.py:264-373), vectorised over rows.

For row r, list c (its priority) contributes what path 7 keeps of it (tests/popular_oracle.py: `rank_list_np`), entry j
of rank j; an entry is main when j < quota[c], fallback otherwise.
  1. main entries in (c, j) order, then fallback entries in (c, j) order: the first entry of each id survives
     (the reference's `drop_duplicates`, keep first);
  2. survivors ordered by (main first, j, c), the first k kept (every main survivor is: sum(quota) <= k);
  3. group: kept entries by (c, j); rotate: by (r', c), r' = the entry's index among the kept entries of its list.
"""
import numpy as np

from tests.popular_oracle import rank_list_np


def rank_list_mix_np(lists, quota, mixing, indptr, indices, n_rows, k):
    """`(positions int32 [n_rows, k_out], counts int32 [n_rows])` as the export writes them: positions into the
    concatenation of `lists`, k_out = min(k, total length), unfilled slots -1.  `mixing`: "rotate" or "group".
    `indptr` None: nothing viewed."""
    lists = [np.asarray(x, dtype=np.int64) for x in lists]
    offsets = np.concatenate(([0], np.cumsum([len(x) for x in lists]))).astype(np.int64)
    all_ids = np.concatenate(lists) if lists else np.zeros(0, np.int64)
    k_out = min(k, len(all_ids))
    positions = np.full((n_rows, k_out), -1, dtype=np.int32)
    counts = np.zeros(n_rows, dtype=np.int32)
    if n_rows == 0 or k_out == 0:
        return positions, counts
    # every entry (row, list, rank, position) of every row
    row, cat, rank, pos = [], [], [], []
    for c, lst in enumerate(lists):
        p, n = rank_list_np(lst, indptr, indices, n_rows, k)
        take = np.arange(p.shape[1])[None, :] < n[:, None]
        rr, jj = np.nonzero(take)
        row.append(rr)
        cat.append(np.full(len(rr), c))
        rank.append(jj)
        pos.append(p[rr, jj].astype(np.int64) + offsets[c])
    row, cat, rank, pos = (np.concatenate(x).astype(np.int64) for x in (row, cat, rank, pos))
    fallback = (rank >= np.asarray(quota, dtype=np.int64)[cat]).astype(np.int64)
    ids = all_ids[pos]
    # 1. the first of each (row, id) in the sequence (row, fallback, c, j)
    o = np.lexsort((rank, cat, fallback, ids, row))
    first = np.ones(len(o), dtype=bool)
    first[1:] = (row[o][1:] != row[o][:-1]) | (ids[o][1:] != ids[o][:-1])
    s = o[first]
    # 2. (row, fallback, j, c): the first k of each row
    s = s[np.lexsort((cat[s], rank[s], fallback[s], row[s]))]
    s = s[_index_in_group(row[s]) < k]
    # 3. the final order
    s = s[np.lexsort((rank[s], cat[s], row[s]))]
    if mixing == "rotate":
        r2 = _index_in_group(row[s] * (len(lists) + 1) + cat[s])
        s = s[np.lexsort((cat[s], r2, row[s]))]
    slot = _index_in_group(row[s])
    positions[row[s], slot] = pos[s]
    counts[:] = np.bincount(row[s], minlength=n_rows)
    return positions, counts


def _index_in_group(keys):
    """Index of each element among the equal keys before it (keys grouped, i.e. equal keys adjacent)."""
    n = len(keys)
    if n == 0:
        return np.zeros(0, np.int64)
    starts = np.ones(n, dtype=bool)
    starts[1:] = keys[1:] != keys[:-1]
    start_idx = np.maximum.accumulate(np.where(starts, np.arange(n), 0))
    return np.arange(n) - start_idx


def recommend_in_category_u2i_np(model, user_ids, viewed_csr, k, filter_viewed, sorted_item_ids_to_recommend):
    """The reference's `_recommend_u2i` triplet as arrays, from the model's quotas and category lists and the viewed CSR:
    rows grouped by ascending user id."""
    num_recs = model._get_num_recs_for_each_category(k)  # pylint: disable=protected-access
    lists = [model.models[c]._get_filtered_popularity_list(sorted_item_ids_to_recommend) for c in num_recs.index]  # pylint: disable=protected-access
    items = [np.asarray(x) for x, _ in lists]
    all_items = np.concatenate(items)
    all_scores = np.concatenate([np.asarray(s) for _, s in lists])
    users = np.sort(np.asarray(user_ids))
    mixing = model.mixing_strategy.value
    if filter_viewed:
        rows = viewed_csr[users]
        positions, counts = rank_list_mix_np(items, num_recs.values, mixing, rows.indptr, rows.indices, len(users), k)
    else:
        positions, counts = rank_list_mix_np(items, num_recs.values, mixing, None, None, len(users), k)
    flat = positions[np.arange(positions.shape[1])[None, :] < counts[:, None]]
    return np.repeat(users, counts), all_items[flat], all_scores[flat]

"""Popularity lists on the GPU (engine path 7, `b200_rank_topk_list`): `PopularModel._recommend_u2i` without its per-user
Python loop.

`PopularModel._recommend_u2i` (rectools/models/popular.py:229-277) rebuilds the viewed-items CSR from the whole
interactions table on every call, then, for each user, takes the first `k + |viewed|` entries of the (whitelist-filtered)
popularity list, drops the viewed ones and keeps the first k.  `popular_recommend_u2i` returns the same triplet:

  * the list comes from the model's own `_get_filtered_popularity_list`;
  * the viewed rows come from the cached `recommend.viewed_csr(dataset)`, so repeated calls -- and the per-category calls
    of `PopularInCategoryModel`, which all receive the same dataset -- share one CSR;
  * one kernel pass returns the kept list positions of every user, and the ids and scores are gathered from the list in
    their own dtypes;
  * `filter_viewed=False` tiles the list's first k entries on the host, as the reference does, with no GPU call.

An empty result is returned as three empty lists, as the reference returns it (`PopularInCategoryModel` builds DataFrames
from the triplet, and empty lists give object columns where empty arrays would not).  A list holding ids that int32
cannot represent goes to the original method.  The triplet's arrays hold what the reference's lists hold: user ids in the
dtype of `user_ids`, item ids and scores in the dtypes of the popularity list.
"""
from __future__ import annotations

import ctypes as C
import typing as tp

import numpy as np

from . import _lib

_INT32_MAX = np.iinfo(np.int32).max
_K_MAX = 2**31 - 1


def _int32_ids(list_ids) -> np.ndarray:
    """`list_ids` as a contiguous int32 array, refused unless they are integers in [0, 2^31 - 1]."""
    ids = np.asarray(list_ids).reshape(-1)
    if ids.size and not np.issubdtype(ids.dtype, np.integer):
        raise TypeError(f"list_ids must be integers, got {ids.dtype}")
    if ids.size and (int(ids.min()) < 0 or int(ids.max()) > _INT32_MAX):
        raise ValueError("list_ids must lie in [0, 2^31 - 1]")
    return np.ascontiguousarray(ids, dtype=np.int32)


def _viewed_arrays(viewed_rows, n_rows: tp.Optional[int]) -> tp.Tuple[tp.Optional[np.ndarray], tp.Optional[np.ndarray], int]:
    """`(indptr int64, indices int32, n_rows)` of the viewed rows `rank_list` and `rank_list_mix` take (None, None: nothing
    viewed), rebased to start at 0."""
    if viewed_rows is None:
        if n_rows is None or n_rows < 0:
            raise ValueError("without viewed_rows, n_rows must be given")
        indptr, indices = None, None
    else:
        if hasattr(viewed_rows, "indptr"):
            if not getattr(viewed_rows, "has_sorted_indices", True):
                viewed_rows = viewed_rows.sorted_indices()
            indptr, indices = viewed_rows.indptr, viewed_rows.indices
        else:
            indptr, indices = viewed_rows
        indptr = np.asarray(indptr, dtype=np.int64).reshape(-1)
        indices = np.asarray(indices).reshape(-1)
        if len(indptr) == 0:
            raise ValueError("viewed_rows has no row pointers")
        if n_rows is not None and n_rows != len(indptr) - 1:
            raise ValueError(f"n_rows = {n_rows} but viewed_rows has {len(indptr) - 1} rows")
        n_rows = len(indptr) - 1
        if indptr[0] != 0:  # a view into a larger CSR
            if indptr[0] < 0 or indptr[-1] > len(indices):
                raise ValueError("the row pointers of viewed_rows lie outside its indices")
            indices = indices[indptr[0] : indptr[-1]]
            indptr = indptr - indptr[0]
        if indices.dtype != np.int32:
            if indices.size and (int(indices.min()) < np.iinfo(np.int32).min or int(indices.max()) > _INT32_MAX):
                raise ValueError("viewed ids must fit int32")
        indptr = np.ascontiguousarray(indptr)
        indices = np.ascontiguousarray(indices, dtype=np.int32)
        if indptr[-1] > len(indices):
            raise ValueError("the row pointers of viewed_rows run past its indices")
    return indptr, indices, int(n_rows)


def rank_list(list_ids, viewed_rows, k: int, device: int = 0, stats: tp.Optional[tp.Dict[str, tp.Any]] = None,
              n_rows: tp.Optional[int] = None) -> tp.Tuple[np.ndarray, np.ndarray]:
    """For each row, the first k positions of the shared list `list_ids` whose id the row has not viewed:
    `(positions int32 [n_rows, k_out], counts int32 [n_rows])`, k_out = min(k, len(list_ids)), row r's positions ascending
    in `positions[r, :counts[r]]` and -1 after them.

    `list_ids`: ids >= 0 that fit int32, in list order.  `viewed_rows`: a scipy CSR matrix whose row r's column ids are
    row r's viewed ids (structure only), an `(indptr, indices)` pair with ascending ids within a row, or None (nothing
    viewed; then `n_rows` gives the row count).  A row scans the reference's window, the positions below k + its viewed
    count; with distinct list ids that is the whole list.  `stats`: a dict that receives the call's `b200_rank_stats`."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1:
        raise ValueError(f"k must be a positive int, got {k!r}")
    ids = _int32_ids(list_ids)
    indptr, indices, n_rows = _viewed_arrays(viewed_rows, n_rows)
    k = min(int(k), _K_MAX)
    k_out = min(k, len(ids))
    positions = np.empty((n_rows, k_out), dtype=np.int32)
    counts = np.empty(n_rows, dtype=np.int32)
    st = _lib.Stats()
    _lib.check(_lib.load().b200_rank_topk_list(
        int(device), len(ids), ids.ctypes.data if len(ids) else None, n_rows,
        indptr.ctypes.data if indptr is not None else None,
        indices.ctypes.data if indices is not None and len(indices) else None, k,
        positions.ctypes.data if positions.size else None, counts.ctypes.data if n_rows else None, C.byref(st),
    ))
    if stats is not None:
        stats.update(st.as_dict())
    return positions, counts


def _original_u2i():
    """`PopularModel._recommend_u2i` as RecTools defines it, also while `install(popular=True)` has rebound it."""
    from rectools.models.popular import PopularModel

    from .integration import _ORIGINALS, _POPULAR_KEY

    return _ORIGINALS.get(_POPULAR_KEY, PopularModel._recommend_u2i)  # pylint: disable=protected-access


def popular_recommend_u2i(model, user_ids, dataset, k: int, filter_viewed: bool, sorted_item_ids_to_recommend,
                          device: int = 0, stats: tp.Optional[tp.Dict[str, tp.Any]] = None):
    """`PopularModel._recommend_u2i(user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend)`
    (rectools/models/popular.py:229-255) with the per-user step on `device`; see the module docstring.  `stats` (not in the
    reference): a dict that receives the call's `b200_rank_stats` when the GPU ranks it."""
    items, scores = model._get_filtered_popularity_list(sorted_item_ids_to_recommend)  # pylint: disable=protected-access
    items, scores = np.asarray(items), np.asarray(scores)
    if items.size and (not np.issubdtype(items.dtype, np.integer) or int(items.min()) < 0 or int(items.max()) > _INT32_MAX):
        return _original_u2i()(model, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend)
    user_ids = np.asarray(user_ids)
    n = len(user_ids)
    if not filter_viewed:  # every user gets the list's first k entries (popular.py:266-270)
        k_out = min(int(k), len(items))
        if n * k_out == 0:
            return [], [], []
        return np.repeat(user_ids, k_out), np.tile(items[:k_out], n), np.tile(scores[:k_out], n)
    if n == 0 or len(items) == 0:
        return [], [], []
    from .recommend import _rows_of, viewed_csr

    csr = _rows_of(viewed_csr(dataset), user_ids.astype(np.int64, copy=False))
    positions, counts = rank_list(items.astype(np.int32, copy=False), csr, int(k), device=device, stats=stats)
    total = int(counts.sum(dtype=np.int64))
    if total == 0:
        return [], [], []
    if total == positions.size:
        flat = positions.reshape(-1)
    else:
        flat = positions[np.arange(positions.shape[1], dtype=np.int32)[None, :] < counts[:, None]]
    return np.repeat(user_ids, counts), items[flat], scores[flat]


_MIXINGS = {"rotate": _lib.MIX_ROTATE, "group": _lib.MIX_GROUP}


def rank_list_mix(lists, quota, mixing, viewed_rows, k: int, device: int = 0,
                  stats: tp.Optional[tp.Dict[str, tp.Any]] = None,
                  n_rows: tp.Optional[int] = None) -> tp.Tuple[np.ndarray, np.ndarray]:
    """For each row, the per-category lists `lists` (in priority order), each minus the row's viewed ids, mixed as
    `PopularInCategoryModel._recommend_u2i` mixes its category models' recommendations:
    `(positions int32 [n_rows, k_out], counts int32 [n_rows])`, positions into the concatenation of `lists`,
    k_out = min(k, total length), row r's in `positions[r, :counts[r]]` in their final order and -1 after them.

    Each list contributes what `rank_list` takes from it (its first k unviewed ids in the reference's window); its entries
    of rank below `quota[c]` are main, the others fallback.  The first entry of each id among the main entries, then the
    fallback entries, both in (list, rank) order, survives; every main survivor is kept, then fallback survivors in
    (rank, list) order up to k.  `mixing` "group" (or `_lib.MIX_GROUP`) orders the kept entries by (list, rank), "rotate"
    (`_lib.MIX_ROTATE`) by (index among the kept entries of their list, list).  `quota`: ints >= 0 summing to at most k.
    `viewed_rows`, `n_rows`, `stats`: as for `rank_list`."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1:
        raise ValueError(f"k must be a positive int, got {k!r}")
    mix = _MIXINGS.get(mixing, mixing) if isinstance(mixing, str) else mixing
    if isinstance(mix, bool) or not isinstance(mix, (int, np.integer)) or mix not in _MIXINGS.values():
        raise ValueError(f"mixing must be 'rotate' or 'group', got {mixing!r}")
    parts = [_int32_ids(lst) for lst in lists]
    q = np.asarray(quota).reshape(-1)
    if len(q) != len(parts):
        raise ValueError(f"{len(q)} quotas for {len(parts)} lists")
    if q.size and not np.issubdtype(q.dtype, np.integer):
        raise TypeError(f"quota must be integers, got {q.dtype}")
    if q.size and (int(q.min()) < 0 or int(q.sum(dtype=object)) > min(int(k), _K_MAX)):
        raise ValueError("quota must be >= 0 and sum to at most k (and at most 2^31 - 1)")
    q = np.ascontiguousarray(q, dtype=np.int32)
    offsets = np.zeros(len(parts) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in parts], out=offsets[1:])
    if offsets[-1] > _INT32_MAX:
        raise ValueError("the lists hold more than 2^31 - 1 ids")
    ids = np.concatenate(parts) if parts else np.zeros(0, np.int32)
    indptr, indices, n_rows = _viewed_arrays(viewed_rows, n_rows)
    k = min(int(k), _K_MAX)
    k_out = min(k, len(ids))
    positions = np.empty((n_rows, k_out), dtype=np.int32)
    counts = np.empty(n_rows, dtype=np.int32)
    st = _lib.Stats()
    _lib.check(_lib.load().b200_rank_topk_list_mix(
        int(device), len(parts), offsets.ctypes.data, ids.ctypes.data if len(ids) else None,
        q.ctypes.data if len(q) else None, int(mix), n_rows, indptr.ctypes.data if indptr is not None else None,
        indices.ctypes.data if indices is not None and len(indices) else None, k,
        positions.ctypes.data if positions.size else None, counts.ctypes.data if n_rows else None, C.byref(st),
    ))
    if stats is not None:
        stats.update(st.as_dict())
    return positions, counts


def _original_in_category_u2i():
    """`PopularInCategoryModel._recommend_u2i` as RecTools defines it, also while `install(popular_in_category=True)` has
    rebound it."""
    from rectools.models.popular_in_category import PopularInCategoryModel

    from .integration import _ORIGINALS, _POPULAR_IN_CATEGORY_KEY

    return _ORIGINALS.get(_POPULAR_IN_CATEGORY_KEY, PopularInCategoryModel._recommend_u2i)  # pylint: disable=protected-access


def popular_in_category_recommend_u2i(model, user_ids, dataset, k: int, filter_viewed: bool, sorted_item_ids_to_recommend,
                                      device: int = 0, stats: tp.Optional[tp.Dict[str, tp.Any]] = None):
    """`PopularInCategoryModel._recommend_u2i(user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend)`
    (rectools/models/popular_in_category.py:333-373) with every category's list and the mixing of each user in one
    `rank_list_mix` call on `device`, instead of one `PopularModel._recommend_u2i` call per category and the mixing in
    pandas.

      * the quotas are the model's own `_get_num_recs_for_each_category(k)`, the lists each category model's
        `_get_filtered_popularity_list`, in the quotas' (priority) order;
      * the viewed rows come from the cached `recommend.viewed_csr(dataset)`: one upload for every category;
      * `filter_viewed=False`: every user gets the same result, so one row with nothing viewed is ranked and tiled;
      * the triplet is grouped by ascending user id, as the reference sorts it, and holds the user ids in the dtype of
        `user_ids`, item ids and scores in the dtypes of the concatenated lists; with no user or no list entry it is three
        empty lists, as `popular_recommend_u2i` returns an empty result.

    Goes to the original method, unchanged: no category model (the reference's own error), repeated user ids, k < 1, list
    ids that int32 cannot represent, and quotas that are not ints >= 0 summing to at most k.  `stats` (not in the
    reference): a dict that receives the call's `b200_rank_stats` when the GPU ranks it."""
    from rectools.models.popular_in_category import MixingStrategy

    def stock():
        return _original_in_category_u2i()(model, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend)

    num_recs = model._get_num_recs_for_each_category(k)  # pylint: disable=protected-access
    quota = np.asarray(num_recs.values)
    users = np.asarray(user_ids)
    if (len(num_recs) == 0 or any(c not in model.models for c in num_recs.index) or int(k) < 1
            or not np.issubdtype(quota.dtype, np.integer) or int(quota.min()) < 0 or int(quota.sum(dtype=np.int64)) > int(k)
            or len(np.unique(users)) != len(users)):
        return stock()
    lists = [model.models[c]._get_filtered_popularity_list(sorted_item_ids_to_recommend)  # pylint: disable=protected-access
             for c in num_recs.index]
    items = [np.asarray(ids) for ids, _ in lists]
    if any(x.size and (not np.issubdtype(x.dtype, np.integer) or int(x.min()) < 0 or int(x.max()) > _INT32_MAX) for x in items):
        return stock()
    all_items = np.concatenate(items)
    all_scores = np.concatenate([np.asarray(sc) for _, sc in lists])
    mixing = "group" if model.mixing_strategy == MixingStrategy.GROUP else "rotate"
    users = users[np.argsort(users, kind="stable")]
    if len(users) == 0 or len(all_items) == 0:  # nothing to rank: the empty triplet, as `popular_recommend_u2i` returns it
        return [], [], []
    if filter_viewed:
        from .recommend import _rows_of, viewed_csr

        csr = _rows_of(viewed_csr(dataset), users.astype(np.int64, copy=False))
        positions, counts = rank_list_mix(items, quota, mixing, csr, int(k), device=device, stats=stats)
    else:
        one, n_one = rank_list_mix(items, quota, mixing, None, int(k), device=device, stats=stats, n_rows=1)
        positions = np.broadcast_to(one, (len(users), one.shape[1]))
        counts = np.broadcast_to(n_one, (len(users),))
    if int(counts.sum(dtype=np.int64)) == positions.size:
        flat = positions.reshape(-1)
    else:
        flat = positions[np.arange(positions.shape[1], dtype=np.int32)[None, :] < counts[:, None]]
    return np.repeat(users, counts), all_items[flat], all_scores[flat]

"""ItemKNN on the GPU: `ImplicitItemKNNWrapperModel` without its per-target Python loops.

u2i (engine path 9, `b200_rank_topk_knn`).  `_recommend_u2i` (rectools/models/implicit_knn.py:152-211) calls implicit's
`recommend` once per user and filters the result.  `item_knn_recommend_u2i` returns the same triplet from one call: for
user u with entries (j_e, w_e) of `get_user_item_matrix(include_weights=True)` in CSR order, item i of the touched set
(the union of the rows S[j_e] of `model.similarity`) scores (((0 + p_1) + p_2) + ...) over the entries whose S row holds
i, p = S[j_e, i] * float64(w_e), each product and each sum rounded to fp64.  The candidates are the touched items minus
the viewed ones (`filter_viewed`) within the whitelist; each user keeps min(k, their count), ordered by (score desc, id
asc) on the fp64 value.  Scores are returned as float64 (`ModelBase` casts them to float32).

i2i (engine path 6, `b200_rank_topk_pairs`).  `_recommend_i2i` (:213-255) ranks the stored entries of S[target] on the
whitelist columns.  `item_knn_recommend_i2i` gathers those rows on the host, in ascending id, and selects each target's
min(k, stored entries) by (value desc, id asc) in one call.  The reference's numpy selection leaves the order of equal
values to the implementation; outside groups of equal values the results are the same.

Served: any `ItemItemRecommender` whose class does not override implicit's `recommend` (a bare subclass is served), with a
`similarity` that is a CSR matrix of finite float values, and finite weights.  Anything else goes to the original method.
"""
from __future__ import annotations

import ctypes as C
import typing as tp

import numpy as np
from scipy import sparse

from . import _lib

_K_MAX = 2**31 - 1


def _csr_arrays(m: sparse.csr_matrix) -> tp.Tuple[np.ndarray, np.ndarray]:
    """(indptr int64 starting at 0, indices int32) of a CSR matrix."""
    indptr = np.asarray(m.indptr, dtype=np.int64)
    indices = np.asarray(m.indices)
    if indptr[0] != 0:
        indices = indices[indptr[0] : indptr[-1]]
        indptr = indptr - indptr[0]
    return np.ascontiguousarray(indptr), np.ascontiguousarray(indices, dtype=np.int32)


def rank_knn(similarity, user_rows, k: int, filter_rows=None, whitelist=None, device: int = 0,
             stats: tp.Optional[tp.Dict[str, tp.Any]] = None) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Each user row's k best items by ItemKNN score (see the module docstring): `(ids, scores, counts)`, ids int32 and
    scores float64 of shape [n_rows, k] (unfilled slots -1 and 0), counts int32 [n_rows].

    `similarity`: S, a square CSR (n_items x n_items; each item at most once per row).  `user_rows`: a CSR of the users'
    weighted entries, ranked in their stored order (weights are cast to float32, as implicit's user-items matrix holds
    them).  `filter_rows`: None or a CSR with one row per user of ids to drop.  `whitelist`: None or the ids that may be
    returned.  `stats`: a dict that receives the call's `b200_rank_stats`."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= _K_MAX:
        raise ValueError(f"k must be an int in [1, 2^31 - 1], got {k!r}")
    S = sparse.csr_matrix(similarity)
    n_items = S.shape[0]
    if S.shape[1] != n_items:
        raise ValueError(f"similarity must be square, got {S.shape}")
    U = sparse.csr_matrix(user_rows)
    n_rows = U.shape[0]
    s_indptr, s_indices = _csr_arrays(S)
    s_data = np.ascontiguousarray(S.data[S.indptr[0] : S.indptr[-1]], dtype=np.float64)
    u_indptr, u_indices = _csr_arrays(U)
    u_data = np.ascontiguousarray(U.data[U.indptr[0] : U.indptr[-1]], dtype=np.float32)
    f_indptr = f_indices = None
    if filter_rows is not None:
        F = sparse.csr_matrix(filter_rows)
        if F.shape[0] != n_rows:
            raise ValueError(f"filter_rows has {F.shape[0]} rows, user_rows {n_rows}")
        if not F.has_sorted_indices:
            F = F.sorted_indices()
        f_indptr, f_indices = _csr_arrays(F)
    wl = None
    if whitelist is not None:
        wl = np.ascontiguousarray(np.unique(np.asarray(whitelist)), dtype=np.int32)
    ids = np.empty((n_rows, k), dtype=np.int32)
    scores = np.empty((n_rows, k), dtype=np.float64)
    counts = np.empty(n_rows, dtype=np.int32)
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data  # noqa: E731
    st = _lib.Stats()
    _lib.check(_lib.load().b200_rank_topk_knn(
        int(device), n_items, s_indptr.ctypes.data, ptr(s_indices), ptr(s_data), n_rows, u_indptr.ctypes.data, ptr(u_indices),
        ptr(u_data), None if f_indptr is None else f_indptr.ctypes.data, ptr(f_indices), ptr(wl), -1 if wl is None else len(wl),
        int(k), ptr(ids), ptr(scores), ptr(counts), C.byref(st),
    ))
    if stats is not None:
        stats.update(st.as_dict())
    return ids, scores, counts


def _stock_recommend():
    from implicit.nearest_neighbours import ItemItemRecommender

    return getattr(ItemItemRecommender, "recommend", None)


def _served_similarity(self) -> tp.Optional[sparse.csr_matrix]:
    """`self.model.similarity` when the GPU gives the original method's result for it, else None."""
    model = getattr(self, "model", None)
    if model is None or getattr(type(model), "recommend", None) is not _stock_recommend():
        return None
    S = getattr(model, "similarity", None)
    if not (sparse.issparse(S) and S.format == "csr" and S.dtype in (np.float32, np.float64) and S.shape[0] == S.shape[1]):
        return None
    if not np.isfinite(S.data).all():
        return None
    if not S.has_canonical_format:  # implicit adds a repeated entry twice; the kernel takes each item once per row
        summed = S.copy()
        summed.sum_duplicates()
        if summed.nnz != S.nnz:
            return None
    return S


def _original(name: str):
    from rectools.models.implicit_knn import ImplicitItemKNNWrapperModel

    from .integration import _ORIGINALS, _ITEM_KNN_KEY

    orig = _ORIGINALS.get(_ITEM_KNN_KEY)
    return orig[name] if orig is not None else getattr(ImplicitItemKNNWrapperModel, name)


def item_knn_recommend_u2i(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend, device: int = 0,
                           stats: tp.Optional[tp.Dict[str, tp.Any]] = None):
    """`ImplicitItemKNNWrapperModel._recommend_u2i` (rectools/models/implicit_knn.py:152-211) with every user ranked in one
    call on `device`; see the module docstring.  `stats` (not in the reference): a dict that receives the call's
    `b200_rank_stats`."""
    S = _served_similarity(self)
    user_items = dataset.get_user_item_matrix(include_weights=True) if S is not None else None
    if S is None or not np.isfinite(user_items.data).all() or S.shape[0] != user_items.shape[1]:
        return _original("_recommend_u2i")(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend)
    user_ids = np.asarray(user_ids)
    rows = user_items[user_ids]
    n_cand = S.shape[0] if sorted_item_ids_to_recommend is None else len(sorted_item_ids_to_recommend)
    k_call = max(1, min(int(k), n_cand, _K_MAX))
    ids, scores, counts = rank_knn(S, rows, k_call, rows if filter_viewed else None, sorted_item_ids_to_recommend,
                                   device=device, stats=stats)
    mask = np.arange(k_call)[None, :] < counts[:, None]
    return np.repeat(user_ids, counts), ids[mask].astype(np.int64), scores[mask]


def item_knn_recommend_i2i(self, target_ids, dataset, k, sorted_item_ids_to_recommend, device: int = 0,  # pylint: disable=unused-argument
                           stats: tp.Optional[tp.Dict[str, tp.Any]] = None):
    """`ImplicitItemKNNWrapperModel._recommend_i2i` (rectools/models/implicit_knn.py:213-255) with every target selected
    in one call on `device`; see the module docstring."""
    from .rerank import rank_pairs

    S = _served_similarity(self)
    if S is None:
        return _original("_recommend_i2i")(self, target_ids, dataset, k, sorted_item_ids_to_recommend)
    target_ids = np.asarray(target_ids)
    rows = S[target_ids]
    cols_map = None
    if sorted_item_ids_to_recommend is not None:
        cols_map = np.asarray(sorted_item_ids_to_recommend)
        rows = rows[:, cols_map]  # as the reference slices S: positions into the whitelist, mapped back below
    rows = sparse.csr_matrix(rows)
    rows.sort_indices()  # ascending id within a row: path 6's position order is then id order
    codes = np.repeat(np.arange(len(target_ids), dtype=np.int64), np.diff(rows.indptr))
    positions, offsets = rank_pairs(codes, rows.data, int(k), device=device, n_groups=len(target_ids), stats=stats)
    reco = rows.indices[positions].astype(np.int64)
    if cols_map is not None:
        reco = cols_map[reco]
    return np.repeat(target_ids, np.diff(offsets)), reco, rows.data[positions]

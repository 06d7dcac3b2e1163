"""Exact stand-ins for RecTools' nmslib recommenders (rectools/tools/ann.py:32-474) on the engine.

`B200UserToItemAnnRecommender` and `B200ItemToItemAnnRecommender` take the constructor arguments and offer the methods of
`UserToItemAnnRecommender` / `ItemToItemAnnRecommender` -- `fit()`, `get_item_list_for_user[_batch]` /
`get_item_list_for_item[_batch]`, pickling -- without nmslib: a per-row allow-list is ranked by
`B200Ranker.rank_candidates` (engine path 5), a call without lists by `B200Ranker.rank_padded`.

Answers are exact: the `min(top_n, |allowed|)` allowed items of smallest distance, ties by internal id.  The reference
queries an approximate HNSW index for `top_n + index_top_k` neighbours and keeps the allowed ones among them
(`_truncate_item_list`, ann.py:146-189), so it returns the same list whenever that window holds the exact answer, and
fewer than `top_n` items (or other ones) when it does not.  The set semantics of `_truncate_item_list` are kept:
  * allowed lists are sets (a repeated id counts once);
  * u2i without lists is plain `rank`;
  * i2i without lists excludes each row's own item only;
  * i2i with lists excludes EVERY target of the batch from every row (`set(available_list).difference(set(self_indices))`
    with `self_indices` = all targets of the call), as the reference does.
The index parameters (`index_top_k`, `index_query_time_params`, `create_index_params`, `method`) are accepted and
ignored; the space of `index_init_params` picks the distance: "cosinesimil" -> COSINE, "negdotprod" -> DOT, "l2" ->
EUCLIDEAN.  A prebuilt `index` cannot be taken.  These classes are standalone (subclassing the reference would import
nmslib) and `install()` does not touch RecTools' own classes.
"""
from __future__ import annotations

import typing as tp

import numpy as np
from scipy import sparse

from .ranker import B200Ranker, Distance

_SPACES = {"cosinesimil": Distance.COSINE, "negdotprod": Distance.DOT, "l2": Distance.EUCLIDEAN}


def _id_map(id_map: tp.Any) -> tp.Any:
    """`IdMap.from_dict` for a dict (ann.py:82-85), else the IdMap given."""
    if isinstance(id_map, dict):
        from rectools.dataset import IdMap  # pylint: disable=import-outside-toplevel

        return IdMap.from_dict(id_map)
    return id_map


def _lists_csr(lists: tp.Sequence[np.ndarray], n_objects: int) -> sparse.csr_matrix:
    """Internal-id lists as the structure of a CSR matrix (duplicates and order are normalised by the ranker)."""
    lens = np.fromiter((len(x) for x in lists), dtype=np.int64, count=len(lists))
    indptr = np.zeros(len(lists) + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    indices = np.concatenate([np.asarray(x, dtype=np.int64) for x in lists]) if len(lists) else np.empty(0, np.int64)
    return sparse.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(len(lists), n_objects))


def _rows(out: tp.Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]) -> tp.List[np.ndarray]:
    _, ids, _, counts = out
    return [ids[r, : counts[r]].astype(np.int64) for r in range(len(counts))]


class _B200AnnBase:
    """Constructor, pickling and the exact query of both classes (`BaseNmslibRecommender`, ann.py:32-197).

    `device`: the CUDA device of the engine.  `ranker_factory(distance, subjects_factors, objects_factors)`: the ranker
    class (default `B200Ranker`); it must offer `rank_padded` and `rank_candidates_padded`."""

    _subjects_attr = "item_vectors"

    def __init__(
        self,
        item_vectors: np.ndarray,
        item_id_map: tp.Any,
        index_top_k: int = 0,
        index_init_params: tp.Optional[tp.Dict[str, str]] = None,
        index_query_time_params: tp.Optional[tp.Dict[str, int]] = None,
        create_index_params: tp.Optional[tp.Dict[str, int]] = None,
        index: tp.Any = None,
        *,
        device: int = 0,
        ranker_factory: tp.Optional[tp.Callable[..., tp.Any]] = None,
    ) -> None:
        if index is not None:
            raise ValueError("`index`: an exact ranker builds no nmslib index, so a prebuilt one cannot be used")
        self.item_vectors = item_vectors
        self.item_id_map = _id_map(item_id_map)
        self.index_top_k = index_top_k
        self.index_init_params = {"method": "hnsw", "space": "cosinesimil"} if index_init_params is None else index_init_params
        self.index_query_time_params = {"efSearch": 100} if index_query_time_params is None else index_query_time_params
        self.create_index_params = (
            {"M": 100, "efConstruction": 100, "post": 0} if create_index_params is None else create_index_params
        )
        space = self.index_init_params.get("space", "cosinesimil")
        if space not in _SPACES:
            raise ValueError(f"space {space!r} is not supported: use one of {sorted(_SPACES)}")
        self.distance = _SPACES[space]
        self.device = device
        self.ranker_factory = ranker_factory
        self._ranker: tp.Any = None

    def __getstate__(self) -> tp.Dict[str, tp.Any]:
        state = self.__dict__.copy()
        state["_ranker"] = None  # the engine lives on a device: rebuilt on first use
        return state

    def __setstate__(self, state: tp.Dict[str, tp.Any]) -> None:
        self.__dict__.update(state)

    def fit(self, verbose: bool = False) -> "_B200AnnBase":  # pylint: disable=unused-argument
        """Build the engine over the item vectors (the counterpart of the index build).  Returns self."""
        self._get_ranker()
        return self

    def _get_ranker(self) -> tp.Any:
        if self._ranker is None:
            subjects = getattr(self, self._subjects_attr)
            if self.ranker_factory is not None:
                self._ranker = self.ranker_factory(self.distance, subjects, self.item_vectors)
            else:
                self._ranker = B200Ranker(self.distance, subjects, self.item_vectors, device=self.device)
        return self._ranker

    def _map_to_external_id(self, item_arrays: tp.Sequence[np.ndarray]) -> tp.List[tp.Any]:
        return [self.item_id_map.convert_to_external(item_array) for item_array in item_arrays]

    def _query(
        self,
        subject_ids: np.ndarray,
        top_n: int,
        lists: tp.Optional[tp.Sequence[np.ndarray]],
        self_filter: bool,
    ) -> tp.List[tp.Any]:
        """The `min(top_n, |allowed|)` allowed items of each row, nearest first.  `self_filter` (i2i): without lists each
        row's own item is excluded, with lists every target of the batch is."""
        subject_ids = np.asarray(subject_ids, dtype=np.int64).reshape(-1)
        if top_n < 0:
            raise ValueError("`top_n` must be non-negative")
        n_items = int(np.shape(self.item_vectors)[0])
        if top_n == 0 or len(subject_ids) == 0 or n_items == 0:
            return self._map_to_external_id([np.empty(0, np.int64) for _ in subject_ids])
        ranker = self._get_ranker()
        if lists is None:
            filter_csr = None
            if self_filter:
                n = len(subject_ids)
                filter_csr = sparse.csr_matrix(
                    (np.ones(n, np.float32), subject_ids, np.arange(n + 1, dtype=np.int64)), shape=(n, n_items)
                )
            out = ranker.rank_padded(subject_ids, top_n, filter_csr)
        else:
            if self_filter:
                lists = [np.setdiff1d(np.asarray(x, dtype=np.int64), subject_ids) for x in lists]
            out = ranker.rank_candidates_padded(subject_ids, _lists_csr(lists, n_items), top_n)
        return self._map_to_external_id(_rows(out))


class B200UserToItemAnnRecommender(_B200AnnBase):
    """`UserToItemAnnRecommender` (ann.py:200-353), exact, on the engine."""

    _subjects_attr = "user_vectors"

    def __init__(
        self,
        user_vectors: np.ndarray,
        item_vectors: np.ndarray,
        user_id_map: tp.Any,
        item_id_map: tp.Any,
        index_top_k: int = 0,
        index_init_params: tp.Optional[tp.Dict[str, str]] = None,
        index_query_time_params: tp.Optional[tp.Dict[str, int]] = None,
        create_index_params: tp.Optional[tp.Dict[str, int]] = None,
        index: tp.Any = None,
        *,
        device: int = 0,
        ranker_factory: tp.Optional[tp.Callable[..., tp.Any]] = None,
    ) -> None:
        super().__init__(
            item_vectors=item_vectors,
            item_id_map=item_id_map,
            index_top_k=index_top_k,
            index_init_params=index_init_params,
            index_query_time_params=index_query_time_params,
            create_index_params=create_index_params,
            index=index,
            device=device,
            ranker_factory=ranker_factory,
        )
        self.user_vectors = user_vectors
        self.user_id_map = _id_map(user_id_map)
        if self.user_vectors.shape[1] != self.item_vectors.shape[1]:
            raise ValueError(
                f"Vectors shape mismatch: user vectors dim={self.user_vectors.shape[1]} != "
                f"item vectors dim={self.item_vectors.shape[1]}"
            )

    def get_item_list_for_user(self, user_id: tp.Any, top_n: int, item_ids: tp.Optional[tp.Sequence[tp.Any]] = None) -> tp.Any:
        """The `top_n` nearest items of one user, among `item_ids` when given (external ids)."""
        users = self.user_id_map.convert_to_internal([user_id])
        lists = None if item_ids is None else [self.item_id_map.convert_to_internal(item_ids)]
        return self._query(users, top_n, lists, self_filter=False)[0]

    def get_item_list_for_user_batch(
        self, user_ids: tp.Sequence[tp.Any], top_n: int, item_ids: tp.Optional[tp.Sequence[tp.Sequence[tp.Any]]] = None
    ) -> tp.List[tp.Any]:
        """The `top_n` nearest items of each user, among that user's list of `item_ids` when given (external ids)."""
        users = self.user_id_map.convert_to_internal(user_ids)
        lists = None if item_ids is None else [self.item_id_map.convert_to_internal(x) for x in item_ids]
        return self._query(users, top_n, lists, self_filter=False)


class B200ItemToItemAnnRecommender(_B200AnnBase):
    """`ItemToItemAnnRecommender` (ann.py:356-474), exact, on the engine."""

    def get_item_list_for_item(
        self, item_id: tp.Any, top_n: int, item_available_ids: tp.Optional[tp.Sequence[tp.Any]] = None
    ) -> tp.Any:
        """The `top_n` nearest other items of one item, among `item_available_ids` when given (external ids)."""
        items = self.item_id_map.convert_to_internal([item_id])
        lists = None if item_available_ids is None else [self.item_id_map.convert_to_internal(item_available_ids)]
        return self._query(items, top_n, lists, self_filter=True)[0]

    def get_item_list_for_item_batch(
        self, item_ids: tp.Sequence[tp.Any], top_n: int, item_available_ids: tp.Optional[tp.Sequence[tp.Sequence[tp.Any]]] = None
    ) -> tp.List[tp.Any]:
        """The `top_n` nearest items of each item, among its list of `item_available_ids` when given (external ids); with
        lists, no target of the batch is returned for any row, as in the reference."""
        items = self.item_id_map.convert_to_internal(item_ids)
        lists = None if item_available_ids is None else [self.item_id_map.convert_to_internal(x) for x in item_available_ids]
        return self._query(items, top_n, lists, self_filter=True)

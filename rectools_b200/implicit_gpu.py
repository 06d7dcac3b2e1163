"""The lowest seam (SURVEY.md section 8b): stand-ins for the four `implicit.gpu` names RecTools' GPU ranking path uses, so
that the UNMODIFIED `ImplicitRanker(..., use_gpu=True)` lands in the B200 engine.

`ImplicitRanker._rank_on_gpu` (rectools/models/rank/rank_implicit.py:148-185) does

    items  = implicit.gpu.Matrix(object_factors)            (models/utils.py:136)
    m      = implicit.gpu.Matrix(subject_factors)
    norms  = implicit.gpu.Matrix(object_norms[None, :])     (COSINE only)
    filt   = implicit.gpu.COOMatrix(filter_csr.tocoo())     (None when the filter has no non-zero)
    ids, scores = implicit.gpu.KnnQuery().topk(items=items, m=m, k=k, item_norms=norms, query_filter=filt, item_filter=None)

and afterwards strips, per row, the trailing entries whose score is at most `_get_neginf_score()` (:83-92, :107-118).
`KnnQuery.topk` below answers with padded `[n_queries, k]` arrays whose unfilled slots carry `-FLT_MAX`, which that strip
removes.  `patch_implicit_gpu()` puts the classes into an importable `implicit.gpu` module and flips the `HAS_CUDA` names
RecTools copied at import time (rank_implicit.py:24, vector.py:21); `unpatch_implicit_gpu()` undoes it.

Upstream signature reproduced from the call site above; `implicit` itself (pm-implicit 0.7.3) is not vendored.
"""
from __future__ import annotations

import typing as tp

import numpy as np
from scipy import sparse

HAS_CUDA = True


class Matrix:
    """`implicit.gpu.Matrix(ndarray)`: here just a C-contiguous fp32 host copy; the engine owns the device copies."""

    def __init__(self, arr: tp.Any) -> None:
        arr = np.asarray(arr)
        if arr.ndim == 1:
            arr = arr[None, :]
        self.arr = np.ascontiguousarray(arr, dtype=np.float32)

    @property
    def shape(self) -> tp.Tuple[int, int]:
        return self.arr.shape

    def to_numpy(self) -> np.ndarray:
        return self.arr


class COOMatrix:
    """`implicit.gpu.COOMatrix(coo)`: the query filter; kept as a CSR with sorted column ids (what the engine takes)."""

    def __init__(self, coo: tp.Any) -> None:
        csr = sparse.csr_matrix(coo)
        csr.sum_duplicates()
        if not csr.has_sorted_indices:
            csr.sort_indices()
        self.csr = csr


TopkBackend = tp.Callable[[np.ndarray, np.ndarray, int, tp.Optional[np.ndarray], tp.Optional[sparse.csr_matrix]],
                          tp.Tuple[np.ndarray, np.ndarray, np.ndarray]]
_BACKEND: tp.Optional[TopkBackend] = None  # tests inject a CPU provider; None = the B200 engine


def _engine_backend(items, queries, k, item_norms, csr):
    """`(ids [n, k_out], scores [n, k_out], counts [n])` from a B200 engine built for this call.

    The reference uploads the item matrix on every call on this path too (`implicit.gpu.Matrix(arr)`, rank_implicit.py:156);
    `Matrix` receives a fresh copy each time (models/utils.py:136), so there is no identity to key a cache on here -- the
    `Ranker`-level seam (`install()`, engine cached per factor matrix) is the fast one."""
    from .integration import B200ImplicitRanker
    from .ranker import new_engine

    eng = new_engine(items, cosine=item_norms is not None, device=B200ImplicitRanker.default_device, tc_mode=B200ImplicitRanker.default_tc_mode)
    try:
        indptr = indices = None
        if csr is not None:
            indptr, indices = csr.indptr, csr.indices
        return eng.topk(k, subjects=queries, indptr=indptr, indices=indices)
    finally:
        eng.close()


class KnnQuery:
    """`implicit.gpu.KnnQuery(max_temp_memory=...)` with the one method RecTools calls."""

    def __init__(self, max_temp_memory: int = 0) -> None:  # pylint: disable=unused-argument
        pass

    def topk(  # pylint: disable=too-many-arguments
        self,
        items: Matrix,
        m: Matrix,
        k: int,
        item_norms: tp.Optional[Matrix] = None,
        query_filter: tp.Optional[COOMatrix] = None,
        item_filter: tp.Any = None,
    ) -> tp.Tuple[np.ndarray, np.ndarray]:
        if item_filter is not None:
            raise NotImplementedError("item_filter is not used by RecTools (rank_implicit.py:181) and not supported here")
        items_arr, queries = items.arr, m.arr
        if queries.shape[1] != items_arr.shape[1]:
            raise ValueError("items and queries must have the same number of factors")
        n = queries.shape[0]
        k = int(min(k, items_arr.shape[0]))
        norms = None if item_norms is None else np.ascontiguousarray(item_norms.arr.reshape(-1), dtype=np.float32)
        csr = None
        if query_filter is not None:
            csr = query_filter.csr
            if csr.shape[0] != n:
                raise ValueError("query_filter must have one row per query")
        ids = np.full((n, k), -1, dtype=np.int32)
        scores = np.full((n, k), -np.finfo(np.float32).max, dtype=np.float32)
        if n and k:
            backend = _BACKEND or _engine_backend
            got_ids, got_scores, counts = backend(items_arr, queries, k, norms, csr)
            k_out = got_ids.shape[1]
            mask = np.arange(k_out, dtype=np.int32)[None, :] < np.asarray(counts)[:, None]
            ids[:, :k_out] = np.where(mask, got_ids, -1)
            scores[:, :k_out] = np.where(mask, got_scores, -np.finfo(np.float32).max)
        return ids, scores


_PATCHED: tp.Dict[str, tp.Any] = {}


def patch_implicit_gpu(backend: tp.Optional[TopkBackend] = None) -> None:
    """Make `implicit.gpu.{HAS_CUDA, Matrix, COOMatrix, KnnQuery}` resolve to this module for an imported RecTools."""
    import importlib

    global _BACKEND  # pylint: disable=global-statement
    if _PATCHED:
        unpatch_implicit_gpu()
    _BACKEND = backend
    # import RecTools first: its modules copy `HAS_CUDA` at import time and must copy (and later get back) the original value
    mods = [importlib.import_module(m) for m in ("rectools.models.rank.rank_implicit", "rectools.models.vector")]
    gpu = importlib.import_module("implicit.gpu")
    for name in ("HAS_CUDA", "Matrix", "COOMatrix", "KnnQuery"):
        _PATCHED["gpu." + name] = (gpu, name, getattr(gpu, name, None))
        setattr(gpu, name, globals()[name])
    for mod in mods:
        if hasattr(mod, "HAS_CUDA"):
            _PATCHED[mod.__name__] = (mod, "HAS_CUDA", mod.HAS_CUDA)
            mod.HAS_CUDA = True


def unpatch_implicit_gpu() -> None:
    global _BACKEND  # pylint: disable=global-statement
    for obj, name, old in _PATCHED.values():
        if old is None:
            try:
                delattr(obj, name)
            except AttributeError:
                pass
        else:
            setattr(obj, name, old)
    _PATCHED.clear()
    _BACKEND = None

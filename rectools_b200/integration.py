"""Wiring into an installed RecTools (all imports of `rectools` are lazy: the package works without it).

Seams (SURVEY.md section 8b):
  * `VectorModel._recommend_u2i/_recommend_i2i` construct `ImplicitRanker(...)` inline (rectools/models/vector.py:66-72,
    :90-96; name imported at vector.py:28) and `EASEModel._recommend_u2i` does the same (rectools/models/ease.py:144,
    import at ease.py:31)  ->  `install()` rebinds that module-level name to `B200ImplicitRanker`.
  * `EASEModel._recommend_i2i` copies the weight rows of the targets and ranks them with numpy (rectools/models/ease.py:163-188)
    ->  `install()` rebinds it to `ease_recommend_i2i`, which ranks those rows where the u2i engine already holds them.
  * transformer models take `similarity_module_type` (rectools/models/nn/transformers/base.py:219, :423); their
    `DistanceSimilarityModule._recommend_u2i` builds a `TorchRanker` (rectools/models/nn/transformers/similarity.py:127-132)
    ->  `make_similarity_module()` returns a subclass that builds a `B200TorchRanker` instead, and
    `install(transformers=True)` rebinds the module-level `TorchRanker` of similarity.py and of lightning.py (item-to-item,
    `TransformerLightningModule._recommend_i2i`, lightning.py:428-449) for the stock module.
"""
from __future__ import annotations

import hashlib
import os
import threading
import typing as tp
from concurrent.futures import ThreadPoolExecutor

import numpy as np
from scipy import sparse

from .ranker import (
    B200Ranker, Devices, Distance, Engine, _as_distance, _dense_f32, _is_cuda_tensor, flatten_padded, new_engine, parse_devices,
    rank_object_rows_padded,
)

_ENGINE_CACHE: "tp.Dict[tp.Tuple, Engine]" = {}
_ENGINE_CACHE_MAX = 2
_CACHE_LOCK = threading.Lock()

_HASH_BLOCK = 1 << 15  # 64-bit words per block (256 KiB)
_HASH_WEIGHTS = np.random.default_rng(0x5EED).integers(1, 2**63, size=_HASH_BLOCK, dtype=np.uint64) | np.uint64(1)
_HASH_POOL: tp.Optional[ThreadPoolExecutor] = None


def content_hash(a: np.ndarray) -> bytes:
    """Digest of the WHOLE buffer of a C-contiguous array (shape and dtype included), position sensitive: every 64-bit
    word is multiplied by a fixed odd weight of its position inside a 256 KiB block and summed (wrapping), the block sums
    go through blake2b in order.  numpy releases the GIL, so the blocks are spread over a thread pool: ~10 ms per
    512 MB on a many-core host -- cheap next to the upload it saves, and unlike a sampled fingerprint it cannot miss an
    in-place refit (ADVICE r1, VERDICT r1 weak #3)."""
    global _HASH_POOL  # pylint: disable=global-statement
    a = np.ascontiguousarray(a)
    raw = a.reshape(-1).view(np.uint8)
    n_words = raw.size // 8
    words = raw[: n_words * 8].view(np.uint64)
    seg = 64 * _HASH_BLOCK  # words per task (16 MiB)

    def work(i: int) -> np.ndarray:
        chunk = words[i * seg : (i + 1) * seg]
        full = (len(chunk) // _HASH_BLOCK) * _HASH_BLOCK
        out = []
        if full:
            # (einsum: the weighted sums without the product temporary, 3x the multiply-then-sum rate; same wrapping result)
            out.append(np.einsum("ij,j->i", chunk[:full].reshape(-1, _HASH_BLOCK), _HASH_WEIGHTS))
        if full < len(chunk):
            rest = chunk[full:]
            out.append(np.array([np.einsum("i,i->", rest, _HASH_WEIGHTS[: len(rest)])], dtype=np.uint64))
        return np.concatenate(out) if out else np.empty(0, np.uint64)

    n_tasks = -(-n_words // seg) if n_words else 0
    if n_tasks > 1:
        if _HASH_POOL is None:
            _HASH_POOL = ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 1), thread_name_prefix="b200hash")
        parts = list(_HASH_POOL.map(work, range(n_tasks)))
    else:
        parts = [work(i) for i in range(n_tasks)]
    h = hashlib.blake2b(digest_size=16)
    for part in parts:
        h.update(part.tobytes())
    h.update(raw[n_words * 8 :].tobytes())
    h.update(repr((a.shape, a.dtype.str)).encode())
    return h.digest()


def cached_engine(objects: np.ndarray, cosine: bool, device: tp.Union[int, tp.Tuple[int, ...]], tc_mode: str) -> Engine:
    """`VectorModel` builds a new ranker on every `recommend()` call (vector.py:66); keep the resident object factors
    across calls instead of re-uploading them (the reference GPU path re-uploads per call, rank_implicit.py:156).
    Keyed by the CONTENT of the matrix.  Evicted engines are only dropped from the cache: a ranker that still holds one
    keeps it alive, the device memory is released when the last reference goes (`Engine.__del__`).  `device`: an int
    (one engine) or a tuple of devices (an `EngineGroup`); the two never share an entry, even for one device.
    Cached engines are always fp32 engines: `objects` is the fp32 matrix (its dtype is part of `content_hash`), and no
    engine kept at 16 bits (B200_F_OBJECTS_16BIT) is ever built or returned here."""
    key = (content_hash(objects), cosine, device, tc_mode)
    with _CACHE_LOCK:
        eng = _ENGINE_CACHE.get(key)
        if eng is not None:
            return eng
    eng = new_engine(objects, cosine=cosine, device=device, tc_mode=tc_mode)
    with _CACHE_LOCK:
        while len(_ENGINE_CACHE) >= _ENGINE_CACHE_MAX:
            _ENGINE_CACHE.pop(next(iter(_ENGINE_CACHE)))
        _ENGINE_CACHE[key] = eng
    return eng


def clear_engine_cache() -> None:
    with _CACHE_LOCK:
        _ENGINE_CACHE.clear()


class B200ImplicitRanker(B200Ranker):
    """`ImplicitRanker(distance, subjects_factors, objects_factors, num_threads=0, use_gpu=False)`-compatible
    constructor (rank_implicit.py:58-65) with a per-process engine cache keyed by the object matrix."""

    default_device: tp.Union[int, tp.Tuple[int, ...]] = 0  # a tuple: an engine group (install(device=[...]))
    default_tc_mode: str = "auto"

    def __init__(self, distance, subjects_factors, objects_factors, num_threads: int = 0, use_gpu: bool = False) -> None:
        dist = _as_distance(distance)
        engine = None
        subjects_key = None
        if dist != Distance.EUCLIDEAN and isinstance(objects_factors, np.ndarray):
            objects = _dense_f32(objects_factors)
            engine = cached_engine(objects, dist == Distance.COSINE, self.default_device, self.default_tc_mode)
            objects_factors = objects
            if isinstance(subjects_factors, np.ndarray) and not sparse.issparse(subjects_factors):
                subjects_factors = _dense_f32(subjects_factors)
                subjects_key = content_hash(subjects_factors)  # same content as in the previous call: stays resident
        super().__init__(
            dist, subjects_factors, objects_factors, num_threads=num_threads, use_gpu=use_gpu,
            device=self.default_device, tc_mode=self.default_tc_mode, engine=engine, subjects_key=subjects_key,
        )


class B200TorchRanker(B200Ranker):
    """`TorchRanker(distance, device, subjects_factors, objects_factors, batch_size=128, dtype=torch.float32)`-compatible
    constructor (rectools/models/rank/rank_torch.py:59-67).  `batch_size` is meaningless here (no score matrix is ever
    materialised) and `dtype` other than fp32 is ignored: inputs are cast to fp32 like `_normalize_tensor` does by default.

    Difference kept from the reference: `TorchRanker` filters on CSR *values* != 0 (rank_torch.py:143) whereas the
    implicit path uses the stored structure; explicit zeros are dropped here to keep the torch semantics.

    `devices` (not in the reference): rank on an engine group over these devices (a sequence or "all"); the factors'
    device is its home device.

    `keep_16bit` (not in the reference): fp16 / bf16 `objects_factors` stay at 16 bits in the engine, read in place with
    no fp32 master copy (the ranker keeps the tensor alive); False widens them into an fp32 copy.  Same results.

    One CUDA tensor passed as both factors (item-to-item, lightning.py:440-442) takes the identity route of `B200Ranker`:
    no copy of the catalogue; each call gathers its target rows in their own dtype.  Same results as a copy."""

    def __init__(self, distance, device, subjects_factors, objects_factors, batch_size: int = 128, dtype=None,
                 devices: tp.Optional[Devices] = None, keep_16bit: bool = True) -> None:
        dev_index = 0
        dev = str(device)
        if dev.startswith("cuda") and ":" in dev:
            dev_index = int(dev.split(":")[1])
        if hasattr(objects_factors, "detach") and dev.startswith("cuda") and not objects_factors.is_cuda:
            objects_factors = objects_factors.to(device)  # `TorchRanker` scores on `device` (rank_torch.py:135)
        super().__init__(distance, subjects_factors, objects_factors, device=dev_index if devices is None else devices,
                         keep_16bit=keep_16bit)
        self.batch_size = batch_size

    def rank(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None):
        if filter_pairs_csr is not None and filter_pairs_csr.nnz and (filter_pairs_csr.data == 0).any():
            filter_pairs_csr = filter_pairs_csr.copy()
            filter_pairs_csr.eliminate_zeros()
        return super().rank(subject_ids, k, filter_pairs_csr, sorted_object_whitelist)


_ORIGINALS: tp.Dict[tp.Any, tp.Any] = {}  # (name, module) tuples: rebound module-level names
_FAST_KEY = "VectorModel.recommend"
_EASE_I2I_KEY = "EASEModel._recommend_i2i"
_RERANK_KEY = "Reranker.recommend"
_POPULAR_KEY = "PopularModel._recommend_u2i"
_POPULAR_IN_CATEGORY_KEY = "PopularInCategoryModel._recommend_u2i"
_ITEM_KNN_KEY = "ImplicitItemKNNWrapperModel._recommend_u2i/_recommend_i2i"
_METRICS_KEY = "calc_metrics"
# the modules whose attribute `calc_metrics` install(metrics=True) rebinds: the definition, the package's re-export and
# `cross_validate`'s import (rectools/model_selection/cross_validate.py:20)
_METRICS_MODULES = ("rectools.metrics.scoring", "rectools.metrics", "rectools.model_selection.cross_validate")
# the transformer modules whose module-level `TorchRanker` ranks: u2i (`DistanceSimilarityModule._recommend_u2i`,
# similarity.py:127-132) and i2i (`TransformerLightningModule._recommend_i2i`, lightning.py:440-442)
_TRANSFORMER_MODULES = ("rectools.models.nn.transformers.similarity", "rectools.models.nn.transformers.lightning")


def transformer_ranker(ranker_factory: tp.Callable[..., tp.Any] = B200TorchRanker) -> tp.Callable[..., tp.Any]:
    """The `TorchRanker` stand-in `install(transformers=True)` binds: `ranker_factory` (a `TorchRanker`-signature class)
    on the device of `objects_factors`, as `TorchRanker` ranks (rank_torch.py:135).  When `install(device=...)` named a group
    that contains that device, the group ranks, with that device as home (`devices=`); host factors rank on the installed
    device."""

    def make(distance, device, subjects_factors, objects_factors, *args: tp.Any, **kwargs: tp.Any) -> tp.Any:
        installed = B200ImplicitRanker.default_device
        target = str(objects_factors.device if _is_cuda_tensor(objects_factors) else device)
        if target.startswith("cuda"):
            home = int(target.split(":")[1]) if ":" in target else 0
            if isinstance(installed, tuple) and home in installed:
                kwargs["devices"] = installed
        elif installed != 0:
            kwargs["devices"] = installed
        return ranker_factory(distance, device, subjects_factors, objects_factors, *args, **kwargs)

    return make


def ease_recommend_i2i(self, target_ids, dataset, k, sorted_item_ids_to_recommend):
    """`EASEModel._recommend_i2i` (rectools/models/ease.py:163-188) on the GPU: row t of `self.weight` is the score row of
    target t, and the engine of `_recommend_u2i` (cached by the content of `self.weight`) holds exactly that matrix, so the
    rows are ranked where they lie -- no copy of the rows, no extra device memory.  Returns the reference's triplet: best
    first, ids remapped through the whitelist, `min(k, n_pos)` entries per target for finite weights (what EASE fits).
    Unlike the reference, -inf and NaN weights are never returned, so a target with such entries may get fewer.  Tie order
    among equal scores is id ascending (the reference leaves it undefined).  Every call finds the engine through
    `cached_engine`, i.e. one `content_hash` of the whole weight per call.  A weight that is not a C-contiguous fp32 matrix (a float64 weight
    ranks in fp64 in the reference) goes to the original method."""
    weight = getattr(self, "weight", None)
    if not (isinstance(weight, np.ndarray) and weight.dtype == np.float32 and weight.ndim == 2 and weight.flags.c_contiguous):
        return _ORIGINALS[_EASE_I2I_KEY](self, target_ids, dataset, k, sorted_item_ids_to_recommend)
    engine = cached_engine(weight, False, B200ImplicitRanker.default_device, B200ImplicitRanker.default_tc_mode)
    target_ids, ids, scores, counts = rank_object_rows_padded(engine, target_ids, k, None, sorted_item_ids_to_recommend)
    return flatten_padded(target_ids, ids, scores, counts)


def install(device: Devices = 0, tc_mode: str = "auto", fast_recommend: bool = True, rerank: bool = False,
            popular: bool = False, transformers: bool = False, popular_in_category: bool = False, item_knn: bool = False,
            metrics: bool = False, ranker_factory: tp.Optional[tp.Callable[..., tp.Any]] = None) -> None:
    """Route `VectorModel` (ALS / PureSVD / LightFM / BPR / DSSM) and `EASEModel` ranking (u2i and i2i) through the B200
    engine.

    `device`: an int ranks on that GPU; a sequence of ints (`[0, 1, 2, 3]`) or "all" (every visible GPU) ranks on an
    engine group, one engine per entry, each call's rows split between them (same results; each member holds the whole
    catalogue).

    `fast_recommend`: also give `VectorModel` the vectorised `recommend()` of `rectools_b200.recommend` (cached viewed-items
    CSR, id maps by array indexing, no per-user Python loop); warm / cold targets and context models still go through
    `ModelBase.recommend` (rectools/models/base.py:385-519).

    `rerank`: also rebind the classmethod `Reranker.recommend` (rectools/models/ranking/candidate_ranking.py:203-236), the
    per-user top-k that ends `CandidateRankingModel.recommend`, to `rectools_b200.rerank.reranker_recommend` on the home
    device (`device`, or its first entry).

    `popular`: also rebind `PopularModel._recommend_u2i` (rectools/models/popular.py:229-255), the per-user loop over the
    popularity list, to `rectools_b200.popular.popular_recommend_u2i` on the home device.  `PopularInCategoryModel` ranks
    through its per-category `PopularModel`s, so it is served as well.

    `popular_in_category`: also rebind `PopularInCategoryModel._recommend_u2i` (rectools/models/popular_in_category.py:333-373),
    one `PopularModel` call per category and the mixing in pandas, to
    `rectools_b200.popular.popular_in_category_recommend_u2i` on the home device: every category's list and the mixing of
    each user in one kernel pass.  `popular=True` alone leaves this method as it is.

    `item_knn`: also rebind `ImplicitItemKNNWrapperModel._recommend_u2i` and `._recommend_i2i`
    (rectools/models/implicit_knn.py:152-255), one implicit `recommend` call or one numpy selection per target, to
    `rectools_b200.item_knn.item_knn_recommend_u2i` / `item_knn_recommend_i2i` on the home device: every user's scores
    accumulated from `model.similarity` in one sparse pass, and every target's neighbour row selected in one call.

    `metrics`: also rebind the module attribute `calc_metrics` of rectools.metrics.scoring, rectools.metrics and
    rectools.model_selection.cross_validate (so `cross_validate` scores each fold through it) to
    `rectools_b200.metrics.calc_metrics` on the home device: the classification and ranking metrics from one device join
    of the test interactions with the reco table, every value equal to the stock one.  A name imported before `install()`
    (`from rectools.metrics import calc_metrics`) keeps the stock function, as with the other rebound names.

    `transformers`: also rebind the module-level `TorchRanker` of rectools.models.nn.transformers.similarity (u2i of
    `DistanceSimilarityModule`) and of rectools.models.nn.transformers.lightning (item-to-item of
    `TransformerLightningModule`) to `transformer_ranker()`: SASRec / BERT4Rec / HSTU rank on the engine with their stock
    similarity module, so their configs stay serialisable.  Item-to-item passes one tensor as both factors, which
    `B200TorchRanker` ranks without a copy of the catalogue.  Needs `pytorch_lightning` (an ImportError names what is
    missing, and nothing is rebound).  `ranker_factory`: another `TorchRanker`-signature class to bind (the CPU tests plug an
    oracle-backed stand-in in; default `B200TorchRanker`)."""
    import importlib

    transformer_modules = []
    if transformers:
        for modname in _TRANSFORMER_MODULES:
            try:
                transformer_modules.append(importlib.import_module(modname))
            except ImportError as e:
                raise ImportError(f"install(transformers=True) needs the package {e.name!r} to import {modname}: {e}", name=e.name) from e
    B200ImplicitRanker.default_device = parse_devices(device)
    B200ImplicitRanker.default_tc_mode = tc_mode
    for modname in ("rectools.models.vector", "rectools.models.ease"):
        mod = importlib.import_module(modname)
        if modname not in _ORIGINALS:
            _ORIGINALS[modname] = mod.ImplicitRanker
        mod.ImplicitRanker = B200ImplicitRanker
    if _EASE_I2I_KEY not in _ORIGINALS:
        from rectools.models.ease import EASEModel

        _ORIGINALS[_EASE_I2I_KEY] = EASEModel._recommend_i2i  # pylint: disable=protected-access
        EASEModel._recommend_i2i = ease_recommend_i2i  # pylint: disable=protected-access
    if fast_recommend and _FAST_KEY not in _ORIGINALS:
        from rectools.models.base import ModelBase
        from rectools.models.vector import VectorModel

        from .recommend import recommend as fast
        from .recommend import recommend_to_items as fast_i2i

        def _recommend(self, users, dataset, k, filter_viewed, items_to_recommend=None, add_rank_col=True,
                       on_unsupported_targets="raise", context=None):
            return fast(self, users, dataset, k, filter_viewed, items_to_recommend, add_rank_col, on_unsupported_targets, context,
                        reference_recommend=lambda *a, **kw: ModelBase.recommend(self, *a, **kw))

        def _recommend_to_items(self, target_items, dataset, k, filter_itself=True, items_to_recommend=None, add_rank_col=True,
                                on_unsupported_targets="raise"):
            return fast_i2i(self, target_items, dataset, k, filter_itself, items_to_recommend, add_rank_col, on_unsupported_targets,
                            reference_recommend=lambda *a, **kw: ModelBase.recommend_to_items(self, *a, **kw))

        _recommend.__doc__ = ModelBase.recommend.__doc__
        _recommend_to_items.__doc__ = ModelBase.recommend_to_items.__doc__
        # (None: the attribute is inherited from ModelBase)
        _ORIGINALS[_FAST_KEY] = (VectorModel.__dict__.get("recommend"), VectorModel.__dict__.get("recommend_to_items"))
        VectorModel.recommend = _recommend
        VectorModel.recommend_to_items = _recommend_to_items
    if rerank and _RERANK_KEY not in _ORIGINALS:
        from rectools.models.ranking.candidate_ranking import Reranker

        from .rerank import reranker_recommend

        def _rerank_recommend(cls, scored_pairs, k, add_rank_col=True):  # pylint: disable=unused-argument
            home = B200ImplicitRanker.default_device
            return reranker_recommend(scored_pairs, k, add_rank_col, device=home[0] if isinstance(home, tuple) else home)

        _rerank_recommend.__doc__ = Reranker.recommend.__doc__
        _ORIGINALS[_RERANK_KEY] = Reranker.__dict__["recommend"]
        Reranker.recommend = classmethod(_rerank_recommend)
    if popular and _POPULAR_KEY not in _ORIGINALS:
        from rectools.models.popular import PopularModel

        from .popular import popular_recommend_u2i

        def _popular_recommend_u2i(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend):
            home = B200ImplicitRanker.default_device
            return popular_recommend_u2i(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend,
                                         device=home[0] if isinstance(home, tuple) else home)

        _popular_recommend_u2i.__doc__ = PopularModel._recommend_u2i.__doc__  # pylint: disable=protected-access
        _ORIGINALS[_POPULAR_KEY] = PopularModel.__dict__["_recommend_u2i"]
        PopularModel._recommend_u2i = _popular_recommend_u2i  # pylint: disable=protected-access
    if popular_in_category and _POPULAR_IN_CATEGORY_KEY not in _ORIGINALS:
        from rectools.models.popular_in_category import PopularInCategoryModel

        from .popular import popular_in_category_recommend_u2i

        def _in_category_recommend_u2i(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend):
            home = B200ImplicitRanker.default_device
            return popular_in_category_recommend_u2i(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend,
                                                     device=home[0] if isinstance(home, tuple) else home)

        _in_category_recommend_u2i.__doc__ = PopularInCategoryModel._recommend_u2i.__doc__  # pylint: disable=protected-access
        _ORIGINALS[_POPULAR_IN_CATEGORY_KEY] = PopularInCategoryModel.__dict__["_recommend_u2i"]
        PopularInCategoryModel._recommend_u2i = _in_category_recommend_u2i  # pylint: disable=protected-access
    if item_knn and _ITEM_KNN_KEY not in _ORIGINALS:
        from rectools.models.implicit_knn import ImplicitItemKNNWrapperModel

        from .item_knn import item_knn_recommend_i2i, item_knn_recommend_u2i

        def _knn_recommend_u2i(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend):
            home = B200ImplicitRanker.default_device
            return item_knn_recommend_u2i(self, user_ids, dataset, k, filter_viewed, sorted_item_ids_to_recommend,
                                          device=home[0] if isinstance(home, tuple) else home)

        def _knn_recommend_i2i(self, target_ids, dataset, k, sorted_item_ids_to_recommend):
            home = B200ImplicitRanker.default_device
            return item_knn_recommend_i2i(self, target_ids, dataset, k, sorted_item_ids_to_recommend,
                                          device=home[0] if isinstance(home, tuple) else home)

        cls = ImplicitItemKNNWrapperModel
        _knn_recommend_u2i.__doc__ = cls._recommend_u2i.__doc__  # pylint: disable=protected-access
        _knn_recommend_i2i.__doc__ = cls._recommend_i2i.__doc__  # pylint: disable=protected-access
        _ORIGINALS[_ITEM_KNN_KEY] = {name: cls.__dict__[name] for name in ("_recommend_u2i", "_recommend_i2i")}
        cls._recommend_u2i = _knn_recommend_u2i  # pylint: disable=protected-access
        cls._recommend_i2i = _knn_recommend_i2i  # pylint: disable=protected-access
    if metrics and _METRICS_KEY not in _ORIGINALS:
        from .metrics import calc_metrics as device_calc_metrics

        modules = [importlib.import_module(modname) for modname in _METRICS_MODULES]

        def _calc_metrics(metrics, reco, interactions=None, prev_interactions=None, catalog=None, ref_reco=None):  # pylint: disable=redefined-outer-name
            home = B200ImplicitRanker.default_device
            return device_calc_metrics(metrics, reco, interactions, prev_interactions, catalog, ref_reco,
                                       device=home[0] if isinstance(home, tuple) else home)

        _calc_metrics.__doc__ = modules[0].calc_metrics.__doc__
        _ORIGINALS[_METRICS_KEY] = {mod.__name__: mod.calc_metrics for mod in modules}
        for mod in modules:
            mod.calc_metrics = _calc_metrics
    if transformer_modules:
        bound = transformer_ranker(ranker_factory or B200TorchRanker)
        for mod in transformer_modules:
            _ORIGINALS.setdefault(("TorchRanker", mod.__name__), mod.TorchRanker)
            mod.TorchRanker = bound


def uninstall() -> None:
    import importlib

    for key in [k for k in _ORIGINALS if isinstance(k, tuple)]:
        setattr(importlib.import_module(key[1]), key[0], _ORIGINALS.pop(key))
    if _FAST_KEY in _ORIGINALS:
        from rectools.models.vector import VectorModel

        for name, orig in zip(("recommend", "recommend_to_items"), _ORIGINALS.pop(_FAST_KEY)):
            if orig is None:
                delattr(VectorModel, name)
            else:
                setattr(VectorModel, name, orig)
    if _RERANK_KEY in _ORIGINALS:
        from rectools.models.ranking.candidate_ranking import Reranker

        Reranker.recommend = _ORIGINALS.pop(_RERANK_KEY)
    if _POPULAR_KEY in _ORIGINALS:
        from rectools.models.popular import PopularModel

        PopularModel._recommend_u2i = _ORIGINALS.pop(_POPULAR_KEY)  # pylint: disable=protected-access
    if _POPULAR_IN_CATEGORY_KEY in _ORIGINALS:
        from rectools.models.popular_in_category import PopularInCategoryModel

        PopularInCategoryModel._recommend_u2i = _ORIGINALS.pop(_POPULAR_IN_CATEGORY_KEY)  # pylint: disable=protected-access
    if _ITEM_KNN_KEY in _ORIGINALS:
        from rectools.models.implicit_knn import ImplicitItemKNNWrapperModel

        for name, orig in _ORIGINALS.pop(_ITEM_KNN_KEY).items():
            setattr(ImplicitItemKNNWrapperModel, name, orig)
    if _METRICS_KEY in _ORIGINALS:
        for modname, orig in _ORIGINALS.pop(_METRICS_KEY).items():
            importlib.import_module(modname).calc_metrics = orig
    if _EASE_I2I_KEY in _ORIGINALS:
        from rectools.models.ease import EASEModel

        EASEModel._recommend_i2i = _ORIGINALS.pop(_EASE_I2I_KEY)  # pylint: disable=protected-access
    for modname, orig in list(_ORIGINALS.items()):
        importlib.import_module(modname).ImplicitRanker = orig
        del _ORIGINALS[modname]
    clear_engine_cache()


def make_similarity_module(
    ranker_factory: tp.Optional[tp.Callable[..., tp.Any]] = None, devices: tp.Optional[Devices] = None,
    keep_16bit: tp.Optional[bool] = None,
) -> type:
    """`similarity_module_type` for SASRec / BERT4Rec / HSTU (rectools/models/nn/transformers/base.py:219, :423): the
    reference's `DistanceSimilarityModule` with `B200TorchRanker` as the scorer of `_recommend_u2i`
    (similarity.py:117-140).  `item_embs` stays on its device (and in its dtype: fp16 / bf16 embeddings are handed to the
    engine as they are); the filter stays a CSR (the reference densifies [batch, n_items] per batch, rank_torch.py:138-144).
    `ranker_factory`: another `TorchRanker`-signature class (the CPU tests plug an oracle-backed stand-in in).
    `devices`: rank on an engine group over these devices (a sequence or "all", passed to the factory as `devices=`);
    None ranks on the device of `item_embs`.
    `keep_16bit`: passed to the factory as `keep_16bit=` (None: the factory's default, which for `B200TorchRanker` keeps
    fp16 / bf16 `item_embs` at 16 bits in the engine; False widens them into an fp32 copy)."""
    from rectools.models.nn.transformers.similarity import DistanceSimilarityModule  # needs torch only

    factory = ranker_factory or B200TorchRanker
    group_kw = {} if devices is None else {"devices": parse_devices(devices)}
    if keep_16bit is not None:
        group_kw["keep_16bit"] = bool(keep_16bit)

    class B200DistanceSimilarityModule(DistanceSimilarityModule):
        def _recommend_u2i(self, user_embs, item_embs, user_ids, k, sorted_item_ids_to_recommend, ui_csr_for_filter):
            ranker = factory(
                distance=self.distance, device=item_embs.device, subjects_factors=user_embs[user_ids],
                objects_factors=item_embs, **group_kw,
            )
            user_ids_indices, all_reco_ids, all_scores = ranker.rank(
                subject_ids=np.arange(len(user_ids)), k=k, filter_pairs_csr=ui_csr_for_filter,
                sorted_object_whitelist=sorted_item_ids_to_recommend,
            )
            return user_ids[user_ids_indices], all_reco_ids, all_scores

    return B200DistanceSimilarityModule

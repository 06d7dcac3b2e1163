"""rectools_b200: an H100-native (sm_90a) scoring + top-K engine for RecTools' vector-ranking path.

Public surface (host-side mirror of `rectools.models.rank`):
  * `Distance`, `B200Ranker`              -- drop-in for `ImplicitRanker` / the `Ranker` protocol
  * `B200TorchRanker`                     -- `TorchRanker`-signature adapter (transformer id-embedding scorers)
  * `install()` / `uninstall()`           -- rebind the ranker used by `VectorModel` / `EASEModel` in an installed rectools
  * `recommend()`                         -- vectorised `ModelBase.recommend` around the ranker (cached viewed CSR, id maps, table)
  * `EngineGroup`                         -- one engine per GPU of the host (`device=[...]` / "all"), rows split between them
  * `rank_pairs()`, `reranker_recommend()` -- per-group top-k of scored pairs (`Reranker.recommend`, install(rerank=True))
  * `rank_list()`                         -- a shared ordered list minus each row's viewed ids (`PopularModel`, install(popular=True))
  * `rank_list_mix()`                     -- per-category lists minus viewed ids, mixed (`PopularInCategoryModel`,
                                             install(popular_in_category=True))
  * `ShardedB200Ranker`                   -- item-sharded multi-GPU ranking (one process per GPU, NCCL all-gather + merge)
The CUDA library is `rectools_b200/libb200rank.so` (C ABI: include/b200_rank.h); build it with
`python -m rectools_b200.build`.  There is no CPU fallback.
"""
from .ranker import B200Ranker, Distance, Engine, EngineGroup, flatten_padded  # noqa: F401
from .integration import B200ImplicitRanker, B200TorchRanker, install, uninstall  # noqa: F401
from .recommend import recommend, recommend_to_items  # noqa: F401
from .rerank import rank_pairs, reranker_recommend  # noqa: F401
from .popular import rank_list, rank_list_mix  # noqa: F401

__all__ = [
    "B200Ranker",
    "B200ImplicitRanker",
    "B200TorchRanker",
    "Distance",
    "Engine",
    "EngineGroup",
    "flatten_padded",
    "install",
    "rank_list",
    "rank_list_mix",
    "rank_pairs",
    "recommend",
    "recommend_to_items",
    "reranker_recommend",
    "uninstall",
]
__version__ = "0.1.0"

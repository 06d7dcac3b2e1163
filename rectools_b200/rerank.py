"""Scored pairs on the GPU (engine path 6, `b200_rank_topk_pairs`): the last step of RecTools' two-stage model.

`CandidateRankingModel.recommend` (rectools/models/ranking/candidate_ranking.py:794-868) ends in
`Reranker.recommend(scored_pairs, k, add_rank_col)` (:203-236), which keeps the k best scored pairs of each user with one
pandas sort per user.  `reranker_recommend` returns that result from one segmented selection on the device:

  * users in order of first occurrence, NA users dropped (`groupby(sort=False)`, `dropna=True`);
  * within a user, score descending: -0 equals +0, +-inf are ordinary values, NaN scores come last and are kept when the
    user has fewer than k other rows; float64 is ordered as float64, float32 as float32, int64 / int32 exactly;
  * ties by input position ascending (the reference's numpy quicksort leaves their order to the implementation);
  * every column with its dtype, the index reset, and `rank` (cumcount + 1, int64) added or overwritten.

Other score dtypes (bool, object, pandas extension dtypes), a categorical user column and a k that is not a positive int
go to the original method unchanged.  `pd.factorize` of the user column runs on the host.
"""
from __future__ import annotations

import ctypes as C
import typing as tp

import numpy as np

from . import _lib

_SCORE_TYPES = {
    np.dtype(np.float64): _lib.PAIRS_F64,
    np.dtype(np.float32): _lib.PAIRS_F32,
    np.dtype(np.int64): _lib.PAIRS_I64,
    np.dtype(np.int32): _lib.PAIRS_I32,
}
_TORCH_SCORE_TYPES = {"torch.float64": _lib.PAIRS_F64, "torch.float32": _lib.PAIRS_F32, "torch.int64": _lib.PAIRS_I64,
                      "torch.int32": _lib.PAIRS_I32}
_K_MAX = 2**31 - 1


def rank_pairs(group_codes, scores, k: int, device: int = 0, n_groups: tp.Optional[int] = None,
               stats: tp.Optional[tp.Dict[str, tp.Any]] = None):
    """The k best rows of each group: `(positions, offsets)`, group g's rows being `positions[offsets[g]:offsets[g+1]]`,
    input positions ordered by (score desc, position asc).

    `group_codes`: int64 codes in [0, n_groups), -1 drops the row.  `scores`: float64 / float32 / int64 / int32 of the
    same length.  numpy arrays are ranked on `device` and give numpy results; CUDA tensors are read in place on their
    device, on its current stream, and give CUDA tensors.  `n_groups`: None means max(code) + 1.  `stats`: a dict that
    receives the call's `b200_rank_stats`."""
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1:
        raise ValueError(f"k must be a positive int, got {k!r}")
    if hasattr(group_codes, "is_cuda") and group_codes.is_cuda:
        return _rank_pairs_device(group_codes, scores, int(k), n_groups, stats)
    codes = np.ascontiguousarray(group_codes, dtype=np.int64).reshape(-1)
    sc = np.ascontiguousarray(scores).reshape(-1)
    if sc.dtype not in _SCORE_TYPES:
        raise TypeError(f"scores must be float64, float32, int64 or int32, got {sc.dtype}")
    if len(sc) != len(codes):
        raise ValueError(f"group_codes and scores differ in length ({len(codes)} != {len(sc)})")
    n = len(codes)
    if n_groups is None:
        n_groups = int(codes.max()) + 1 if n else 0
    k = min(int(k), max(n, 1), _K_MAX)  # no group has more than n rows
    offsets = np.empty(n_groups + 1, dtype=np.int64)
    positions = np.empty(min(n, n_groups * k), dtype=np.int64)
    st = _lib.Stats()
    _lib.check(_lib.load().b200_rank_topk_pairs(
        int(device), None, n, codes.ctypes.data, sc.ctypes.data, _SCORE_TYPES[sc.dtype], n_groups, k, 0,
        positions.ctypes.data if len(positions) else None, offsets.ctypes.data, C.byref(st),
    ))
    if stats is not None:
        stats.update(st.as_dict())
    return positions[: offsets[-1]], offsets


def _rank_pairs_device(codes, scores, k, n_groups, stats):
    import torch

    if not (hasattr(scores, "is_cuda") and scores.is_cuda and scores.device == codes.device):
        raise ValueError("group_codes and scores must be CUDA tensors on one device")
    if codes.dtype != torch.int64:
        raise TypeError(f"group_codes must be int64, got {codes.dtype}")
    stype = _TORCH_SCORE_TYPES.get(str(scores.dtype))
    if stype is None:
        raise TypeError(f"scores must be float64, float32, int64 or int32, got {scores.dtype}")
    codes, scores = codes.reshape(-1).contiguous(), scores.reshape(-1).contiguous()
    if codes.numel() != scores.numel():
        raise ValueError(f"group_codes and scores differ in length ({codes.numel()} != {scores.numel()})")
    n = codes.numel()
    if n_groups is None:
        n_groups = int(codes.max()) + 1 if n else 0
    k = min(k, max(n, 1), _K_MAX)
    dev = codes.device
    offsets = torch.empty(n_groups + 1, dtype=torch.int64, device=dev)
    positions = torch.empty(min(n, n_groups * k), dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev)
    st = _lib.Stats()
    _lib.check(_lib.load().b200_rank_topk_pairs(
        dev.index, stream.cuda_stream or None, n, codes.data_ptr(), scores.data_ptr(), stype, n_groups, k,
        _lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE, positions.data_ptr() if positions.numel() else None,
        offsets.data_ptr(), C.byref(st),
    ))
    if stats is not None:
        stats.update(st.as_dict())
    return positions[: int(offsets[-1])], offsets


def _served(scored_pairs, k) -> bool:
    """Whether `reranker_recommend` gives the reference's result itself (else it calls the original method)."""
    import pandas as pd
    from rectools import Columns

    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1:
        return False
    if not isinstance(scored_pairs, pd.DataFrame) or Columns.User not in scored_pairs or Columns.Score not in scored_pairs:
        return False
    if not scored_pairs.columns.is_unique:
        return False
    score_dtype = scored_pairs[Columns.Score].dtype
    if not isinstance(score_dtype, np.dtype) or score_dtype not in _SCORE_TYPES:
        return False
    return not isinstance(scored_pairs[Columns.User].dtype, pd.CategoricalDtype)


def _original_recommend():
    """`Reranker.recommend` as RecTools defines it, also while `install(rerank=True)` has rebound it."""
    from rectools.models.ranking.candidate_ranking import Reranker

    from .integration import _ORIGINALS, _RERANK_KEY

    orig = _ORIGINALS.get(_RERANK_KEY)
    return orig.__get__(None, Reranker) if orig is not None else Reranker.recommend


def reranker_recommend(scored_pairs, k: int, add_rank_col: bool = True, device: int = 0, stats: tp.Optional[tp.Dict[str, tp.Any]] = None):
    """`Reranker.recommend(scored_pairs, k, add_rank_col)` (rectools/models/ranking/candidate_ranking.py:203-236) with the
    per-user top-k on `device`; see the module docstring for the result.  `stats` (not in the reference): a dict that
    receives the call's `b200_rank_stats` when the GPU ranks it."""
    if not _served(scored_pairs, k):
        return _original_recommend()(scored_pairs, k, add_rank_col)
    import pandas as pd
    from rectools import Columns

    codes, uniques = pd.factorize(scored_pairs[Columns.User], sort=False, use_na_sentinel=True)
    positions, offsets = rank_pairs(codes, scored_pairs[Columns.Score].to_numpy(), int(k), device=device,
                                    n_groups=len(uniques), stats=stats)
    reco = scored_pairs.take(positions).reset_index(drop=True)
    if add_rank_col:
        starts = np.repeat(offsets[:-1], np.diff(offsets))
        reco[Columns.Rank] = np.arange(len(positions), dtype=np.int64) - starts + 1
    return reco

"""numpy restatement of path 6 (`b200_rank_topk_pairs`, `rectools_b200.rerank`): the order key and the per-group top-k
by (key descending, position ascending), stable, with no GPU.  Shared by the CPU and GPU tests of scored pairs."""
import numpy as np

SIGN = np.uint64(1 << 63)


def order_key(scores: np.ndarray) -> np.ndarray:
    """Descending uint64 order key.  Floats (fp32 widened exactly): -0 -> +0, NaN -> 0 (below -inf), then the IEEE
    order-preserving map; ints: the sign bit flipped."""
    s = np.asarray(scores)
    if s.dtype.kind == "f":
        v = s.astype(np.float64)
        v = np.where(v == 0, 0.0, v)
        b = v.view(np.uint64)
        key = np.where((b >> np.uint64(63)) == 1, ~b, b | SIGN)
        key[np.isnan(v)] = 0
        return key
    return s.astype(np.int64).view(np.uint64) ^ SIGN


def rank_pairs_np(codes, scores, k: int, n_groups: int):
    """(positions, offsets) of the k best rows per group: lexsort on position, key and code."""
    codes = np.asarray(codes, dtype=np.int64)
    key = order_key(scores)
    pos = np.arange(len(codes), dtype=np.int64)
    order = np.lexsort((pos, ~key, codes))
    order = order[codes[order] >= 0]
    c = codes[order]
    counts = np.bincount(c, minlength=n_groups).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
    within = np.arange(len(order), dtype=np.int64) - starts[c] if len(order) else np.zeros(0, np.int64)
    kept = np.minimum(counts, k)
    offsets = np.concatenate([[0], np.cumsum(kept)]).astype(np.int64)
    return order[within < k].astype(np.int64), offsets


def reranker_recommend_np(scored_pairs, k: int, add_rank_col: bool = True):
    """`Reranker.recommend`'s result under the fixed tie rule (position ascending), from the numpy restatement."""
    import pandas as pd

    codes, uniques = pd.factorize(scored_pairs["user_id"], sort=False, use_na_sentinel=True)
    positions, offsets = rank_pairs_np(codes, scored_pairs["score"].to_numpy(), k, len(uniques))
    reco = scored_pairs.take(positions).reset_index(drop=True)
    if add_rank_col:
        reco["rank"] = np.arange(len(positions), dtype=np.int64) - np.repeat(offsets[:-1], np.diff(offsets)) + 1
    return reco

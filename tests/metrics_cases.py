"""Seeded reco / interactions tables for the path-10 tests (tests/test_metrics_cpu.py, tests/test_gpu_metrics.py) and
scripts/metrics_ab.py, and the metric dicts they are scored with."""
from __future__ import annotations

import typing as tp

import numpy as np

USER, ITEM, RANK = "user_id", "item_id", "rank"


def tables(seed: int, n_users: int = 60, n_items: int = 40, k_reco: int = 10, max_test: int = 8, hit_share: float = 0.3,
           dup_share: float = 0.1, id_dtype: tp.Any = np.int64, shuffle: bool = True, extra_test_users: int = 5,
           extra_reco_users: int = 5, ragged: bool = True):
    """(reco, interactions) DataFrames.  Each reco user gets up to `k_reco` distinct items with ranks 1..len (a ragged
    list when `ragged`); each test user 1..`max_test` rows, about `hit_share` of them taken from its reco list, with
    `dup_share` of the rows repeated; `extra_test_users` test users have no reco and `extra_reco_users` reco users no test
    rows.  `shuffle` interleaves the users in the interactions, so first-appearance order is not sorted order.  Ids are
    spread (not 0..n) and cast to `id_dtype`."""
    import pandas as pd

    rng = np.random.default_rng(seed)
    user_ids = rng.choice(np.arange(3, 50 * (n_users + extra_test_users + extra_reco_users) + 3), replace=False,
                          size=n_users + extra_test_users + extra_reco_users)
    item_ids = rng.choice(np.arange(7, 40 * n_items + 7), replace=False, size=n_items)
    both, test_only, reco_only = (user_ids[:n_users], user_ids[n_users : n_users + extra_test_users],
                                  user_ids[n_users + extra_test_users :])
    k_items = min(k_reco, n_items)
    ru, ri, rr = [], [], []
    lists = {}
    for u in np.concatenate([both, reco_only]):
        length = int(rng.integers(1, k_items + 1)) if ragged else k_items
        items = rng.choice(item_ids, size=length, replace=False)
        lists[u] = items
        ru.append(np.full(length, u))
        ri.append(items)
        rr.append(np.arange(1, length + 1))
    iu, ii = [], []
    for u in np.concatenate([both, test_only]):
        m = int(rng.integers(1, max_test + 1))
        own = lists.get(u)
        for _ in range(m):
            if own is not None and rng.random() < hit_share:
                i = own[rng.integers(len(own))]
            else:
                i = item_ids[rng.integers(len(item_ids))]
            iu.append(u)
            ii.append(i)
            if rng.random() < dup_share:
                iu.append(u)
                ii.append(i)
    iu, ii = np.array(iu), np.array(ii)
    if shuffle:
        p = rng.permutation(len(iu))
        iu, ii = iu[p], ii[p]
    reco = pd.DataFrame({USER: np.concatenate(ru).astype(id_dtype), ITEM: np.concatenate(ri).astype(id_dtype),
                         RANK: np.concatenate(rr).astype(np.int64)})
    reco = reco.sample(frac=1.0, random_state=seed).reset_index(drop=True)  # the reco table in no particular order
    interactions = pd.DataFrame({USER: iu.astype(id_dtype), ITEM: ii.astype(id_dtype)})
    return reco, interactions


def served_metrics(ks: tp.Sequence[int] = (1, 3, 10), log_bases: tp.Sequence[float] = (2, 3, 10)) -> tp.Dict[str, tp.Any]:
    """Every served metric at every k, NDCG at every log base and both variants, MAP both ways, in a mixed dict order."""
    from rectools.metrics import MAP, MCC, MRR, NDCG, Accuracy, F1Beta, HitRate, Precision, Recall

    out: tp.Dict[str, tp.Any] = {}
    for k in ks:
        out[f"ndcg@{k}"] = NDCG(k=k)
        out[f"prec@{k}"] = Precision(k=k)
        out[f"map@{k}"] = MAP(k=k)
        out[f"rprec@{k}"] = Precision(k=k, r_precision=True)
        out[f"recall@{k}"] = Recall(k=k)
        out[f"mrr@{k}"] = MRR(k=k)
        out[f"f1@{k}"] = F1Beta(k=k)
        out[f"f2@{k}"] = F1Beta(k=k, beta=2.0)
        out[f"hit@{k}"] = HitRate(k=k)
        out[f"acc@{k}"] = Accuracy(k=k)
        out[f"mcc@{k}"] = MCC(k=k)
        out[f"map_k@{k}"] = MAP(k=k, divide_by_k=True)
        for base in log_bases:
            out[f"ndcg_b{base}@{k}"] = NDCG(k=k, log_base=base)
            out[f"ndcg_ach_b{base}@{k}"] = NDCG(k=k, log_base=base, divide_by_achievable=True)
    return out


def nine_metrics(k: int = 10) -> tp.Dict[str, tp.Any]:
    """Precision, Recall, HitRate, F1Beta, Accuracy, MCC, MAP, NDCG and MRR at one k."""
    from rectools.metrics import MAP, MCC, MRR, NDCG, Accuracy, F1Beta, HitRate, Precision, Recall

    return {f"precision@{k}": Precision(k=k), f"recall@{k}": Recall(k=k), f"hitrate@{k}": HitRate(k=k), f"f1@{k}": F1Beta(k=k),
            f"accuracy@{k}": Accuracy(k=k), f"mcc@{k}": MCC(k=k), f"map@{k}": MAP(k=k), f"ndcg@{k}": NDCG(k=k), f"mrr@{k}": MRR(k=k)}


def large_tables(n_users: int, seed: int = 0, k: int = 10, n_items: int = 20_000, max_test: int = 10, hit_share: float = 0.3):
    """Vectorised synthetic tables at scale: every user has a reco list of k distinct items (ranks 1..k) and 1..max_test
    test rows, each a hit (an item of its list) with probability `hit_share`; users interleaved in the interactions."""
    import pandas as pd

    rng = np.random.default_rng(seed)
    users = np.arange(n_users, dtype=np.int64) * 7 + 11
    # k distinct items per user: a random start and a random odd stride modulo n_items (n_items even -> odd strides are units
    # only for odd n_items, so use a prime-sized catalogue)
    n_cat = n_items if n_items % 2 else n_items + 1
    start = rng.integers(0, n_cat, size=n_users)
    step = rng.integers(1, n_cat // k, size=n_users)
    items = (start[:, None] + step[:, None] * np.arange(k)[None, :]) % n_cat
    reco = pd.DataFrame({USER: np.repeat(users, k), ITEM: items.reshape(-1).astype(np.int64),
                         RANK: np.tile(np.arange(1, k + 1, dtype=np.int64), n_users)})
    m = rng.integers(1, max_test + 1, size=n_users)
    iu_idx = np.repeat(np.arange(n_users), m)
    hit = rng.random(len(iu_idx)) < hit_share
    ii = np.where(hit, items[iu_idx, rng.integers(0, k, size=len(iu_idx))], rng.integers(0, n_cat, size=len(iu_idx)))
    p = rng.permutation(len(iu_idx))
    interactions = pd.DataFrame({USER: users[iu_idx[p]], ITEM: ii[p].astype(np.int64)})
    return reco, interactions

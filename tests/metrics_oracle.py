"""A numpy definition of what `b200_rank_metrics` (engine path 10) returns, written from the stock pandas / numpy / scipy
operations it replaces, with the same signature and result as `rectools_b200.metrics.device_metrics`:

- the join: interaction row j is a hit of rank r when the reco table holds its (user, item) pair with rank r;
- per distinct test user in ascending id: its rows (LIKED), its hits of rank <= k per k (TP), its smallest hit rank;
- NDCG: pandas' compensated group sum (`group_sum`: y = v - c, t = s + y, c = (t - s) - y, NaN c reset to 0) of the term
  of each hit, in row order; a hit past the term table adds 0.0;
- MAP: per distinct hit rank r <= k, ascending, the precision C(r) / r, C(r) = hits of rank <= r counted with repeats,
  summed as np.add.reduceat sums a row of scipy's CSR: the first precision plus numpy's pairwise sum of the rest, which is
  restated here (`pairwise_sum`) rather than called, so that the CPU tests check the device's order against stock.
Python floats are IEEE doubles and every operation below is one rounded operation, as on the device."""
from __future__ import annotations

import typing as tp

import numpy as np


def pairwise_sum(a: tp.Sequence[float]) -> float:
    """numpy's pairwise summation (`@TYPE@_pairwise_sum`): in order below 8 entries, 8 accumulators up to 128, halves
    (rounded down to a multiple of 8) above."""
    n = len(a)
    if n < 8:
        r = -0.0
        for x in a:
            r = r + x
        return r
    if n <= 128:
        acc = [a[j] for j in range(8)]
        i = 8
        while i < n - (n % 8):
            for j in range(8):
                acc[j] = acc[j] + a[i + j]
            i += 8
        res = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]))
        while i < n:
            res = res + a[i]
            i += 1
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


def kahan_sum(values: tp.Iterable[float]) -> float:
    s = c = 0.0
    for v in values:
        if v != v:
            continue
        y = v - c
        t = s + y
        c = (t - s) - y
        if c != c:
            c = 0.0
        s = t
    return s


def device_metrics_np(inter_users, inter_items, reco_users, reco_items, reco_ranks, ks, ndcg_tables, want_map,
                      device: int = 0, stats=None) -> tp.Dict[str, tp.Any]:  # pylint: disable=unused-argument
    iu, ii = np.asarray(inter_users, np.int64), np.asarray(inter_items, np.int64)
    ru, ri, rr = (np.asarray(a, np.int64) for a in (reco_users, reco_items, reco_ranks))
    keys = list(zip(ru.tolist(), ri.tolist()))
    flags = (1 if len(set(keys)) != len(keys) else 0) | (2 if len(rr) and rr.min() < 1 else 0)
    n_k, n_t = len(ks), len(ndcg_tables)
    if flags or len(iu) == 0:
        e = np.zeros(0, np.int64)
        return {"flags": flags, "users": e, "first_order": e, "liked": e, "min_rank": e, "tp": np.zeros((n_k, 0), np.int64),
                "map": np.zeros((n_k, 0)) if want_map else None, "ndcg": np.zeros((n_t, 0))}
    rank_of = dict(zip(keys, rr.tolist()))
    hit = np.array([rank_of.get(p, 0) for p in zip(iu.tolist(), ii.tolist())], dtype=np.int64)
    users, inv = np.unique(iu, return_inverse=True)
    U, n = len(users), len(iu)
    liked = np.bincount(inv, minlength=U).astype(np.int64)
    first_row = np.full(U, n, dtype=np.int64)
    np.minimum.at(first_row, inv, np.arange(n))
    first_order = np.argsort(first_row, kind="stable").astype(np.int64)
    is_hit = hit >= 1
    tp_ = np.stack([np.bincount(inv, weights=is_hit & (hit <= k), minlength=U).astype(np.int64) for k in ks]) if n_k \
        else np.zeros((0, U), np.int64)
    min_rank = np.zeros(U, dtype=np.int64)
    order = np.argsort(inv, kind="stable")  # each user's rows in row order
    bounds = np.concatenate([[0], np.cumsum(liked)])
    ndcg = np.zeros((n_t, U))
    map_ = np.zeros((n_k, U)) if want_map else None
    for s in range(U):
        rows = order[bounds[s] : bounds[s + 1]]
        ranks = [int(r) for r in hit[rows] if r >= 1]
        min_rank[s] = min(ranks) if ranks else 0
        for t, T in enumerate(ndcg_tables):
            ndcg[t, s] = kahan_sum(float(T[r - 1]) if r <= len(T) else 0.0 for r in ranks)
        if want_map:
            distinct, counts = np.unique([r for r in ranks if r <= max(ks)], return_counts=True)
            prec = [float(c) / float(r) for c, r in zip(np.cumsum(counts).tolist(), distinct.tolist())]
            for q, k in enumerate(ks):
                p = prec[: int(np.searchsorted(distinct, k, side="right"))]
                map_[q, s] = p[0] + pairwise_sum(p[1:]) if p else 0.0
    return {"flags": 0, "users": users.astype(np.int64), "first_order": first_order, "liked": liked, "min_rank": min_rank,
            "tp": tp_, "map": map_, "ndcg": ndcg}

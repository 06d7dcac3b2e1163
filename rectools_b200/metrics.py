"""RecTools' `calc_metrics` with its classification and ranking metrics computed from one device join (engine path 10,
`b200_rank_metrics`).

The stock function (rectools/metrics/scoring.py:37-223) left-merges the test interactions with the whole reco table
(`merge_reco`, rectools/metrics/base.py:81-103) and runs each family's groupbys over the merged rows in pandas.  Here the
join and the per-user reductions run on the GPU and return, per distinct test user: its interaction rows (LIKED), its hits
of rank <= k per k (TP), its smallest hit rank, pandas' compensated sum of its NDCG terms per (k, log_base, variant) and
its MAP precision sums per k.  The host then does what stock does with those arrays:

- classification: the confusion table of `calc_confusions` (user index, int64 LIKED / TP / FP / FN) goes to each metric's
  own `calc_from_confusion_df`;
- ranking: the per-user values are put in the order stock averages them (first appearance in the interactions for NDCG
  and MRR, sorted user id for MAP) and averaged by `pd.Series(values).mean()`, as stock does.

So every value is the stock value, bit for bit.  Any other metric of the dict (AUC, novelty, popularity, diversity,
serendipity, intersection, DQ, catalog, custom) is computed by the stock function on the rest of the dict, with the same
arguments, and appended after these two families: stock's order.

Served: exact `Precision`, `Recall`, `F1Beta`, `HitRate`, `Accuracy`, `MCC`, `MAP`, `NDCG` (a real `log_base` > 1) and `MRR`
instances with `debias_config=None` and an int `k` >= 1.  The whole call goes to the stock function when
- no metric of these two families is in the dict, `interactions` is None or empty, or `catalog` is None with an
  `Accuracy` / `MCC` present (stock then raises its own ValueError);
- a metric of these families is not served (a subclass, a debias config);
- a user / item column of either table, or the rank column, is missing or not a plain numpy integer dtype, a uint64 id
  is >= 2^63, or the two tables' id dtypes have no common integer type;
- the reco table holds a (user, item) pair twice (stock's merge would multiply rows) or a rank below 1, both found on the
  device;
- the device refuses an allocation (a RuntimeWarning names it).
"""
from __future__ import annotations

import ctypes as C
import time
import typing as tp
import warnings

import numpy as np

from . import _lib

if tp.TYPE_CHECKING:
    import pandas as pd

_U63 = np.uint64(2**63)


def _stock_calc_metrics() -> tp.Callable[..., tp.Dict[str, float]]:
    """The stock `calc_metrics`, also while `install(metrics=True)` has rebound the module attribute."""
    from rectools.metrics import scoring

    from .integration import _METRICS_KEY, _ORIGINALS

    orig = _ORIGINALS.get(_METRICS_KEY)
    return orig["rectools.metrics.scoring"] if orig is not None else scoring.calc_metrics


def device_metrics(inter_users: np.ndarray, inter_items: np.ndarray, reco_users: np.ndarray, reco_items: np.ndarray,
                   reco_ranks: np.ndarray, ks: tp.Sequence[int], ndcg_tables: tp.Sequence[np.ndarray], want_map: bool,
                   device: int = 0, stats: tp.Optional[tp.Dict[str, tp.Any]] = None) -> tp.Dict[str, tp.Any]:
    """One `b200_rank_metrics` call on int64 columns (see include/b200_rank.h).  Returns a dict with `flags` and, when no
    flag is set, per test user in ascending id: `users`, `first_order` (positions of the users in first-appearance
    order), `liked`, `min_rank` (0: no hit), `tp` [n_k, U], `map` [n_k, U] (None without `want_map`) and `ndcg`
    [n_tables, U].  Raises MemoryError when the device refuses an allocation."""
    n = len(inter_users)
    m = len(reco_users)
    ks_a = np.ascontiguousarray(ks, dtype=np.int64)
    n_k, n_t = len(ks_a), len(ndcg_tables)
    t_off = np.zeros(n_t + 1, dtype=np.int64)
    t_off[1:] = np.cumsum([len(t) for t in ndcg_tables])
    terms = np.ascontiguousarray(np.concatenate(ndcg_tables) if n_t else np.zeros(0), dtype=np.float64)
    users = np.empty(n, np.int64)
    first = np.empty(n, np.int64)
    liked = np.empty(n, np.int64)
    min_rank = np.empty(n, np.int64)
    tp_ = np.empty((n_k, n), np.int64)
    map_ = np.empty((n_k, n), np.float64) if want_map else None
    ndcg = np.empty((n_t, n), np.float64)
    n_users = C.c_int64(0)
    flags = C.c_int32(0)
    ptr = lambda a: None if a is None or a.size == 0 else a.ctypes.data  # noqa: E731
    st = _lib.Stats()
    _lib.check(_lib.load().b200_rank_metrics(
        int(device), None, n, ptr(inter_users), ptr(inter_items), m, ptr(reco_users), ptr(reco_items), ptr(reco_ranks),
        n_k, ptr(ks_a), n_t, t_off.ctypes.data, ptr(terms), C.byref(n_users), ptr(users), ptr(first), ptr(liked),
        ptr(min_rank), ptr(tp_), ptr(map_), ptr(ndcg), C.byref(flags), C.byref(st),
    ))
    if stats is not None:
        stats.update(st.as_dict())
    U = n_users.value
    return {
        "flags": flags.value, "users": users[:U], "first_order": first[:U], "liked": liked[:U], "min_rank": min_rank[:U],
        "tp": tp_[:, :U], "map": None if map_ is None else map_[:, :U], "ndcg": ndcg[:, :U],
    }


def _int_k(k: tp.Any) -> bool:
    return isinstance(k, (int, np.integer)) and not isinstance(k, (bool, np.bool_)) and k >= 1


def _served_families(metrics: tp.Mapping[str, tp.Any]) -> tp.Optional[tp.Tuple[tp.Dict[str, tp.Any], tp.Dict[str, tp.Any]]]:
    """(classification, ranking) sub-dicts in dict order when every metric of the two families is served, else None."""
    from rectools.metrics import MAP, MCC, MRR, NDCG, Accuracy, F1Beta, HitRate, Precision, Recall
    from rectools.metrics.classification import ClassificationMetric, SimpleClassificationMetric

    classification, ranking = {}, {}
    for name, m in metrics.items():
        if isinstance(m, (ClassificationMetric, SimpleClassificationMetric)):
            family, served = classification, (Precision, Recall, F1Beta, HitRate, Accuracy, MCC)
        elif isinstance(m, (NDCG, MAP, MRR)):
            family, served = ranking, (NDCG, MAP, MRR)
        else:
            continue
        if type(m) not in served or getattr(m, "debias_config", None) is not None or not _int_k(m.k):
            return None
        if type(m) is NDCG:
            base = m.log_base
            if isinstance(base, (bool, np.bool_)) or not isinstance(base, (int, float, np.integer, np.floating)):
                return None
            if not (np.isfinite(base) and base > 1):
                return None
        family[name] = m
    return classification, ranking


def _id_column(df: pd.DataFrame, name: str) -> tp.Optional[np.ndarray]:
    """The column as a numpy integer array (a view where possible), or None when it cannot be served."""
    import pandas as pd

    if name not in df.columns:
        return None
    col = df[name]
    if not isinstance(col, pd.Series) or not isinstance(col.dtype, np.dtype) or col.dtype.kind not in "iu":
        return None
    a = col.to_numpy()
    if a.dtype == np.uint64 and len(a) and a.max() >= _U63:
        return None
    return a


def ranking_per_user(m: tp.Any, out: tp.Dict[str, tp.Any], tables: tp.Sequence[np.ndarray],
                     specs: tp.Mapping[tp.Tuple[int, tp.Any, bool], int], k_index: tp.Mapping[int, int]) -> np.ndarray:
    """The per-user values of an NDCG / MRR / MAP metric from the device outputs, float64 in the order in which stock
    averages them: first appearance in the interactions for NDCG and MRR (`groupby(sort=False)`), ascending user id for
    MAP (`np.unique`)."""
    from rectools.metrics import MAP, NDCG

    k = int(m.k)
    liked, first_order = out["liked"], out["first_order"]
    if type(m) is NDCG:
        spec = specs[(k, m.log_base, bool(m.divide_by_achievable))]
        dcg = out["ndcg"][spec]
        if m.divide_by_achievable:  # the user's DCG over the ideal one of min(LIKED, k) hits, as stock maps it
            dcg = dcg / tables[spec].cumsum()[np.minimum(liked, k) - 1]
        return dcg[first_order]
    if type(m) is MAP:
        sums = out["map"][k_index[k]]
        return sums / m.k if m.divide_by_k else sums / liked
    r = out["min_rank"]  # MRR: 1 / the smallest hit rank <= k, 0 without one
    hit = (r >= 1) & (r <= k)
    values = np.zeros(len(r), dtype=np.float64)
    values[hit] = 1.0 / r[hit].astype(np.float64)
    return values[first_order]


def ndcg_tables(ranking: tp.Mapping[str, tp.Any]) -> tp.Tuple[tp.List[np.ndarray], tp.Dict[tp.Tuple[int, tp.Any, bool], int]]:
    """The term table of each distinct (k, log_base, divide_by_achievable) of the NDCG metrics, and its index: the term of
    rank r <= k is `1 / log_at_base(r + 1, log_base)`, over the ideal DCG `discounted_gains.sum()` unless
    divide_by_achievable, by the numpy calls of `NDCG.calc_per_user_from_merged`."""
    from rectools.metrics import NDCG
    from rectools.utils import log_at_base

    specs: tp.Dict[tp.Tuple[int, tp.Any, bool], int] = {}
    tables = []
    for m in ranking.values():
        if type(m) is NDCG:
            key = (int(m.k), m.log_base, bool(m.divide_by_achievable))
            if key not in specs:
                dg = 1 / log_at_base(np.arange(1, key[0] + 1) + 1, m.log_base)
                specs[key] = len(tables)
                tables.append(dg if key[2] else dg / dg.sum())
    return tables, specs


def confusion_df(users: np.ndarray, liked: np.ndarray, tp_k: np.ndarray, k: int) -> pd.DataFrame:
    """`calc_confusions(merged, k)`: int64 LIKED / TP / FP / FN per test user, indexed by the user id."""
    import pandas as pd
    from rectools import Columns
    from rectools.metrics.classification import FN, FP, LIKED, TP

    return pd.DataFrame({LIKED: liked, TP: tp_k, FP: k - tp_k, FN: liked - tp_k}, index=pd.Index(users, name=Columns.User))


def calc_metrics(metrics: tp.Mapping[str, tp.Any], reco: pd.DataFrame, interactions: tp.Optional[pd.DataFrame] = None,
                 prev_interactions: tp.Optional[pd.DataFrame] = None, catalog: tp.Any = None, ref_reco: tp.Any = None,
                 device: int = 0, stats: tp.Optional[tp.Dict[str, tp.Any]] = None) -> tp.Dict[str, float]:
    """`rectools.metrics.calc_metrics` with the classification and ranking metrics computed on `device`; see the module
    docstring.  Returns exactly what the stock function returns.  `stats` (not in the reference): a dict that receives
    the device call's `b200_rank_stats` and the host times `ms_extract` (column checks and int64 copies, NDCG tables)
    and `ms_assemble` (confusion tables, per-user values and means)."""
    import pandas as pd
    from rectools import Columns
    from rectools.metrics import MAP, MCC, MRR, NDCG, Accuracy
    from rectools.metrics.classification import SimpleClassificationMetric

    stock = _stock_calc_metrics()
    args = (reco, interactions, prev_interactions, catalog, ref_reco)
    families = _served_families(metrics)
    if families is None or not (families[0] or families[1]) or interactions is None:
        return stock(metrics, *args)
    classification, ranking = families
    if catalog is None and any(type(m) in (Accuracy, MCC) for m in classification.values()):
        return stock(metrics, *args)
    t0 = time.perf_counter()
    cols = [_id_column(interactions, Columns.User), _id_column(interactions, Columns.Item), _id_column(reco, Columns.User),
            _id_column(reco, Columns.Item), _id_column(reco, Columns.Rank)]
    if any(c is None for c in cols) or len(cols[0]) == 0:
        return stock(metrics, *args)
    for a, b in ((cols[0], cols[2]), (cols[1], cols[3])):
        if np.result_type(a.dtype, b.dtype).kind not in "iu":
            return stock(metrics, *args)
    iu, ii, ru, ri, rr = (np.ascontiguousarray(c, dtype=np.int64) for c in cols)
    ks = sorted({int(m.k) for m in classification.values()} | {int(m.k) for m in ranking.values() if type(m) is MAP})
    k_index = {k: q for q, k in enumerate(ks)}
    tables, specs = ndcg_tables(ranking)
    want_map = any(type(m) is MAP for m in ranking.values())
    t1 = time.perf_counter()
    try:
        out = device_metrics(iu, ii, ru, ri, rr, ks, tables, want_map, device=device, stats=stats)
    except MemoryError as e:
        warnings.warn(f"calc_metrics: the device refused an allocation, the stock function computes the call ({e})", RuntimeWarning)
        return stock(metrics, *args)
    if out["flags"]:
        return stock(metrics, *args)
    t2 = time.perf_counter()

    users = out["users"].astype(cols[0].dtype)
    results: tp.Dict[str, tp.Any] = {}
    confusions: tp.Dict[int, pd.DataFrame] = {}
    for name, m in classification.items():
        k = int(m.k)
        if k not in confusions:
            confusions[k] = confusion_df(users, out["liked"], out["tp"][k_index[k]], k)
        if isinstance(m, SimpleClassificationMetric):
            results[name] = m.calc_from_confusion_df(confusions[k], is_debiased=False)
        else:
            results[name] = m.calc_from_confusion_df(confusions[k], catalog, is_debiased=False)
    for cls in (NDCG, MRR, MAP):  # stock's order inside the ranking family
        for name, m in ranking.items():
            if type(m) is cls:
                results[name] = pd.Series(ranking_per_user(m, out, tables, specs, k_index)).mean()
    results = {k: v.item() if hasattr(v, "item") else v for k, v in results.items()}
    if stats is not None:
        stats["ms_extract"] = 1e3 * (t1 - t0)
        stats["ms_assemble"] = 1e3 * (time.perf_counter() - t2)
    rest = {name: m for name, m in metrics.items() if name not in classification and name not in ranking}
    if rest:
        results.update(stock(rest, *args))
    return results

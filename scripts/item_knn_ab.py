"""ItemKNN (path 9 u2i, path 6 i2i): `ImplicitItemKNNWrapperModel._recommend_u2i` / `_recommend_i2i` stock against
`install(item_knn=True)`, for DESIGN section 3.12.

    python scripts/item_knn_ab.py [--users 100000] [--items 20000] [--K 100] [--per-user 20] [--repeats 3] [--out results.json]

Workload: a K-neighbour S with random fp64 values injected into an `ItemItemRecommender` on the `implicit` stub (its
`recommend` is the numpy definition of tests/knn_oracle.py, so the stock arm times the reference's per-user loop around a
numpy scorer, not implicit's C++), users with ~`per_user` weighted interactions, k = 10, filter_viewed.  Arms, each a
median with [min, max] over repeats:
  stock    the reference's method on a subsample of users, scaled to all users (labelled as such);
  rebound  the same method after `install(item_knn=True)`;
  kernel   the export's CUDA-event times (`ms_h2d`, `ms_main`, `ms_select`, `ms_d2h`, `ms_total`) of one call.
The rebound u2i triplet on the subsample equals the stock one, or the script fails.  The card's name and power limit are
printed first and stored with the result.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
from scipy import sparse

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def _card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return {"card": name, "power_limit": power}


def _stat(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=100_000)
    ap.add_argument("--items", type=int, default=20_000)
    ap.add_argument("--K", type=int, default=100)
    ap.add_argument("--per-user", type=int, default=20)
    ap.add_argument("--stock-users", type=int, default=2_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("item_knn_ab.py needs a CUDA device")
    card = _card()
    print(json.dumps(card))
    from oracle import stage_reference
    from tests import knn_oracle

    stage_reference.add_to_path()
    import pandas as pd
    from implicit.nearest_neighbours import ItemItemRecommender
    from rectools.dataset import Dataset, IdMap, Interactions
    from rectools.models import ImplicitItemKNNWrapperModel

    import rectools_b200 as rb
    from rectools_b200 import item_knn

    rng = np.random.default_rng(0)
    n_users, n_items, K = a.users, a.items, a.K
    per = rng.integers(1, 2 * a.per_user, size=n_users)
    users = np.repeat(np.arange(n_users), per)
    items = rng.integers(0, n_items, size=len(users))
    df = pd.DataFrame({"user_id": users, "item_id": items, "weight": rng.choice([1.0, 2.0, 3.0], size=len(users)),
                       "datetime": np.datetime64("2024-01-01", "ns")}).drop_duplicates(["user_id", "item_id"])
    ds = Dataset(IdMap(np.arange(n_users)), IdMap(np.arange(n_items)), Interactions(df))
    cols = rng.integers(0, n_items, size=(n_items, K))
    cols[:, 0] = np.arange(n_items)
    S = sparse.csr_matrix((rng.standard_normal(n_items * K), (np.repeat(np.arange(n_items), K), cols.reshape(-1))), shape=(n_items, n_items))
    S.sum_duplicates()
    model = ImplicitItemKNNWrapperModel(model=ItemItemRecommender(K=K))
    model.is_fitted = True
    model.model = ItemItemRecommender(K=K)
    model.model.similarity = S
    uids = np.arange(n_users)
    sub = np.sort(rng.choice(n_users, size=min(a.stock_users, n_users), replace=False))
    k = 10
    result = dict(card, users=n_users, items=n_items, K=K, k=k, nnz_users=int(len(df)))
    with knn_oracle.stub_methods():
        stock_t, stock_i2i_t = [], []
        for _ in range(a.repeats):
            t0 = time.perf_counter()
            stock = model._recommend_u2i(sub, ds, k, True, None)  # pylint: disable=protected-access
            stock_t.append((time.perf_counter() - t0) * n_users / len(sub))
            t0 = time.perf_counter()
            model._recommend_i2i(np.arange(n_items), ds, k, None)  # pylint: disable=protected-access
            stock_i2i_t.append(time.perf_counter() - t0)
        rb.install(item_knn=True, fast_recommend=False)
        try:
            check = model._recommend_u2i(sub, ds, k, True, None)  # pylint: disable=protected-access
            for x, y in zip(stock, check):
                np.testing.assert_array_equal(np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64))
            reb_t, reb_i2i_t, stats = [], [], {}
            model._recommend_u2i(uids, ds, k, True, None)  # pylint: disable=protected-access  (warm-up)
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                model._recommend_u2i(uids, ds, k, True, None)  # pylint: disable=protected-access
                reb_t.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                model._recommend_i2i(np.arange(n_items), ds, k, None)  # pylint: disable=protected-access
                reb_i2i_t.append(time.perf_counter() - t0)
            rows = ds.get_user_item_matrix(include_weights=True)
            item_knn.rank_knn(S, rows, k, rows, stats=stats)
        finally:
            rb.uninstall()
    result.update({
        "u2i_stock_s (scaled from %d users)" % len(sub): _stat(stock_t),
        "u2i_rebound_s": _stat(reb_t),
        "i2i_stock_s": _stat(stock_i2i_t),
        "i2i_rebound_s": _stat(reb_i2i_t),
        "kernel": {key: stats[key] for key in ("ms_h2d", "ms_main", "ms_select", "ms_d2h", "ms_total", "n_chunks", "n_launches")},
    })
    print(json.dumps(result, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

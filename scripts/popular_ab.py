"""Popularity lists (path 7): `PopularModel` and `PopularInCategoryModel` stock against `install(popular=True)`, for
DESIGN section 3.10.

    python scripts/popular_ab.py [--repeats 3] [--out results.json] [--small] [--parts popular,category]

Workloads: 10^5 and 10^6 users x 10^5 items, 100 distinct viewed items per user (`n_interactions` popularity), k = 10 and
100; `PopularInCategoryModel` (5 categories, rotate / proportional) at 10^5 users.  Arms, each a median with [min, max]:
  stock      the reference's method.  At 10^6 users it runs on a subsample of users, and the full-size figure is
             extrapolated: the viewed-CSR rebuild (timed on its own, a fixed cost of every call) plus the rest scaled by
             users -- labelled as such;
  rebound    the same method after `install(popular=True)` (its first call builds and caches the viewed CSR; the timed
             calls reuse it, as repeated calls on one dataset do);
  kernel     the export's CUDA-event time of the selection (`ms_main`) and of the whole call (`ms_total`, copies included).
Every timed stock call is compared with the rebound call on the same users: equal triplets / `assert_frame_equal`, or the
script fails.  The card's name and power limit are printed first and stored with every row.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

N_ITEMS, PER_USER = 100_000, 100
SUB_USERS = 50_000  # users the stock method is timed on at 10^6 users


def _dataset(n_users, n_items, per_user, seed, categories=False):
    """Internal ids equal external ids; user u views `per_user` distinct items starting at a skewed offset with a stride
    coprime to the catalogue, so a few thousand items are popular with many users."""
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset, IdMap, Interactions

    rng = np.random.default_rng(seed)
    start = (rng.pareto(1.2, n_users) * 200).astype(np.int64) % n_items
    stride = rng.choice(np.array([1, 3, 7, 11, 13, 17, 19, 23]), n_users)
    items = (start[:, None] + stride[:, None] * np.arange(per_user)[None, :]) % n_items
    n = n_users * per_user
    df = pd.DataFrame({
        Columns.User: np.repeat(np.arange(n_users, dtype=np.int64), per_user),
        Columns.Item: items.reshape(-1),
        Columns.Weight: np.ones(n),
        Columns.Datetime: np.full(n, np.datetime64("2024-01-01", "ns")),
    })
    if not categories:
        return Dataset(IdMap(np.arange(n_users)), IdMap(np.arange(n_items)), Interactions(df))
    features = pd.DataFrame({"id": np.arange(n_items), "feature": "category", "value": [f"c{i % 5}" for i in range(n_items)]})
    return Dataset.construct(df, item_features_df=features, cat_item_features=["category"])


def _stat(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def _timed(fn, repeats):
    out, t = None, []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        t.append(time.perf_counter() - t0)
    return out, _stat(t)


def _same_triplet(a, b, what):
    for x, y in zip(a, b):
        if not np.array_equal(np.asarray(x), np.asarray(y)):
            raise SystemExit(f"rebound and stock triplets differ: {what}")


def main() -> None:  # pylint: disable=too-many-locals,too-many-statements
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    ap.add_argument("--small", action="store_true", help="tiny workloads (a rehearsal of the script)")
    ap.add_argument("--parts", default="popular,category", help="PopularModel shapes, the PopularInCategoryModel one, or both")
    args = ap.parse_args()
    parts = args.parts.split(",")

    import pandas as pd
    import torch

    import rectools_b200 as rb
    from oracle import stage_reference
    from rectools_b200.popular import popular_recommend_u2i

    stage_reference.add_to_path()
    from rectools.models import PopularInCategoryModel, PopularModel

    props = torch.cuda.get_device_properties(0)
    header = {"gpu": props.name}
    try:
        import subprocess

        header["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # pylint: disable=broad-except
        header["power_limit"] = "unknown"
    print(json.dumps(header), flush=True)
    n_items, per_user, sub_users = (2000, 20, 300) if args.small else (N_ITEMS, PER_USER, SUB_USERS)
    user_counts = (1000, 5000) if args.small else (100_000, 1_000_000)
    stock_u2i = PopularModel._recommend_u2i  # pylint: disable=protected-access
    results = []

    for n_users in user_counts if "popular" in parts else ():
        ds = _dataset(n_users, n_items, per_user, seed=n_users)
        model = PopularModel(popularity="n_interactions").fit(ds)
        all_users = np.arange(n_users, dtype=np.int64)
        sub = all_users if n_users <= user_counts[0] else all_users[:: n_users // sub_users][:sub_users]
        _, csr_s = _timed(lambda: ds.get_user_item_matrix(include_weights=False), args.repeats)
        popular_recommend_u2i(model, all_users, ds, 10, True, None)  # builds the cached CSR, warms the kernel
        for k in (10, 100):
            row = {**header, "model": "PopularModel", "n_users": n_users, "n_items": n_items, "per_user": per_user, "k": k}
            scale = n_users / len(sub)
            # _recommend_u2i
            stock, t = _timed(lambda: stock_u2i(model, sub, ds, k, True, None), 1 if scale > 1 else args.repeats)
            st = {}
            got, t_new = _timed(lambda: popular_recommend_u2i(model, all_users, ds, k, True, None, stats=st), args.repeats)
            if scale > 1:
                _same_triplet(stock, popular_recommend_u2i(model, sub, ds, k, True, None), f"{row} subsample")
            else:
                _same_triplet(stock, got, str(row))
            row["stock_u2i_s" if scale == 1 else "stock_u2i_s_subsample"] = t
            if scale > 1:
                row["stock_u2i_subsample_users"] = int(len(sub))
                row["stock_u2i_s_extrapolated"] = csr_s["median"] + (t["median"] - csr_s["median"]) * scale
            row["viewed_csr_rebuild_s"] = csr_s
            row["rebound_u2i_s"] = t_new
            row["kernel_ms_main"] = st["ms_main"]
            row["export_ms_total"] = st["ms_total"]
            row["export_n_chunks"] = st["n_chunks"]
            # model.recommend
            users_ext = ds.user_id_map.external_ids
            sub_ext = users_ext[sub]
            stock_df, t = _timed(lambda: model.recommend(sub_ext, ds, k, True), 1 if scale > 1 else args.repeats)
            rb.install(popular=True)
            try:
                got_df, t_new = _timed(lambda: model.recommend(users_ext, ds, k, True), args.repeats)
                check = got_df if scale == 1 else model.recommend(sub_ext, ds, k, True)
            finally:
                rb.uninstall()
            pd.testing.assert_frame_equal(check, stock_df)
            row["stock_recommend_s" if scale == 1 else "stock_recommend_s_subsample"] = t
            if scale > 1:
                row["stock_recommend_s_extrapolated"] = csr_s["median"] + (t["median"] - csr_s["median"]) * scale
            row["rebound_recommend_s"] = t_new
            print(json.dumps(row), flush=True)
            results.append(row)
        del ds, model

    # PopularInCategoryModel: one dataset, 5 categories
    if "category" not in parts:
        user_counts = ()
    n_users = user_counts[0] if user_counts else 0
    if n_users:
        ds = _dataset(n_users, n_items, per_user, seed=7, categories=True)
        model = PopularInCategoryModel(category_feature="category", n_categories=5, popularity="n_interactions").fit(ds)
        users_ext = ds.user_id_map.external_ids
    for k in (10, 100) if n_users else ():
        row = {**header, "model": "PopularInCategoryModel", "n_categories": 5, "n_users": n_users, "n_items": n_items,
               "per_user": per_user, "k": k}
        stock_df, t = _timed(lambda: model.recommend(users_ext, ds, k, True), args.repeats)
        rb.install(popular=True)
        try:
            model.recommend(users_ext[:10], ds, k, True)  # builds the cached CSR
            got_df, t_new = _timed(lambda: model.recommend(users_ext, ds, k, True), args.repeats)
        finally:
            rb.uninstall()
        pd.testing.assert_frame_equal(got_df, stock_df)
        row["stock_recommend_s"] = t
        row["rebound_recommend_s"] = t_new
        print(json.dumps(row), flush=True)
        results.append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"header": header, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()

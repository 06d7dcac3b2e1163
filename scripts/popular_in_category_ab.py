"""Per-category lists mixed (path 8): `PopularInCategoryModel` stock, under `install(popular=True)`, and under
`install(popular=True, popular_in_category=True)`, for DESIGN section 3.11.

    python scripts/popular_in_category_ab.py [--users 100000] [--categories 5,50] [--ks 10,100] [--sub 0]
                                             [--repeats 5] [--base-repeats 2] [--out results.json] [--small]

Workload: 10^5 items, each in 1 to 3 of `--categories` categories, 100 distinct viewed items per user (`n_users`
popularity, rotate / proportional), k in `--ks`.  The model is fitted on the first min(users, 10^5) users'
interactions (the "fit" dataset, whose users are the first users of the full one).  Arms, each a median with [min, max]:
  stock        the reference's methods;
  popular      after `install(popular=True)` (each category's list on the GPU, the mixing in pandas);
  in_category  after `install(popular=True, popular_in_category=True)` (lists and mixing in one kernel pass), timed on
               the fit dataset and on the full one (`--repeats` each);
  kernel       the export's CUDA-event time of the mixing kernels (`ms_main`) and of the whole call (`ms_total`).
`_recommend_u2i` and `recommend()` are timed.  `--sub 0`: stock and popular are timed on every user of the fit dataset
(`--base-repeats` each).  `--sub n`: they are timed on the first n users of the fit dataset and the full-size figures
are EXTRAPOLATED, and labelled so:
  stock    = its fixed cost (one viewed-CSR rebuild per category, the rebuild timed on its own on the dataset in
             question) + the rest of the subsample time scaled by users;
  popular  = a line through its times at n and 4 n users (its CSR is cached, so its fixed cost is what the line finds;
             stock is timed at n users only).
Every timed stock / popular call is compared with the in_category call on the same users (equal triplets and frames),
and the full-size in_category frame on the first users with the stock frame on them, or the script stops.  The card's
name and power limit are read in the same run and stored with every row.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

N_ITEMS, PER_USER, FIT_USERS = 100_000, 100, 100_000


def _dataset(n_users, n_items, n_categories, seed):
    """Internal ids equal external ids; user u views `PER_USER` distinct items from a skewed offset with a stride coprime
    to the catalogue; item i is in 1 to 3 categories."""
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset, IdMap, Interactions
    from rectools.dataset.features import SparseFeatures

    rng = np.random.default_rng(seed)
    start = (rng.pareto(1.2, n_users) * 200).astype(np.int64) % n_items
    stride = rng.choice(np.array([1, 3, 7, 11, 13, 17, 19, 23]), n_users)
    items = (start[:, None] + stride[:, None] * np.arange(PER_USER)[None, :]) % n_items
    n = n_users * PER_USER
    df = pd.DataFrame({
        Columns.User: np.repeat(np.arange(n_users, dtype=np.int64), PER_USER),
        Columns.Item: items.reshape(-1),
        Columns.Weight: np.ones(n),
        Columns.Datetime: np.full(n, np.datetime64("2024-01-01", "ns")),
    })
    crng = np.random.default_rng(1000 + n_categories)
    n_cat = crng.integers(1, 4, n_items)
    ids = np.repeat(np.arange(n_items), n_cat)
    cats = (crng.integers(0, n_categories, len(ids)) + np.concatenate([np.arange(c) for c in n_cat])) % n_categories
    feats = pd.DataFrame({"id": ids, "feature": "category", "value": [f"c{c}" for c in cats]}).drop_duplicates()
    item_map = IdMap(np.arange(n_items))
    features = SparseFeatures.from_flatten(feats, item_map, cat_features=["category"])
    return Dataset(IdMap(np.arange(n_users)), item_map, Interactions(df), item_features=features)


def _stat(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def _timed(fn, repeats):
    out, times = None, []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t0)
    return out, times


def _same_triplet(a, b, what):
    for x, y in zip(a, b):
        if not np.array_equal(np.asarray(x), np.asarray(y)):
            raise SystemExit(f"{what}: triplets differ")


def _head(ds, n):
    """The dataset of the first n users of `ds` (same items and features)."""
    from rectools import Columns
    from rectools.dataset import Dataset, IdMap, Interactions

    df = ds.interactions.df
    return Dataset(IdMap(np.arange(n)), ds.item_id_map, Interactions(df[df[Columns.User] < n]), item_features=ds.item_features)


def main() -> None:  # pylint: disable=too-many-locals,too-many-statements
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=100_000)
    ap.add_argument("--categories", default="5,50")
    ap.add_argument("--ks", default="10,100")
    ap.add_argument("--sub", type=int, default=0, help="0: time stock and popular on every fit user; n: on n (and 4 n)")
    ap.add_argument("--repeats", type=int, default=5, help="timed calls of the in_category arm")
    ap.add_argument("--base-repeats", type=int, default=2, help="timed calls of the stock and popular arms")
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    ap.add_argument("--small", action="store_true", help="tiny workloads (a rehearsal of the script)")
    args = ap.parse_args()
    import pandas as pd

    from oracle import stage_reference

    stage_reference.add_to_path()
    import rectools_b200 as rb
    from rectools.models import PopularInCategoryModel
    from rectools_b200.popular import popular_in_category_recommend_u2i

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True, check=True).stdout.strip().splitlines()[0]
    print(f"GPU: {gpu}")
    n_items, n_users, fit_users, sub = N_ITEMS, args.users, min(FIT_USERS, args.users), args.sub
    if args.small:
        n_items, n_users, fit_users, sub = 2000, 6000, 3000, (100 if args.sub else 0)
    rows = []
    for n_categories in [int(x) for x in args.categories.split(",")]:
        t0 = time.perf_counter()
        ds = _dataset(n_users, n_items, n_categories, seed=0)
        fit_ds = ds if n_users == fit_users else _head(ds, fit_users)
        model = PopularInCategoryModel(category_feature="category")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model.fit(fit_ds)
        rebuild = {name: _stat(_timed(lambda d=d: d.get_user_item_matrix(include_weights=False), 2)[1])["median"]
                   for name, d in (("fit", fit_ds), ("full", ds))}
        print(f"{n_categories} categories: data and fit {time.perf_counter() - t0:.1f} s, viewed-CSR rebuild "
              f"{rebuild['fit']:.2f} s ({fit_users} users) / {rebuild['full']:.2f} s ({n_users} users)")
        base_sizes = [fit_users] if sub == 0 else [sub, 4 * sub]
        for k in [int(x) for x in args.ks.split(",")]:
            res = {"viewed_csr_rebuild_s": rebuild}

            def arm(kw, users, dataset, repeats):
                if kw:
                    rb.install(**kw)
                try:
                    model._recommend_u2i(users[:10], dataset, k, True, None)  # warm-up: viewed CSR, module load
                    trip, t_u2i = _timed(lambda: model._recommend_u2i(users, dataset, k, True, None), repeats)
                    frame, t_rec = _timed(lambda: model.recommend(users, dataset, k, True), repeats)
                finally:
                    rb.uninstall()
                return trip, frame, {"users": len(users), "u2i_s": _stat(t_u2i), "recommend_s": _stat(t_rec)}

            mixed = {"popular": True, "popular_in_category": True}
            checked = None  # the in_category frame on the first base size, equal to stock's
            for n in base_sizes:
                users = np.arange(n)
                ref_trip, ref_frame, res[f"in_category_{n}"] = arm(mixed, users, fit_ds, args.repeats)
                checked = ref_frame if checked is None else checked
                stock = (("stock", None),) if n == base_sizes[0] else ()  # (its fixed cost is timed on its own)
                for name, kw in stock + (("popular", {"popular": True}),):
                    trip, frame, res[f"{name}_{n}"] = arm(kw, users, fit_ds, args.base_repeats)
                    _same_triplet(trip, ref_trip, f"{name} u2i, {n_categories} categories, k={k}, {n} users")
                    pd.testing.assert_frame_equal(frame, ref_frame)
            st = {}
            popular_in_category_recommend_u2i(model, np.arange(n_users), ds, k, True, None, stats=st)
            res["kernel"] = {"users": n_users, "ms_main": st["ms_main"], "ms_total": st["ms_total"]}
            first = base_sizes[0]
            if n_users != fit_users:
                _, full, res["in_category_full"] = arm(mixed, np.arange(n_users), ds, args.repeats)
                part = full[full["user_id"] < first].reset_index(drop=True)
                pd.testing.assert_frame_equal(part, checked)
            else:
                res["in_category_full"] = res[f"in_category_{fit_users}"]
            for n_to, name in ((fit_users, "fit"), (n_users, "full")):
                if sub == 0:  # measured directly on the fit users; no extrapolation
                    continue
                for what in ("u2i_s", "recommend_s"):
                    t = res[f"stock_{first}"][what]["median"]
                    fixed = n_categories * rebuild["fit"]
                    res.setdefault(f"stock_extrapolated_{name}", {"users": n_to})[what] = \
                        n_categories * rebuild[name] + (t - fixed) * n_to / first
                    t1, t4 = res[f"popular_{sub}"][what]["median"], res[f"popular_{4 * sub}"][what]["median"]
                    slope = (t4 - t1) / (3 * sub)
                    res.setdefault(f"popular_extrapolated_{name}", {"users": n_to})[what] = t1 + slope * (n_to - sub)
            row = {"gpu": gpu, "n_items": n_items, "n_users": n_users, "fit_users": fit_users, "n_categories": n_categories,
                   "k": k, **res}
            rows.append(row)
            print(json.dumps(row))
            if args.out:
                with open(args.out, "w") as f:
                    json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()

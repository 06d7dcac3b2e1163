"""Datasets and model settings of the `PopularInCategoryModel` tests of path 8 (CPU and GPU).  Needs the reference package
on sys.path (`oracle.stage_reference.add_to_path()`)."""
import itertools

import numpy as np


def category_dataset(n_users=60, n_items=40, n_categories=5, per_user=8, seed=0, heavy_users=2, idle_users=0):
    """`Dataset` with weights, datetimes over 30 days and a categorical item feature `category` with `n_categories`
    values, each item in 1 to 3 of them (so the category lists overlap and the mixing drops repeats).  The first
    `heavy_users` users view every item with interactions; the others about `per_user`; the last three items have no
    interaction (cold items for `add_cold`).  `idle_users` more users come first in the id map, with nothing viewed."""
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset

    rng = np.random.default_rng(seed)
    popular_items = n_items - 3
    users, items = [], []
    for u in range(n_users):
        if u < heavy_users:
            seen = np.arange(popular_items)
        else:
            seen = rng.choice(popular_items, size=min(popular_items, int(rng.integers(1, per_user * 2))), replace=False)
        users.append(np.full(len(seen), u))
        items.append(seen)
    users, items = np.concatenate(users), np.concatenate(items)
    df = pd.DataFrame({
        Columns.User: users * 7 + 1000,
        Columns.Item: items * 3 + 5,
        Columns.Weight: rng.integers(1, 6, len(users)).astype(np.float64),
        Columns.Datetime: pd.Timestamp("2024-01-01") + pd.to_timedelta(rng.integers(0, 30, len(users)), unit="D"),
    })
    ids, values = [], []
    for i in range(n_items):
        n_cat = int(rng.integers(1, min(3, n_categories) + 1))
        for c in rng.choice(n_categories, size=n_cat, replace=False):
            ids.append(i * 3 + 5)
            values.append(f"c{c}")
    features = pd.DataFrame({"id": ids, "feature": "category", "value": values})
    ds = Dataset.construct(df, item_features_df=features, cat_item_features=["category"])
    if idle_users:  # internal ids 0 .. idle_users - 1, below the users with interactions: hot rows with nothing viewed
        from rectools.dataset import IdMap, Interactions

        inter = ds.interactions.df.copy()
        inter[Columns.User] += idle_users
        user_map = IdMap.from_values(np.concatenate((np.arange(idle_users) + 10**6, ds.user_id_map.external_ids)))
        ds = Dataset(user_map, ds.item_id_map, Interactions(inter), item_features=ds.item_features)
    return ds


def in_category_settings(n_categories):
    """PopularInCategoryModel keyword sets for a dataset of `n_categories` categories: both mixings x both ratio
    strategies, `n_categories` unset, below and above the category count, and every `Popularity` kind with `add_cold` /
    `inverse`."""
    for mixing, ratio, n_cat in itertools.product(("rotate", "group"), ("proportional", "equal"),
                                                  (None, max(1, n_categories // 2), n_categories + 3)):
        yield dict(category_feature="category", n_categories=n_cat, mixing_strategy=mixing, ratio_strategy=ratio)
    for popularity, add_cold, inverse in (("n_interactions", True, False), ("mean_weight", False, True),
                                          ("sum_weight", True, True), ("n_users", False, False)):
        yield dict(category_feature="category", popularity=popularity, add_cold=add_cold, inverse=inverse,
                   mixing_strategy="group" if inverse else "rotate", ratio_strategy="equal" if add_cold else "proportional")

"""Datasets and model settings of the `PopularModel` / `PopularInCategoryModel` tests (CPU and GPU).  Needs the reference
package on sys.path (`oracle.stage_reference.add_to_path()`)."""
import itertools
from datetime import timedelta

import numpy as np

N_CATEGORIES = 5


def popular_dataset(n_users=60, n_items=40, per_user=8, seed=0, heavy_users=2):
    """`Dataset` with weights, datetimes over 30 days and a categorical item feature `category` (5 values).  The first
    `heavy_users` users view every item; the others about `per_user` (some items are viewed by nobody, so `add_cold`
    has cold items to add)."""
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset

    rng = np.random.default_rng(seed)
    popular_items = n_items - 3  # the last three items have no interaction
    users, items = [], []
    for u in range(n_users):
        seen = np.arange(popular_items) if u < heavy_users else rng.choice(popular_items, size=rng.integers(1, per_user * 2), replace=False)
        users.append(np.full(len(seen), u))
        items.append(seen)
    users, items = np.concatenate(users), np.concatenate(items)
    df = pd.DataFrame({
        Columns.User: users * 7 + 1000,
        Columns.Item: items * 3 + 5,
        Columns.Weight: rng.integers(1, 6, len(users)).astype(np.float64),
        Columns.Datetime: pd.Timestamp("2024-01-01") + pd.to_timedelta(rng.integers(0, 30, len(users)), unit="D"),
    })
    features = pd.DataFrame({
        "id": np.arange(n_items) * 3 + 5,
        "feature": "category",
        "value": [f"c{i % N_CATEGORIES}" for i in rng.permutation(n_items)],
    })
    return Dataset.construct(df, item_features_df=features, cat_item_features=["category"])


def popular_settings():
    """PopularModel keyword sets: every `Popularity` kind, with and without `add_cold`, `inverse` and `period`."""
    for popularity, add_cold, inverse, period in itertools.product(
        ("n_users", "n_interactions", "mean_weight", "sum_weight"), (False, True), (False, True), (None, timedelta(days=10))
    ):
        yield dict(popularity=popularity, add_cold=add_cold, inverse=inverse, period=period)


def category_settings():
    """PopularInCategoryModel keyword sets: both mixing strategies x both ratio strategies."""
    for mixing, ratio in itertools.product(("rotate", "group"), ("proportional", "equal")):
        yield dict(category_feature="category", n_categories=N_CATEGORIES, mixing_strategy=mixing, ratio_strategy=ratio)


def recommend_cases(dataset):
    """(users, k, filter_viewed, items_to_recommend) of the frame comparisons: all hot users, a subset in another order
    with a cold user, k above the catalogue, a whitelist, and calls whose result is empty."""
    ext_users = dataset.user_id_map.external_ids
    ext_items = dataset.item_id_map.external_ids
    heavy = ext_users[:2]
    n_items = len(ext_items)
    for filter_viewed in (True, False):
        yield ext_users, 5, filter_viewed, None
        yield np.concatenate((ext_users[7:2:-1], [999_999])), 3, filter_viewed, None
        yield ext_users[:10], n_items + 5, filter_viewed, None
        yield ext_users, 4, filter_viewed, ext_items[::3]
        # empty: users that viewed every item with interactions, ranked among items they viewed
        yield heavy, 3, filter_viewed, ext_items[:4]

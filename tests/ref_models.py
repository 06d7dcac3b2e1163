"""Builders of UNMODIFIED reference models on synthetic data (shared by the CPU and GPU integration tests and bench.py's
`model_recommend` leg).  Needs the reference package on sys.path (`oracle.stage_reference.add_to_path()`)."""
import numpy as np


def synthetic_dataset(n_users, n_items, per_user, seed=0, external_offset=True):
    """`Dataset` over ~`per_user` distinct interactions per user.  Internal ids are 0..n-1 in order; external ids are shifted
    (users * 7 + 1000, items * 3 + 5) unless `external_offset=False` (pattern: tests/models/test_implicit_als.py:72-90)."""
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset, IdMap, Interactions

    rng = np.random.default_rng(seed)
    users = np.repeat(np.arange(n_users, dtype=np.int64), per_user)
    items = rng.integers(0, n_items, size=n_users * per_user, dtype=np.int64)
    df = pd.DataFrame({Columns.User: users, Columns.Item: items})
    df = df.drop_duplicates([Columns.User, Columns.Item], ignore_index=True)
    df[Columns.Weight] = np.float64(1.0)
    df[Columns.Datetime] = pd.Timestamp("2024-01-01")
    user_ext = np.arange(n_users, dtype=np.int64) * 7 + 1000 if external_offset else np.arange(n_users, dtype=np.int64)
    item_ext = np.arange(n_items, dtype=np.int64) * 3 + 5 if external_offset else np.arange(n_items, dtype=np.int64)
    return Dataset(IdMap(user_ext), IdMap(item_ext), Interactions(df))


def injected_als(user_factors, item_factors):
    """`ImplicitALSWrapperModel` around a pre-"fitted" implicit ALS object carrying the given factors -- the injection of
    the reference's own test (tests/models/test_implicit_als.py:193-197); the stub's `AlternatingLeastSquares` is an
    attribute carrier (oracle/implicit_stub/implicit/cpu/als.py)."""
    from implicit.cpu.als import AlternatingLeastSquares
    from rectools.models import ImplicitALSWrapperModel

    base = AlternatingLeastSquares(factors=user_factors.shape[1], num_threads=0, iterations=1, random_state=0)
    base.user_factors = np.ascontiguousarray(user_factors, dtype=np.float32)
    base.item_factors = np.ascontiguousarray(item_factors, dtype=np.float32)
    wrapped = ImplicitALSWrapperModel(model=base, fit_features_together=False)
    wrapped.is_fitted = True
    wrapped.model = wrapped._model  # pylint: disable=protected-access
    return wrapped


def injected_lightfm(dataset, user_embeddings, item_embeddings, user_biases, item_biases):
    """`LightFMWrapperModel` "fitted" on `dataset` through the `lightfm` stand-in (tests/lightfm_stub, an attribute carrier
    that does no training), then given these arrays: one row per user / item feature column the wrapper builds (the hot
    users / items, then the feature columns when the dataset has features), `no_components` columns."""
    from lightfm import LightFM
    from rectools.models import LightFMWrapperModel

    model = LightFMWrapperModel(model=LightFM(no_components=user_embeddings.shape[1], random_state=0)).fit(dataset)
    for name, arr in (("user_embeddings", user_embeddings), ("item_embeddings", item_embeddings), ("user_biases", user_biases),
                      ("item_biases", item_biases)):
        old = getattr(model.model, name)
        assert old.shape == arr.shape, f"{name}: {arr.shape}, the dataset needs {old.shape}"
        setattr(model.model, name, np.ascontiguousarray(arr, dtype=np.float32))
    return model


def injected_bpr(user_factors, item_factors, item_bias):
    """`ImplicitBPRWrapperModel` around a pre-"fitted" implicit BPR object in implicit's layout: the last user column is 1,
    the last item column is the item bias.  The same injection as `injected_als`."""
    from implicit.cpu.bpr import BayesianPersonalizedRanking
    from rectools.models import ImplicitBPRWrapperModel

    base = BayesianPersonalizedRanking(factors=user_factors.shape[1], num_threads=0, iterations=1, random_state=0)
    base.user_factors = np.ascontiguousarray(np.hstack([user_factors, np.ones((len(user_factors), 1))]), dtype=np.float32)
    base.item_factors = np.ascontiguousarray(np.hstack([item_factors, np.asarray(item_bias).reshape(-1, 1)]), dtype=np.float32)
    wrapped = ImplicitBPRWrapperModel(model=base)
    wrapped.is_fitted = True
    wrapped.model = wrapped._model  # pylint: disable=protected-access
    return wrapped


def featured_dataset(n_users, n_items, per_user, seed=0, n_warm_users=0, n_warm_items=0):
    """`synthetic_dataset`'s interactions with a categorical and a numeric feature for every user (5 groups, "age") and
    item (8 categories, "price": the items of one category differ), plus `n_warm_users` / `n_warm_items` known only from the feature tables (warm targets)."""
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset

    rng = np.random.default_rng(seed)
    inter = synthetic_dataset(n_users, n_items, per_user, seed=seed).get_raw_interactions()
    users = np.arange(n_users + n_warm_users, dtype=np.int64) * 7 + 1000
    items = np.arange(n_items + n_warm_items, dtype=np.int64) * 3 + 5
    uf = pd.concat([pd.DataFrame({"id": users, "feature": "group", "value": rng.integers(0, 5, len(users)).astype(str)}),
                    pd.DataFrame({"id": users, "feature": "age", "value": rng.random(len(users))})], ignore_index=True)
    itf = pd.concat([pd.DataFrame({"id": items, "feature": "category", "value": rng.integers(0, 8, len(items)).astype(str)}),
                     pd.DataFrame({"id": items, "feature": "price", "value": rng.random(len(items))})], ignore_index=True)
    return Dataset.construct(inter[Columns.Interactions], user_features_df=uf, cat_user_features=["group"], item_features_df=itf,
                             cat_item_features=["category"])


def small_dssm(dataset, n_factors=32, seed=0):
    """`DSSMModel` fitted on CPU through the `pytorch_lightning` stand-in (tests/lightning_stub): one epoch over
    `dataset`, which needs user and item features.  Seconds at a few thousand users and items."""
    import torch
    from rectools.models import DSSMModel

    torch.manual_seed(seed)
    model = DSSMModel(n_factors=n_factors, max_epochs=1, batch_size=256, trainer_accelerator="cpu", deterministic=True,
                      loggers=False)
    return model.fit(dataset)

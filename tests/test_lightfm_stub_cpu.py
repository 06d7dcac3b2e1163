"""CPU: the `lightfm` stand-in (tests/lightfm_stub) under the unmodified `LightFMWrapperModel`.

* The wrapper's `get_vectors` (biases folded as two extra columns) ranks as its own `_recommend_u2i` does, user and item
  features included: the check of the reference's `TestLightFMWrapperModel::test_get_vectors`
  (tests/models/test_lightfm.py:248-267), restated on its fixture data.
* The stand-in's shapes, dtypes, seeding and representations against a numpy restatement of lightfm's documented
  `get_*_representations` (`features @ biases`, `features @ embeddings`), and the config the wrapper reads from it."""
import numpy as np
import pytest

from oracle import stage_reference
from tests import lightfm_stub

pytestmark = pytest.mark.skipif(not stage_reference.available(), reason="reference package not available")


@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    stub = lightfm_stub.add_to_path()
    yield
    lightfm_stub.remove_from_path(stub)
    stage_reference.remove_from_path(added)


def _interactions():
    import pandas as pd
    from rectools import Columns

    data = [[10, 11], [10, 12], [10, 13], [10, 14], [20, 11], [20, 12], [20, 15], [30, 11], [30, 12], [30, 13], [30, 15]]
    data += [[40 + i, iid] for i in range(2) for iid in (11, 12, 13)]
    data += [[50 + i, iid] for i in range(4) for iid in (11, 12)]
    data += [[60 + i, 11] for i in range(50)]
    df = pd.DataFrame(data, columns=Columns.UserItem)
    df[Columns.Weight] = 1
    df[Columns.Datetime] = "2021-09-09"
    return df


def _dataset_with_features():
    import pandas as pd
    from rectools.dataset import Dataset

    user_features = pd.DataFrame({"id": [10, 130], "feature": ["f1", "f1"], "value": [2, 2]})
    item_features = pd.DataFrame({"id": [11, 11, 12, 12, 14, 14, 16, 16], "feature": ["f1", "f2"] * 4,
                                  "value": [100, "a", 100, "a", 100, "a", 100, "a"]})
    return Dataset.construct(interactions_df=_interactions(), user_features_df=user_features, item_features_df=item_features,
                             cat_item_features=["f1", "f2"])


@pytest.mark.parametrize("use_gpu_ranking", [True, False])
def test_get_vectors_rank_as_recommend_u2i(ref, use_gpu_ranking):
    from lightfm import LightFM
    from rectools.models import LightFMWrapperModel
    from rectools.models.utils import recommend_from_scores

    ds = _dataset_with_features()
    model = LightFMWrapperModel(model=LightFM(no_components=2, loss="logistic"), recommend_use_gpu_ranking=use_gpu_ranking).fit(ds)
    users, items = model.get_vectors(ds)
    assert users.shape[1] == items.shape[1] == 4
    np.testing.assert_array_equal(users[:, 1], 1.0)
    np.testing.assert_array_equal(items[:, 0], 1.0)
    scores = users @ items.T
    expected = [recommend_from_scores(scores[i], k=5) for i in range(4)]
    _, reco, reco_scores = model._recommend_u2i(  # pylint: disable=protected-access
        user_ids=ds.user_id_map.convert_to_internal(np.array([10, 20, 30, 40])), dataset=ds, k=5, filter_viewed=False,
        sorted_item_ids_to_recommend=None)
    np.testing.assert_equal(np.concatenate([e[0] for e in expected]), reco)
    np.testing.assert_almost_equal(np.concatenate([e[1] for e in expected]), reco_scores, decimal=5)


def test_representations_follow_lightfm(ref):
    from lightfm import LightFM
    from rectools.models import LightFMWrapperModel
    from scipy import sparse

    ds = _dataset_with_features()
    base = LightFM(no_components=3, k=7, n=11, learning_rate=0.1, item_alpha=0.01, user_alpha=0.02, max_sampled=9, random_state=5)
    model = LightFMWrapperModel(model=base, epochs=2).fit(ds)
    inner = model.model
    uf = model._prepare_features(ds.user_features, ds.n_hot_users)  # pylint: disable=protected-access
    itf = model._prepare_features(ds.item_features, ds.n_hot_items)  # pylint: disable=protected-access
    # n_features x no_components, float32, from the feature matrices the wrapper builds (identity columns + features)
    assert inner.user_embeddings.shape == (uf.shape[1], 3) and inner.item_embeddings.shape == (itf.shape[1], 3)
    assert inner.user_biases.shape == (uf.shape[1],) and inner.item_biases.shape == (itf.shape[1],)
    for a in (inner.user_embeddings, inner.item_embeddings, inner.user_biases, inner.item_biases):
        assert a.dtype == np.float32 and np.isfinite(a).all() and np.abs(a).max() > 0
    # seeded: the same seed gives the same arrays, another seed others
    again = LightFMWrapperModel(model=LightFM(no_components=3, random_state=5)).fit(ds).model
    other = LightFMWrapperModel(model=LightFM(no_components=3, random_state=6)).fit(ds).model
    np.testing.assert_array_equal(again.item_embeddings, inner.item_embeddings)
    assert not np.array_equal(other.item_embeddings, inner.item_embeddings)
    # features @ biases, features @ embeddings; the raw arrays without features
    for get, feats, b, e in ((inner.get_user_representations, uf, inner.user_biases, inner.user_embeddings),
                             (inner.get_item_representations, itf, inner.item_biases, inner.item_embeddings)):
        rb, re_ = get(feats)
        dense = sparse.csr_matrix(feats).toarray().astype(np.float64)
        np.testing.assert_allclose(rb, dense @ b.astype(np.float64), rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(re_, dense @ e.astype(np.float64), rtol=1e-6, atol=1e-7)
        raw_b, raw_e = get()
        assert raw_b is b and raw_e is e
    # what the wrapper's factors are made of
    factors = model._get_items_factors(ds)  # pylint: disable=protected-access
    np.testing.assert_array_equal(factors.biases, inner.get_item_representations(itf)[0])
    # without features: one row per user / item
    plain = LightFMWrapperModel(model=LightFM(no_components=4, random_state=1)).fit(ds_plain := _plain_dataset())
    assert plain.model.user_embeddings.shape == (ds_plain.user_id_map.size, 4)
    assert plain.model.item_embeddings.shape == (ds_plain.item_id_map.size, 4)
    # the config the wrapper reads from the stand-in round-trips
    cfg = model.get_config()
    assert cfg["model"]["no_components"] == 3 and cfg["model"]["k"] == 7 and cfg["model"]["max_sampled"] == 9
    assert cfg["model"]["random_state"] == 5 and cfg["epochs"] == 2
    assert LightFMWrapperModel.from_config(cfg).get_config() == cfg


def _plain_dataset():
    from rectools.dataset import Dataset

    return Dataset.construct(_interactions())

"""GPU: `rectools_b200.recommend()` (vectorised `ModelBase.recommend`, SURVEY section 8f rank 1) with the real CUDA ranker on
BASELINE config 1 -- the factors and the recommendations of the reference's `PureSVDModel(factors=32).recommend(K=10,
filter_viewed=True)` on the 6040 x 3706 synthetic interactions (tests/golden/puresvd_c1.npz, made by oracle/make_golden.py).
rectools itself is not on the GPU box: the dataset / model are the duck-typed stand-ins of tests/helpers.py."""
import os

import numpy as np
import pytest
from scipy import sparse

from tests.helpers import FakeDataset, FakeVectorModel, assert_same_ranking

pytestmark = pytest.mark.gpu


def test_recommend_table_matches_reference_golden(rb, golden_dir):
    from rectools_b200.recommend import clear_viewed_cache, recommend

    g = np.load(os.path.join(golden_dir, "puresvd_c1.npz"))
    n_users, n_items = g["user_factors"].shape[0], g["item_factors"].shape[0]
    sids = g["subject_ids"]
    # full user x item matrix: the golden file holds the rows of the ranked users; everybody else has no interactions
    sub = sparse.csr_matrix((np.ones(len(g["csr_indices"]), np.float32), g["csr_indices"], g["csr_indptr"]), shape=tuple(g["csr_shape"]))
    lens = np.zeros(n_users, dtype=np.int64)
    lens[sids] = np.diff(sub.indptr)
    full = sparse.csr_matrix((n_users, n_items), dtype=np.float32)
    full.indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    order = np.argsort(sids, kind="stable")
    full.indices = np.concatenate([sub.indices[sub.indptr[r] : sub.indptr[r + 1]] for r in order]).astype(np.int32)
    full.data = np.ones(len(full.indices), np.float32)
    user_ext = np.arange(n_users, dtype=np.int64) * 2 + 10
    item_ext = np.arange(n_items, dtype=np.int64) * 3 + 7
    dataset = FakeDataset(user_ext, item_ext, full)
    model = FakeVectorModel("dot", g["user_factors"], g["item_factors"])
    clear_viewed_cache()

    for filt, pre in ((True, "out_"), (False, "out_nf_")):
        df = recommend(model, user_ext[sids], dataset, 10, filt)
        assert list(df.columns) == ["user_id", "item_id", "score", "rank"]
        assert df["user_id"].dtype == np.int64 and df["item_id"].dtype == np.int64 and df["score"].dtype == np.float32
        np.testing.assert_array_equal(df["user_id"].to_numpy(), user_ext[g[pre + "subjects"]])
        np.testing.assert_array_equal(df["rank"].to_numpy(), np.tile(np.arange(1, 11), len(sids)))
        assert_same_ranking((df["item_id"].to_numpy() - 7) // 3, df["score"].to_numpy(), g[pre + "ids"], g[pre + "scores"], tie_tol=2e-6, msg=pre)
    # the viewed-items CSR is built once per interactions table, not per call (vector.py:58-60 rebuilds it every time)
    recommend(model, user_ext[sids][:100], dataset, 5, True)
    assert dataset.n_matrix_builds == 1
    # whitelist + all users: ragged rows keep rank = 1..n per user
    wl_ext = item_ext[:6]
    df = recommend(model, user_ext, dataset, 10, True, items_to_recommend=wl_ext)
    assert df.groupby("user_id", sort=False).size().max() <= 6
    assert (df.groupby("user_id", sort=False).cumcount().to_numpy() + 1 == df["rank"].to_numpy()).all()
    assert set(df["item_id"].unique()) <= set(wl_ext.tolist())


def test_recommend_to_items_matches_oracle(rb, golden_dir):
    """SURVEY 8f rank 2: `recommend_to_items` = the same engine with item vectors as subjects (COSINE), k + 1, self removed."""
    from oracle.topk_oracle import rank_oracle
    from rectools_b200.recommend import recommend_to_items

    g = np.load(os.path.join(golden_dir, "puresvd_c1.npz"))
    items = g["item_factors"]
    n_items = items.shape[0]
    item_ext = np.arange(n_items, dtype=np.int64) * 3 + 7
    dataset = FakeDataset(np.arange(4, dtype=np.int64), item_ext, sparse.csr_matrix((4, n_items), dtype=np.float32))
    model = FakeVectorModel("dot", g["user_factors"][:4], items, i2i_dist="cosine")
    targets = np.random.default_rng(0).permutation(n_items)[:500]
    wl = np.sort(np.random.default_rng(1).choice(n_items, 900, replace=False))
    for whitelist in (None, wl):
        df = recommend_to_items(model, item_ext[targets], dataset, 10, filter_itself=True,
                                items_to_recommend=None if whitelist is None else item_ext[whitelist])
        assert list(df.columns) == ["target_item_id", "item_id", "score", "rank"]
        _, oid, osc = rank_oracle("cosine", items, items, targets, 11, None, whitelist, accum="f64")
        oid, osc = oid.reshape(len(targets), 11), osc.reshape(len(targets), 11)
        keep = oid != targets[:, None]
        keep &= np.cumsum(keep, axis=1) <= 10
        np.testing.assert_array_equal(df["target_item_id"].to_numpy(), np.repeat(item_ext[targets], keep.sum(axis=1)))
        assert_same_ranking((df["item_id"].to_numpy() - 7) // 3, df["score"].to_numpy(), oid[keep], osc[keep], tie_tol=2e-6)
        np.testing.assert_array_equal(df["rank"].to_numpy(), np.cumsum(keep, axis=1)[keep])
        assert not (df["target_item_id"] == df["item_id"]).any()

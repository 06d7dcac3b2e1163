"""GPU: ItemKNN (engine path 9, `b200_rank_topk_knn`, `rectools_b200.item_knn`) bit for bit against the numpy definition
(tests/knn_oracle.py): the full padded arrays -- ids, the fp64 score bits and the counts -- over neighbour counts K,
tie-heavy and signed neighbour matrices, weights, a row where a fused multiply-add would round differently, empty and
fully viewed rows, rows on the dense route, k, filters, whitelists and forced small chunks; then the unmodified
`recommend` / `recommend_to_items` of `ImplicitItemKNNWrapperModel` on the `implicit` stub through `install(item_knn=True)`."""
import os
from fractions import Fraction

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests import knn_oracle

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


def _similarity(n_items, K, rng, kind="random"):
    """A K-neighbour S: each row K distinct items (self included), values by `kind`."""
    rows, cols = [], []
    for i in range(n_items):
        c = rng.choice(n_items, size=min(K, n_items), replace=False)
        c[0] = i if i not in c[1:] else c[0]
        c = np.unique(c)
        rows.append(np.full(len(c), i))
        cols.append(c)
    r, c = np.concatenate(rows), np.concatenate(cols)
    if kind == "counts":
        v = rng.integers(1, 4, size=len(r)).astype(np.float64)  # small integers: many exact ties
    else:
        v = rng.standard_normal(len(r))
        v[rng.random(len(r)) < 0.1] = 0.0  # explicit zeros
    return sparse.csr_matrix((v, (r, c)), shape=(n_items, n_items))


def _users(n_rows, n_items, per_row, rng, unit=False):
    m = np.minimum(rng.integers(0, 2 * per_row + 1, size=n_rows), n_items)
    indptr = np.concatenate([[0], np.cumsum(m)]).astype(np.int64)
    indices = np.concatenate([rng.choice(n_items, size=x, replace=False) for x in m] or [np.zeros(0, int)]).astype(np.int32)
    data = np.ones(len(indices), np.float32) if unit else rng.choice(np.float32([0.5, 1, 1.5, 2, 3.25, 0.1]), size=len(indices))
    return sparse.csr_matrix((data, indices, indptr), shape=(n_rows, n_items))


def _check(S, U, k, F=None, wl=None, **kw):
    from rectools_b200.item_knn import rank_knn

    stats = {}
    ids, sc, cnt = rank_knn(S, U, k, F, wl, stats=stats, **kw)
    oid, osc, ocnt = knn_oracle.rank_knn_np(S, U, k, F, None if wl is None else np.unique(wl))
    np.testing.assert_array_equal(cnt, ocnt)
    np.testing.assert_array_equal(ids, oid)
    np.testing.assert_array_equal(sc.view(np.uint64), osc.view(np.uint64))
    assert stats["path"] == 9
    return stats


@pytest.mark.parametrize("K", [1, 5, 50, 1000])
@pytest.mark.parametrize("kind", ["counts", "random"])
def test_neighbour_counts_and_values(K, kind):
    rng = np.random.default_rng(K)
    n_items = 1500
    S = _similarity(n_items, K, rng, kind)
    U = _users(300, n_items, 6, rng)
    for k in (1, 10, 100):
        _check(S, U, k)
        _check(S, U, k, F=U.sorted_indices())


def test_unit_weights_and_k_above_candidates():
    rng = np.random.default_rng(7)
    S = _similarity(400, 5, rng, "counts")
    U = _users(200, 400, 3, rng, unit=True)
    _check(S, U, 350, F=U.sorted_indices())


def _fma_pair(rng):
    """(c, a, w) with w fp32 such that fl(fl(a * w) + c) != fl(a * w + c)."""
    while True:
        a, c = rng.standard_normal(2)
        w = np.float32(rng.standard_normal())
        two = float(np.float64(a) * np.float64(w)) + c
        one = float(Fraction(a) * Fraction(float(w)) + Fraction(c))
        if one != two:
            return c, a, w


def test_mul_then_add_not_fused():
    rng = np.random.default_rng(11)
    c, a, w = _fma_pair(rng)
    # item 2: entry 0 (S[0, 2] = c, weight 1) then entry 1 (S[1, 2] = a, weight w)
    S = sparse.csr_matrix((np.array([c, 0.25, a, 1.0]), np.array([2, 0, 2, 1]), np.array([0, 2, 3, 4])), shape=(3, 3))
    U = sparse.csr_matrix((np.float32([1.0, w]), np.int32([0, 1]), np.int64([0, 2])), shape=(1, 3))
    _check(S, U, 3)
    from rectools_b200.item_knn import rank_knn

    ids, sc, _ = rank_knn(S, U, 3)
    got = sc[0][list(ids[0]).index(2)]
    assert got == (a * np.float64(w)) + c
    assert got != float(Fraction(a) * Fraction(float(w)) + Fraction(c))


def test_empty_and_fully_viewed_rows():
    rng = np.random.default_rng(13)
    n_items = 50
    S = _similarity(n_items, 4, rng)
    U = _users(60, n_items, 3, rng)
    U = sparse.vstack([U, sparse.csr_matrix((1, n_items), dtype=np.float32)]).tocsr()
    # a row whose filter holds every item it touches
    touched = np.unique(S[U.indices[U.indptr[0] : U.indptr[1]]].indices)
    F = U.sorted_indices().tolil()
    F[0, :] = 0
    F[0, touched] = 1
    F = sparse.csr_matrix(F, dtype=np.float32)
    F.sort_indices()
    _check(S, U, 5, F=F)


def test_dense_route_rows():
    rng = np.random.default_rng(17)
    n_items = 5000
    S = _similarity(n_items, 200, rng)
    U = _users(40, n_items, 30, rng)  # up to 60 entries x 200 neighbours: above the table's 3072
    assert (np.diff(U.indptr) * 200 > 3072).any()
    stats = _check(S, U, 100, F=U.sorted_indices())
    _check(S, U, 7, wl=np.arange(0, n_items, 3))
    assert stats["n_launches"] >= 3


@pytest.mark.parametrize("wl", ["empty", "one", "disjoint", "half"])
def test_whitelists(wl):
    rng = np.random.default_rng(19)
    n_items = 300
    S = sparse.csr_matrix(_similarity(n_items, 6, rng).toarray()[:, :] * (np.arange(n_items) < 200))  # items >= 200 untouched
    S = sparse.csr_matrix(S)
    U = _users(100, n_items, 4, rng)
    w = {"empty": np.zeros(0, np.int32), "one": np.array([5]), "disjoint": np.arange(200, 300), "half": np.arange(0, n_items, 2)}[wl]
    for filt in (None, U.sorted_indices()):
        _check(S, U, 10, F=filt, wl=w)


def test_forced_small_chunks(monkeypatch):
    rng = np.random.default_rng(23)
    S = _similarity(800, 20, rng)
    U = _users(500, 800, 8, rng)
    monkeypatch.setenv("B200_KNN_CHUNK_ROWS", "37")
    stats = _check(S, U, 10, F=U.sorted_indices())
    assert stats["n_chunks"] == -(-500 // 37)


def test_large_shape():
    """10^5 users x 2 10^4 items x K = 100; every row's counts, a sample of rows bit for bit."""
    from rectools_b200.item_knn import rank_knn

    rng = np.random.default_rng(29)
    n_items, n_users, K = 20_000, 100_000, 100
    cols = rng.integers(0, n_items, size=(n_items, K)).astype(np.int64)
    cols[:, 0] = np.arange(n_items)
    S = sparse.csr_matrix((rng.standard_normal(n_items * K), (np.repeat(np.arange(n_items), K), cols.reshape(-1))), shape=(n_items, n_items))
    S.sum_duplicates()
    U = _users(n_users, n_items, 10, rng)
    F = U.sorted_indices()
    stats = {}
    ids, sc, cnt = rank_knn(S, U, 10, F, stats=stats)
    sample = np.sort(rng.choice(n_users, size=1500, replace=False))
    oid, osc, ocnt = knn_oracle.rank_knn_np(S, U[sample], 10, F[sample])
    np.testing.assert_array_equal(cnt[sample], ocnt)
    np.testing.assert_array_equal(ids[sample], oid)
    np.testing.assert_array_equal(sc[sample].view(np.uint64), osc.view(np.uint64))
    assert ((cnt == 10) | (np.diff(U.indptr) == 0) | (cnt < 10)).all()
    assert (cnt[np.diff(U.indptr) == 0] == 0).all()
    print("large shape stats:", stats)


# ---------------------------------------------------------------------------------------------------- through install()
@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    with knn_oracle.stub_methods():
        yield
    stage_reference.remove_from_path(added)


def _dataset(n_users, n_items, per_user, seed):
    from tests.ref_models import synthetic_dataset

    ds = synthetic_dataset(n_users, n_items, per_user, seed=seed)
    raw = ds.get_raw_interactions()
    raw["weight"] = np.random.default_rng(seed).choice([0.5, 1.0, 2.0, 3.0], size=len(raw))
    from rectools.dataset import Dataset

    return Dataset.construct(raw)


def _tie_free_eq(mine, stock, target_col):
    """Frames equal in targets, scores and ranks; items equal as multisets within each run of equal scores, except the
    run a target's list ends in, which the selection may cut at different members."""
    import pandas as pd

    cols = [target_col, "score", "rank"]
    pd.testing.assert_frame_equal(mine[cols].reset_index(drop=True), stock[cols].reset_index(drop=True))
    last = stock.groupby(target_col, sort=False)["score"].transform("last").to_numpy()
    whole = stock["score"].to_numpy() != last
    key = lambda f: sorted(zip(f[target_col], f["score"], f["item_id"]))  # noqa: E731
    assert key(mine[whole]) == key(stock[whole])


@needs_ref
@pytest.mark.parametrize("cls_name", ["ItemItemRecommender", "TFIDFRecommender", "injected"])
def test_install_matches_stock(ref, cls_name):  # pylint: disable=unused-argument,redefined-outer-name
    import implicit.nearest_neighbours as nn
    import pandas as pd
    from rectools.models import ImplicitItemKNNWrapperModel

    import rectools_b200 as rb

    ds = _dataset(400, 250, 12, seed=31)
    model = ImplicitItemKNNWrapperModel(model=getattr(nn, "ItemItemRecommender" if cls_name == "injected" else cls_name)(K=20)).fit(ds)
    if cls_name == "injected":
        S = model.model.similarity.copy()
        S.data = np.random.default_rng(3).standard_normal(S.nnz)
        model.model.similarity = S
    users = ds.user_id_map.external_ids[::3]
    items = ds.item_id_map.external_ids
    calls = [dict(filter_viewed=fv, items_to_recommend=wl, k=k) for fv in (True, False) for wl in (None, items[::4]) for k in (1, 10, 300)]
    i2i_calls = [dict(filter_itself=fi, items_to_recommend=wl, k=k) for fi in (True, False) for wl in (None, items[1::3]) for k in (1, 10)]
    stock = [model.recommend(users, ds, **c) for c in calls]
    stock_i = [model.recommend_to_items(items[:80], ds, **c) for c in i2i_calls]
    rb.install(item_knn=True, fast_recommend=False)
    try:
        for c, s in zip(calls, stock):
            pd.testing.assert_frame_equal(model.recommend(users, ds, **c), s)
        for c, s in zip(i2i_calls, stock_i):
            _tie_free_eq(model.recommend_to_items(items[:80], ds, **c), s, "target_item_id")
    finally:
        rb.uninstall()


@needs_ref
def test_candidate_ranking_model_with_item_knn_generator(ref):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    from implicit.nearest_neighbours import ItemItemRecommender
    from rectools.dataset import Dataset
    from rectools.model_selection import TimeRangeSplitter
    from rectools.models import ImplicitItemKNNWrapperModel, PopularModel
    from rectools.models.ranking import CandidateGenerator, CandidateRankingModel, PerUserNegativeSampler, Reranker
    from sklearn.ensemble import GradientBoostingClassifier

    import rectools_b200 as rb

    raw = _dataset(300, 120, 10, seed=37).get_raw_interactions()
    raw["datetime"] = pd.Timestamp("2024-01-01") + pd.to_timedelta(np.arange(len(raw)) % 10, unit="D")
    ds = Dataset.construct(raw)
    model = CandidateRankingModel(
        candidate_generators=[CandidateGenerator(ImplicitItemKNNWrapperModel(ItemItemRecommender(K=10)), 20, True, True,
                                                 scores_fillna_value=-1.0, ranks_fillna_value=21),
                              CandidateGenerator(PopularModel(), 10, True, True, scores_fillna_value=-1.0, ranks_fillna_value=11)],
        splitter=TimeRangeSplitter("2D", n_splits=1),
        sampler=PerUserNegativeSampler(3, 32),
        reranker=Reranker(GradientBoostingClassifier(random_state=123)),
    )
    model.fit(ds)
    users = ds.user_id_map.external_ids[:150]
    stock = model.recommend(users, ds, k=5, filter_viewed=True)
    rb.install(item_knn=True, fast_recommend=False)
    try:
        mine = model.recommend(users, ds, k=5, filter_viewed=True)
    finally:
        rb.uninstall()
    assert len(stock) > 0
    pd.testing.assert_frame_equal(mine, stock)

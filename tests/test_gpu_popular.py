"""GPU: popularity lists (engine path 7, `b200_rank_topk_list`) on an H100.

- the kernel against the numpy restatement (tests/popular_oracle.py), bit for bit on the full padded arrays: list lengths
  from 0 to 10^6, k from 1 to above the list, rows with nothing viewed, views only outside the list, everything viewed, the
  first k viewed, repeated ids and 10^5 views, 0 / 1 / 10^6 rows, several forced chunks, both kernel shapes;
- every refusal leaves guard-celled outputs untouched;
- through `install(popular=True)`, the unmodified reference's `PopularModel.recommend`, `PopularInCategoryModel.recommend`
  and a `CandidateRankingModel` with a `PopularModel` generator give the stock frames exactly."""
import ctypes as C

import numpy as np
import pytest

from oracle import stage_reference
from tests.popular_oracle import rank_list_np

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


def _rows(rng, n_rows, list_ids, kind, k):
    """(indptr, indices) of `n_rows` viewed rows of one kind."""
    n_list = len(list_ids)
    rows = []
    for r in range(n_rows):
        if kind == "none":
            v = np.zeros(0, np.int64)
        elif kind == "outside":
            v = np.sort(rng.choice(10**7, 20, replace=False)) + 10**7
        elif kind == "all":
            v = np.sort(list_ids)
        elif kind == "first_k":
            v = np.sort(list_ids[:k])
        elif kind == "repeats":
            v = np.sort(np.repeat(list_ids[rng.integers(0, max(n_list, 1), 8)] if n_list else np.zeros(0, np.int64), 3))
        else:  # "mixed": some of the list's head, some of its tail, some outside
            head = list_ids[: min(n_list, 2 * k)][rng.random(min(n_list, 2 * k)) < 0.4]
            v = np.sort(np.concatenate((head, rng.choice(max(n_list, 1), min(30, max(n_list, 1))), [-3, 2**31 - 1])))
        rows.append(v)
    indptr = np.concatenate(([0], np.cumsum([len(v) for v in rows]))).astype(np.int64)
    indices = np.concatenate(rows).astype(np.int32) if rows else np.zeros(0, np.int32)
    return indptr, indices


def _check(list_ids, indptr, indices, n_rows, k, stats=None):
    from rectools_b200 import rank_list

    viewed = None if indptr is None else (indptr, indices)
    st = {}
    pos, cnt = rank_list(list_ids, viewed, k, stats=st, n_rows=n_rows)
    epos, ecnt = rank_list_np(list_ids, indptr, indices, n_rows, k)
    assert pos.shape == epos.shape and pos.dtype == np.int32
    np.testing.assert_array_equal(cnt, ecnt)
    np.testing.assert_array_equal(pos, epos)
    if n_rows and len(list_ids):
        assert st["path"] == 7 and st["k_out"] == min(k, len(list_ids))
    if stats is not None:
        stats.update(st)
    return pos, cnt


@pytest.mark.parametrize("n_list", [0, 1, 31, 32, 33, 1000])
@pytest.mark.parametrize("k", [1, 10, 32, 33, 100, 1000, 10**6])
def test_lengths_and_k_against_oracle(n_list, k):
    rng = np.random.default_rng(n_list * 7 + k)
    list_ids = rng.permutation(n_list * 3)[:n_list].astype(np.int32)
    for kind in ("none", "outside", "all", "first_k", "repeats", "mixed"):
        indptr, indices = _rows(rng, 20, list_ids, kind, k)
        _check(list_ids, indptr, indices, 20, k)
    _check(list_ids, None, None, 5, k)


@pytest.mark.parametrize("k", [1, 100, 1000, 10**6])
def test_list_of_a_million(k):
    rng = np.random.default_rng(k)
    list_ids = rng.permutation(10**6).astype(np.int32)
    n_rows = 40 if k <= 1000 else 8  # (the restatement enumerates every row's whole window)
    indptr, indices = _rows(rng, n_rows, list_ids, "mixed", min(k, 1000))
    _check(list_ids, indptr, indices, n_rows, k)
    # a row with 10^5 viewed ids, most of the list's head among them, and one with everything viewed
    big = np.sort(np.concatenate((list_ids[:90_000], rng.choice(10**6, 10_000, replace=False)))).astype(np.int32)
    allv = np.sort(list_ids)
    indptr = np.array([0, len(big), len(big), len(big) + len(allv)], np.int64)
    _check(list_ids, indptr, np.concatenate((big, allv)), 3, k)


def test_row_counts_and_forced_chunks(monkeypatch):
    rng = np.random.default_rng(7)
    list_ids = rng.permutation(5000).astype(np.int32)
    # 0 and 1 rows
    _check(list_ids, np.zeros(1, np.int64), np.zeros(0, np.int32), 0, 10)
    _check(list_ids, *_rows(rng, 1, list_ids, "mixed", 10), 1, 10)
    # 10^6 rows of ~10 views each, one call
    n = 10**6
    m = rng.integers(0, 20, n)
    indptr = np.concatenate(([0], np.cumsum(m))).astype(np.int64)
    indices = list_ids[rng.integers(0, 60, indptr[-1])]  # from the list's head: most rows lose some of their first k
    indices = indices[np.lexsort((indices, np.repeat(np.arange(n), m)))]  # ascending within each row
    stats = {}
    _check(list_ids, indptr, indices, n, 10, stats)
    assert stats["n_chunks"] == 1
    # several forced chunks, both kernel shapes
    for k in (10, 300):
        monkeypatch.setenv("B200_LIST_CHUNK_ROWS", "333")
        ip, ix = _rows(rng, 1000, list_ids, "mixed", k)
        _check(list_ids, ip, ix, 1000, k, stats)
        assert stats["n_chunks"] == 4
        monkeypatch.delenv("B200_LIST_CHUNK_ROWS")


def test_refusals_leave_outputs_untouched():
    from rectools_b200 import _lib

    lib = _lib.load()
    lst = np.array([4, 2, 7, 1], np.int32)
    indptr = np.array([0, 2, 3], np.int64)
    indices = np.array([2, 7, 4], np.int32)

    def call(n_list=4, lst_=lst, n_rows=2, ip=indptr, ix=indices, k=2):
        pos = np.full((2 + 2, 2), 77, np.int32)  # two guard rows after the outputs
        cnt = np.full(2 + 2, 77, np.int32)
        rc = lib.b200_rank_topk_list(0, n_list, lst_.ctypes.data if lst_ is not None else None, n_rows,
                                     ip.ctypes.data if ip is not None else None, ix.ctypes.data if ix is not None else None, k,
                                     pos.ctypes.data, cnt.ctypes.data, None)
        return rc, pos, cnt

    refusals = [dict(n_list=-1), dict(n_rows=-1), dict(k=0), dict(n_list=2**31), dict(lst_=None),
                dict(lst_=np.array([4, -2, 7, 1], np.int32)), dict(ip=np.array([1, 2, 3], np.int64)),
                dict(ip=np.array([0, 3, 2], np.int64)), dict(ix=None), dict(ix=np.array([7, 2, 4], np.int32))]
    for kw in refusals:
        rc, pos, cnt = call(**kw)
        assert rc == _lib.E_INVALID, kw
        assert (pos == 77).all() and (cnt == 77).all(), kw
    # a row that alone exceeds the chunk budget: 3 * 10^8 viewed ids (1.2 GB of host memory, never copied)
    n_big = 300_000_000
    big = np.zeros(n_big, np.int32)
    pos = np.full((1 + 1, 2), 77, np.int32)
    cnt = np.full(1 + 1, 77, np.int32)
    rc = lib.b200_rank_topk_list(0, 4, lst.ctypes.data, 1, np.array([0, n_big], np.int64).ctypes.data, big.ctypes.data, 2,
                                 pos.ctypes.data, cnt.ctypes.data, None)
    assert rc == _lib.E_NOMEM and "more than a chunk's" in lib.b200_rank_last_error().decode()
    assert (pos == 77).all() and (cnt == 77).all()
    # accepted: the guard rows stay untouched
    rc, pos, cnt = call()
    assert rc == 0
    np.testing.assert_array_equal(pos[:2], [[0, 3], [1, 2]])
    np.testing.assert_array_equal(cnt[:2], [2, 2])
    assert (pos[2:] == 77).all() and (cnt[2:] == 77).all()


# ---------------------------------------------------------------------------------------------- the reference, installed
@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    from rectools.models.popular import PopularModel

    yield PopularModel
    stage_reference.remove_from_path(added)


def _frames_equal(make_models, ds, cases):
    import pandas as pd
    import rectools_b200 as rb

    for model in make_models():
        model.fit(ds)
        expected = []
        for users, k, fv, wl in cases:
            try:
                expected.append(model.recommend(users, ds, k, fv, items_to_recommend=wl))
            except Exception as e:  # pylint: disable=broad-except
                expected.append(e)
        rb.install(popular=True)
        try:
            for (users, k, fv, wl), exp in zip(cases, expected):
                if isinstance(exp, Exception):
                    with pytest.raises(type(exp)):
                        model.recommend(users, ds, k, fv, items_to_recommend=wl)
                    continue
                pd.testing.assert_frame_equal(model.recommend(users, ds, k, fv, items_to_recommend=wl), exp,
                                              obj=f"{model.__class__.__name__} k={k} filter_viewed={fv}")
        finally:
            rb.uninstall()


@needs_ref
def test_popular_model_frames(ref):
    from tests.popular_cases import popular_dataset, popular_settings, recommend_cases

    ds = popular_dataset(n_users=300, n_items=500, per_user=40)
    _frames_equal(lambda: (ref(**kw) for kw in popular_settings()), ds, list(recommend_cases(ds)))


@needs_ref
def test_popular_in_category_frames(ref):
    from rectools.models import PopularInCategoryModel
    from tests.popular_cases import category_settings, popular_dataset, recommend_cases

    ds = popular_dataset(n_users=200, n_items=300, per_user=30, seed=3)
    _frames_equal(lambda: (PopularInCategoryModel(**kw) for kw in category_settings()), ds, list(recommend_cases(ds)))


@needs_ref
def test_candidate_ranking_model_with_popular_generator(ref):
    """`CandidateRankingModel` with `PopularModel` first stages: the candidates, and so the final frame, are the stock ones."""
    import pandas as pd
    import rectools_b200 as rb
    from rectools.model_selection import TimeRangeSplitter
    from rectools.models.ranking import CandidateGenerator, CandidateRankingModel, PerUserNegativeSampler, Reranker
    from sklearn.ensemble import GradientBoostingClassifier
    from tests.popular_cases import popular_dataset

    ds = popular_dataset(n_users=300, n_items=200, per_user=20, seed=4)
    model = CandidateRankingModel(
        candidate_generators=[CandidateGenerator(ref(), 20, True, True, scores_fillna_value=-1.0, ranks_fillna_value=21),
                              CandidateGenerator(ref(popularity="sum_weight", inverse=True), 10, True, True,
                                                 scores_fillna_value=-1.0, ranks_fillna_value=11)],
        splitter=TimeRangeSplitter("5D", n_splits=1),
        sampler=PerUserNegativeSampler(3, 32),
        reranker=Reranker(GradientBoostingClassifier(random_state=123)),
    )
    model.fit(ds)
    users = ds.user_id_map.external_ids[:100]
    expected = model.recommend(users, ds, k=5, filter_viewed=True)
    rb.install(popular=True)
    try:
        got = model.recommend(users, ds, k=5, filter_viewed=True)
    finally:
        rb.uninstall()
    assert len(got) > 0
    pd.testing.assert_frame_equal(got, expected)

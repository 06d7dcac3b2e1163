"""GPU: per-category lists mixed (engine path 8, `b200_rank_topk_list_mix`) on an H100.

- the kernel against the numpy restatement (tests/popular_mix_oracle.py), bit for bit on the full padded arrays: 1 to 200
  lists, k from 1 to 1000, list lengths 0 to 10^5, disjoint and heavily overlapping lists, zero quotas and quotas summing
  below k, both mixings, rows with nothing, everything or 10^4 ids viewed, 0 / 1 / 10^5 rows, forced chunks, and rows
  whose scratch is global memory (forced, and too large for shared memory);
- every refusal leaves guard-celled outputs untouched;
- through `install(popular_in_category=True)`, the unmodified reference's `PopularInCategoryModel.recommend` and a
  `CandidateRankingModel` with a `PopularInCategoryModel` generator give the stock frames exactly."""
import warnings

import numpy as np
import pytest

from oracle import stage_reference
from tests.popular_mix_oracle import rank_list_mix_np

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


def _lists(rng, n_lists, max_len, overlap, universe=None):
    """`n_lists` lists of distinct ids each, lengths 0 .. max_len; `overlap`: drawn from one small pool, so most ids are
    in several lists; otherwise disjoint."""
    lengths = rng.integers(0, max_len + 1, n_lists)
    lengths[rng.random(n_lists) < 0.1] = 0
    if overlap:
        pool = universe or max(2 * max_len, 4)
        return [rng.choice(pool, size=min(int(n), pool), replace=False).astype(np.int32) for n in lengths]
    ids = rng.permutation(int(lengths.sum()) * 2 + 1)
    out, at = [], 0
    for n in lengths:
        out.append(ids[at : at + n].astype(np.int32))
        at += n
    return out


def _quota(rng, n_lists, k, kind):
    if kind == "full":  # sum = k, as the model's ratio strategies give
        return rng.multinomial(k, np.ones(n_lists) / n_lists).astype(np.int32)
    if kind == "zeros":  # most lists get nothing
        q = np.zeros(n_lists, np.int32)
        q[rng.choice(n_lists, size=min(n_lists, max(1, k // 3)), replace=False)[: k]] = 1
        return q
    return rng.multinomial(k // 2, np.ones(n_lists) / n_lists).astype(np.int32)  # below k


def _rows(rng, n_rows, lists, k):
    """(indptr, indices): rows with nothing viewed, everything viewed, part of the lists' heads, and outside ids."""
    all_ids = np.unique(np.concatenate(lists)) if lists and sum(len(x) for x in lists) else np.zeros(0, np.int64)
    rows = []
    for r in range(n_rows):
        kind = r % 4
        if kind == 0 or len(all_ids) == 0:
            v = np.zeros(0, np.int64)
        elif kind == 1:
            v = all_ids
        else:
            heads = np.concatenate([x[: 2 * k] for x in lists])
            v = np.concatenate((heads[rng.random(len(heads)) < 0.4], rng.choice(all_ids, min(20, len(all_ids))), [-3, 2**31 - 1]))
        rows.append(np.unique(v))
    indptr = np.concatenate(([0], np.cumsum([len(v) for v in rows]))).astype(np.int64)
    indices = np.concatenate(rows).astype(np.int32) if rows else np.zeros(0, np.int32)
    return indptr, indices


def _check(lists, quota, mixing, indptr, indices, n_rows, k, stats=None):
    from rectools_b200 import rank_list_mix

    st = {}
    viewed = None if indptr is None else (indptr, indices)
    pos, cnt = rank_list_mix(lists, quota, mixing, viewed, k, stats=st, n_rows=n_rows)
    epos, ecnt = rank_list_mix_np(lists, quota, mixing, indptr, indices, n_rows, k)
    assert pos.shape == epos.shape and pos.dtype == np.int32 and cnt.dtype == np.int32
    np.testing.assert_array_equal(cnt, ecnt)
    np.testing.assert_array_equal(pos, epos)
    if n_rows and epos.shape[1]:
        assert st["path"] == 8 and st["k_out"] == epos.shape[1]
    if stats is not None:
        stats.update(st)
    return pos, cnt


@pytest.mark.parametrize("n_lists", [1, 2, 5, 33, 200])
@pytest.mark.parametrize("k", [1, 10, 32, 33, 100, 1000])
def test_kernel_against_restatement(n_lists, k):
    rng = np.random.default_rng(n_lists * 1009 + k)
    max_len = min(3 * k, 3000) if n_lists <= 33 else min(2 * k, 1200)
    for overlap in (False, True):
        lists = _lists(rng, n_lists, max_len, overlap)
        for q_kind, mixing in (("full", "rotate"), ("zeros", "group"), ("below", "rotate"), ("full", "group")):
            quota = _quota(rng, n_lists, k, q_kind)
            indptr, indices = _rows(rng, 12, lists, k)
            _check(lists, quota, mixing, indptr, indices, 12, k)
        _check(lists, _quota(rng, n_lists, k, "full"), "rotate", None, None, 3, k)


@pytest.mark.parametrize("mixing", ["rotate", "group"])
def test_long_lists_and_many_views(mixing):
    rng = np.random.default_rng(11)
    lists = [rng.permutation(150_000)[:n].astype(np.int32) for n in (100_000, 0, 50_000, 100_000, 7)]
    heavy = np.unique(np.concatenate((lists[0][:5000], rng.choice(150_000, 5000, replace=False))))
    everything = np.unique(np.concatenate(lists))
    rows = [np.zeros(0, np.int64), heavy, everything, heavy[::3]]
    indptr = np.concatenate(([0], np.cumsum([len(v) for v in rows]))).astype(np.int64)
    indices = np.concatenate(rows).astype(np.int32)
    for k in (10, 1000):
        _check(lists, _quota(rng, 5, k, "full"), mixing, indptr, indices, len(rows), k)


def test_row_counts_chunks_and_global_scratch(monkeypatch):
    rng = np.random.default_rng(5)
    lists = _lists(rng, 5, 400, True, universe=600)
    quota = np.array([3, 3, 2, 1, 1], np.int32)
    # 0 and 1 rows
    _check(lists, quota, "rotate", np.zeros(1, np.int64), np.zeros(0, np.int32), 0, 10)
    _check(lists, quota, "group", *_rows(rng, 1, lists, 10), 1, 10)
    # 10^5 rows of ~20 views each from the lists' heads, one call
    n = 10**5
    m = rng.integers(0, 40, n)
    indptr = np.concatenate(([0], np.cumsum(m))).astype(np.int64)
    heads = np.unique(np.concatenate([x[:30] for x in lists]))
    indices = heads[rng.integers(0, len(heads), indptr[-1])].astype(np.int32)
    indices = indices[np.lexsort((indices, np.repeat(np.arange(n), m)))]
    stats = {}
    full, _ = _check(lists, quota, "rotate", indptr, indices, n, 10, stats)
    assert stats["n_chunks"] == 1
    # forced chunks, and the same rows with their scratch in global memory: the same result
    sub = slice(0, 1001)
    ip, ix = indptr[: 1002], indices[: indptr[1001]]
    monkeypatch.setenv("B200_LIST_CHUNK_ROWS", "250")
    pos, _ = _check(lists, quota, "rotate", ip, ix, 1001, 10, stats)
    assert stats["n_chunks"] == 5
    np.testing.assert_array_equal(pos, full[sub])
    monkeypatch.setenv("B200_LIST_MIX_SMEM", "64")
    pos, _ = _check(lists, quota, "rotate", ip, ix, 1001, 10, stats)
    np.testing.assert_array_equal(pos, full[sub])
    monkeypatch.delenv("B200_LIST_CHUNK_ROWS")
    pos, _ = _check(lists, quota, "group", ip, ix, 1001, 100, stats)
    monkeypatch.delenv("B200_LIST_MIX_SMEM")
    np.testing.assert_array_equal(pos, _check(lists, quota, "group", ip, ix, 1001, 100)[0])


def test_rows_beyond_shared_memory():
    """200 lists x k = 1000: 2 * 10^5 entry slots per row, more than shared memory holds, so every row sorts in its global
    slice."""
    rng = np.random.default_rng(9)
    lists = _lists(rng, 200, 2000, True, universe=30_000)
    for mixing in ("rotate", "group"):
        quota = _quota(rng, 200, 1000, "full")
        indptr, indices = _rows(rng, 6, lists, 1000)
        _check(lists, quota, mixing, indptr, indices, 6, 1000)


def test_refusals_leave_outputs_untouched():
    from rectools_b200 import _lib

    lib = _lib.load()
    offs = np.array([0, 2, 4], np.int64)
    ids = np.array([4, 2, 7, 4], np.int32)
    quota = np.array([1, 1], np.int32)
    indptr = np.array([0, 2, 3], np.int64)
    indices = np.array([2, 7, 4], np.int32)

    def p(a):
        return a.ctypes.data if a is not None else None

    def call(n_lists=2, offs_=offs, ids_=ids, q=quota, mixing=0, n_rows=2, ip=indptr, ix=indices, k=2):
        pos = np.full((2 + 2, 2), 77, np.int32)  # two guard rows after the outputs
        cnt = np.full(2 + 2, 77, np.int32)
        rc = lib.b200_rank_topk_list_mix(0, n_lists, p(offs_), p(ids_), p(q), mixing, n_rows, p(ip), p(ix), k,
                                         pos.ctypes.data, cnt.ctypes.data, None)
        return rc, pos, cnt

    refusals = [dict(n_lists=-1), dict(n_rows=-1), dict(k=0), dict(mixing=2), dict(mixing=-1), dict(offs_=None),
                dict(offs_=np.array([1, 2, 4], np.int64)), dict(offs_=np.array([0, 3, 2], np.int64)),
                dict(offs_=np.array([0, 2, 2**31], np.int64)), dict(ids_=None), dict(ids_=np.array([4, -2, 7, 4], np.int32)),
                dict(q=None), dict(q=np.array([-1, 1], np.int32)), dict(q=np.array([2, 1], np.int32)),
                dict(ip=np.array([1, 2, 3], np.int64)), dict(ip=np.array([0, 3, 2], np.int64)), dict(ix=None),
                dict(ix=np.array([7, 2, 4], np.int32))]
    for kw in refusals:
        rc, pos, cnt = call(**kw)
        assert rc == _lib.E_INVALID, kw
        assert (pos == 77).all() and (cnt == 77).all(), kw
    # a row that alone exceeds the chunk budget: 3 * 10^8 viewed ids (1.2 GB of host memory, never copied)
    n_big = 300_000_000
    big = np.zeros(n_big, np.int32)
    pos = np.full((1 + 1, 2), 77, np.int32)
    cnt = np.full(1 + 1, 77, np.int32)
    rc = lib.b200_rank_topk_list_mix(0, 2, offs.ctypes.data, ids.ctypes.data, quota.ctypes.data, 0, 1,
                                     np.array([0, n_big], np.int64).ctypes.data, big.ctypes.data, 2, pos.ctypes.data,
                                     cnt.ctypes.data, None)
    assert rc == _lib.E_NOMEM and "more than a chunk's" in lib.b200_rank_last_error().decode()
    assert (pos == 77).all() and (cnt == 77).all()
    # accepted: the guard rows stay untouched.  Row 0 viewed 2 and 7 (lists [4, 2], [7, 4]): 4 (main of list 0), then 4
    # again (a repeat); row 1 viewed 4: 2, then 7 (rotate: r' 0 of list 0, r' 0 of list 1)
    rc, pos, cnt = call()
    assert rc == 0
    np.testing.assert_array_equal(pos[:2], [[0, -1], [1, 2]])
    np.testing.assert_array_equal(cnt[:2], [1, 2])
    assert (pos[2:] == 77).all() and (cnt[2:] == 77).all()


# ---------------------------------------------------------------------------------------------- the reference, installed
@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    from rectools.models import PopularInCategoryModel

    yield PopularInCategoryModel
    stage_reference.remove_from_path(added)


def _frames_equal(models, ds, cases):
    import pandas as pd
    import rectools_b200 as rb

    for model in models:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            model.fit(ds)
        expected = []
        for users, k, fv, wl in cases:
            try:
                expected.append(model.recommend(users, ds, k, fv, items_to_recommend=wl))
            except Exception as e:  # pylint: disable=broad-except
                expected.append(e)
        rb.install(popular_in_category=True)
        try:
            for (users, k, fv, wl), exp in zip(cases, expected):
                if isinstance(exp, Exception):
                    with pytest.raises(type(exp)):
                        model.recommend(users, ds, k, fv, items_to_recommend=wl)
                    continue
                pd.testing.assert_frame_equal(model.recommend(users, ds, k, fv, items_to_recommend=wl), exp,
                                              obj=f"{type(model).__name__} {model.mixing_strategy} k={k} filter_viewed={fv}")
        finally:
            rb.uninstall()


def _cases(ds):
    ext_users = ds.user_id_map.external_ids
    ext_items = ds.item_id_map.external_ids
    n_items = len(ext_items)
    for fv in (True, False):
        yield ext_users, 7, fv, None
        yield np.concatenate((ext_users[9:2:-1], [999_999])), 1, fv, None  # a cold user in the request
        yield ext_users[:12], n_items + 5, fv, None
        yield ext_users, 5, fv, ext_items[::3]
        yield ext_users, 3, fv, ext_items[-3:]  # items nobody viewed: every list empty unless add_cold


@needs_ref
@pytest.mark.parametrize("n_categories", [1, 2, 5, 40])
def test_popular_in_category_frames(ref, n_categories):
    from tests.popular_in_category_cases import category_dataset, in_category_settings

    ds = category_dataset(n_users=80, n_items=120, n_categories=n_categories, per_user=20, seed=n_categories, idle_users=3)
    _frames_equal([ref(**kw) for kw in in_category_settings(n_categories)], ds, list(_cases(ds)))


@needs_ref
def test_larger_dataset_frames(ref):
    from tests.popular_in_category_cases import category_dataset

    ds = category_dataset(n_users=10_000, n_items=2000, n_categories=20, per_user=30, seed=12)
    users = ds.user_id_map.external_ids
    cases = [(users, 10, True, None), (users[::3], 100, True, ds.item_id_map.external_ids[::2]), (users[::7], 30, False, None)]
    _frames_equal([ref(category_feature="category", mixing_strategy=m, ratio_strategy=r)
                   for m, r in (("rotate", "proportional"), ("group", "equal"))], ds, cases)


@needs_ref
def test_candidate_ranking_model_with_popular_in_category_generator(ref):
    import pandas as pd
    import rectools_b200 as rb
    from rectools.model_selection import TimeRangeSplitter
    from rectools.models.ranking import CandidateGenerator, CandidateRankingModel, PerUserNegativeSampler, Reranker
    from sklearn.ensemble import GradientBoostingClassifier
    from tests.popular_in_category_cases import category_dataset

    ds = category_dataset(n_users=300, n_items=200, n_categories=6, per_user=20, seed=4)
    model = CandidateRankingModel(
        candidate_generators=[CandidateGenerator(ref(category_feature="category"), 20, True, True, scores_fillna_value=-1.0,
                                                 ranks_fillna_value=21),
                              CandidateGenerator(ref(category_feature="category", mixing_strategy="group",
                                                     popularity="sum_weight"), 10, True, True,
                                                 scores_fillna_value=-1.0, ranks_fillna_value=11)],
        splitter=TimeRangeSplitter("5D", n_splits=1),
        sampler=PerUserNegativeSampler(3, 32),
        reranker=Reranker(GradientBoostingClassifier(random_state=123)),
    )
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model.fit(ds)
    users = ds.user_id_map.external_ids[:100]
    expected = model.recommend(users, ds, k=5, filter_viewed=True)
    rb.install(popular_in_category=True)
    try:
        got = model.recommend(users, ds, k=5, filter_viewed=True)
    finally:
        rb.uninstall()
    assert len(got) > 0
    pd.testing.assert_frame_equal(got, expected)

"""GPU: scored pairs (engine path 6, `b200_rank_topk_pairs`) on the H100.

- bit for bit: full `positions` / `offsets` against the stable numpy restatement (tests/pairs_oracle.py) for group sizes
  around k, the warp (32) and shared-memory (256 / 2048 / 8192) class edges and a 200 000-row group; k = 1, 10, 100, 1000
  and k at or above the longest group; 10^7 shuffled pairs; every score type; +-0, +-inf, NaN, subnormals, +-DBL_MAX,
  INT64_MIN / MAX and float64 scores one ulp apart; every row dropped, one group, n_groups = n;
- host and device buffers give identical results; device inputs written behind a sleep on a side stream and on the legacy
  stream; refusals leave guarded outputs untouched;
- `reranker_recommend` against the unmodified reference `Reranker.recommend`, and `CandidateRankingModel.recommend` end to
  end with install(rerank=True) against stock, under the position tie rule."""
import ctypes as C

import numpy as np
import pytest

from oracle import stage_reference
from tests.pairs_oracle import rank_pairs_np, reranker_recommend_np

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


def _check(codes, scores, k, n_groups=None, device_too=True):
    import torch
    from rectools_b200 import rank_pairs

    ng = int(codes.max()) + 1 if n_groups is None and len(codes) else (n_groups or 0)
    exp_pos, exp_off = rank_pairs_np(codes, scores, k, ng)
    stats = {}
    pos, off = rank_pairs(codes, scores, k, n_groups=ng, stats=stats)
    np.testing.assert_array_equal(off, exp_off)
    np.testing.assert_array_equal(pos, exp_pos)
    assert stats["path"] == 6
    if device_too:
        dpos, doff = rank_pairs(torch.from_numpy(codes).cuda(), torch.from_numpy(np.ascontiguousarray(scores)).cuda(), k, n_groups=ng)
        assert dpos.is_cuda and doff.is_cuda
        np.testing.assert_array_equal(doff.cpu().numpy(), exp_off)
        np.testing.assert_array_equal(dpos.cpu().numpy(), exp_pos)
    return stats


def _sized_groups(sizes, rng, ties=True):
    codes = np.repeat(np.arange(len(sizes), dtype=np.int64), sizes)
    perm = rng.permutation(len(codes))
    codes = codes[perm]
    scores = rng.random(len(codes))
    if ties:
        scores = np.round(scores * 50) / 50  # many exact ties: their order is the position rule's
    return codes, scores


@pytest.mark.parametrize("k", [1, 10, 100, 1000])
def test_group_sizes_around_every_class_edge(k):
    rng = np.random.default_rng(k)
    sizes = [1, max(k - 1, 1), k, k + 1, 31, 32, 33, 256, 257, 2048, 2049, 8192, 8193, 200_000]
    codes, scores = _sized_groups(sizes, rng)
    _check(codes, scores, k)
    codes, scores = _sized_groups(sizes, rng, ties=False)
    _check(codes, scores, k)


def test_k_at_or_above_the_longest_group():
    rng = np.random.default_rng(5)
    codes, scores = _sized_groups([3, 40, 300, 5000, 9000, 200_000], rng)
    for k in (200_000, 200_001, 2**31 - 1):
        _check(codes, scores, k)


def test_ten_million_shuffled_pairs():
    rng = np.random.default_rng(7)
    sizes = np.concatenate([rng.integers(1, 200, 60_000), rng.integers(200, 20_000, 200), [1_000_000]])
    codes, scores = _sized_groups(sizes, rng)
    n = 10_000_000
    if len(codes) < n:  # pad with dropped rows
        codes = np.concatenate([codes, -np.ones(n - len(codes), np.int64)])
        scores = np.concatenate([scores, rng.random(n - len(scores))])
        perm = rng.permutation(n)
        codes, scores = codes[perm], scores[perm]
    codes, scores = codes[:n], scores[:n]
    stats = _check(codes, scores, 100, n_groups=len(sizes), device_too=False)
    assert stats["ms_total"] > 0 and stats["n_launches"] > 0


SPECIAL_F64 = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 5e-324, -5e-324, 2.2250738585072014e-308,
                        np.finfo(np.float64).max, -np.finfo(np.float64).max, 1.0, np.nextafter(1.0, 2.0),
                        np.nextafter(1.0, 0.0), 0.1, np.nextafter(0.1, 1.0), -np.nan], dtype=np.float64)


@pytest.mark.parametrize("dtype", [np.float64, np.float32, np.int64, np.int32])
@pytest.mark.parametrize("size", [20, 300, 5000, 50_000])
def test_special_values_every_score_type(dtype, size):
    rng = np.random.default_rng(size)
    if dtype == np.float64:
        pool = SPECIAL_F64
    elif dtype == np.float32:
        pool = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, np.finfo(np.float32).max,
                         -np.finfo(np.float32).max, 1.0, np.nextafter(np.float32(1), np.float32(2)), 0.5], dtype=np.float32)
    else:
        info = np.iinfo(dtype)
        pool = np.array([info.min, info.max, info.min + 1, info.max - 1, 0, -1, 1, 2], dtype=dtype)
    scores = pool[rng.integers(0, len(pool), size * 4)]
    codes = rng.integers(-1, 4, size * 4).astype(np.int64)
    for k in (1, 3, size, size * 4):
        _check(codes, scores, k, n_groups=4)


def test_float64_last_bit_differences_are_kept():
    base = np.linspace(0.25, 0.75, 4000)
    scores = np.concatenate([base, np.nextafter(base, 1.0), np.nextafter(base, 0.0)])
    rng = np.random.default_rng(3)
    perm = rng.permutation(len(scores))
    scores = scores[perm]
    assert len(np.unique(scores.astype(np.float32))) < len(np.unique(scores))  # fp32 would merge them
    for n_groups in (1, 7, 300):
        codes = rng.integers(0, n_groups, len(scores)).astype(np.int64)
        _check(codes, scores, 50, n_groups=n_groups)


def test_degenerate_shapes():
    rng = np.random.default_rng(11)
    n = 10_000
    _check(-np.ones(n, np.int64), rng.random(n), 5, n_groups=3)  # every row dropped
    _check(np.zeros(n, np.int64), rng.random(n), 7)  # one group
    _check(rng.permutation(n).astype(np.int64), rng.random(n), 2)  # n_groups = n
    _check(np.zeros(0, np.int64), np.zeros(0), 3, n_groups=0)
    _check(np.zeros(0, np.int64), np.zeros(0), 3, n_groups=4)
    _check(np.array([2, 2], np.int64), np.array([1.0, 2.0]), 1, n_groups=5)  # empty groups around


# ------------------------------------------------------------------------------------------------------ buffers and streams
def _raw_call(n, codes_p, scores_p, stype, n_groups, k, flags, out_pos_p, out_off_p, stream=None):
    from rectools_b200 import _lib

    st = _lib.Stats()
    return _lib.load().b200_rank_topk_pairs(0, stream, n, codes_p, scores_p, stype, n_groups, k, flags, out_pos_p, out_off_p, C.byref(st))


@pytest.mark.parametrize("legacy", [False, True])
def test_device_inputs_written_behind_a_sleep(legacy):
    import torch
    from rectools_b200 import _lib

    rng = np.random.default_rng(2)
    n, ng, k = 1_000_000, 5000, 20
    codes = rng.integers(-1, ng, n).astype(np.int64)
    scores = rng.random(n)
    exp_pos, exp_off = rank_pairs_np(codes, scores, k, ng)
    src_c, src_s = torch.from_numpy(codes).cuda(), torch.from_numpy(scores).cuda()
    d_c = torch.full_like(src_c, -1)  # decoy: every row dropped
    d_s = torch.zeros_like(src_s)
    out_pos = torch.full((min(n, ng * k),), -7, dtype=torch.int64, device="cuda")
    out_off = torch.full((ng + 1,), -7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    stream = torch.cuda.default_stream() if legacy else side
    with torch.cuda.stream(stream):
        torch.cuda._sleep(200_000_000)  # pylint: disable=protected-access
        d_c.copy_(src_c)
        d_s.copy_(src_s)
        rc = _raw_call(n, d_c.data_ptr(), d_s.data_ptr(), _lib.PAIRS_F64, ng, k,
                       _lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE, out_pos.data_ptr(), out_off.data_ptr(),
                       None if legacy else side.cuda_stream)
        assert rc == 0
        got_off = out_off.clone()  # ordered after the call on the same stream
        got_pos = out_pos.clone()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(got_off.cpu().numpy(), exp_off)
    np.testing.assert_array_equal(got_pos[: exp_off[-1]].cpu().numpy(), exp_pos)


def test_refusals_leave_outputs_untouched():
    import torch
    from rectools_b200 import _lib

    codes = np.array([0, 1, 2, 5], np.int64)  # 5 is out of range for n_groups = 3
    scores = np.array([1.0, 2.0, 3.0, 4.0])
    out_pos = np.full(16, -7, np.int64)
    out_off = np.full(8, -7, np.int64)
    P = lambda a: a.ctypes.data  # noqa: E731
    cases = [
        (4, P(codes), P(scores), _lib.PAIRS_F64, 3, 2, 0),  # code out of range
        (3, P(codes), P(scores), _lib.PAIRS_F64, 3, 0, 0),  # k < 1
        (3, P(codes), P(scores), 9, 3, 2, 0),  # unknown score type
        (3, P(np.array([0, -2, 1], np.int64)), P(scores), _lib.PAIRS_F64, 3, 2, 0),  # code below -1
        (-1, P(codes), P(scores), _lib.PAIRS_F64, 3, 2, 0),
        (3, P(codes), P(scores), _lib.PAIRS_F64, 3, 2, 4),  # unknown flag
    ]
    for n, cp, sp, stype, ng, k, flags in cases:
        assert _raw_call(n, cp, sp, stype, ng, k, flags, P(out_pos), P(out_off)) == _lib.E_INVALID
        assert (out_pos == -7).all() and (out_off == -7).all()
    # device inputs and outputs: the range check happens on the device, before any output is written
    d_codes, d_scores = torch.from_numpy(codes).cuda(), torch.from_numpy(scores).cuda()
    d_pos = torch.full((16,), -7, dtype=torch.int64, device="cuda")
    d_off = torch.full((8,), -7, dtype=torch.int64, device="cuda")
    rc = _raw_call(4, d_codes.data_ptr(), d_scores.data_ptr(), _lib.PAIRS_F64, 3, 2, _lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE,
                   d_pos.data_ptr(), d_off.data_ptr())
    assert rc == _lib.E_INVALID
    torch.cuda.synchronize()
    assert (d_pos == -7).all() and (d_off == -7).all()
    with pytest.raises(ValueError, match="outside"):
        from rectools_b200 import rank_pairs

        rank_pairs(codes, scores, 2, n_groups=3)
    # the library still works after the refusals
    _check(np.array([0, 1, 2, 0], np.int64), scores, 1)


# --------------------------------------------------------------------------------------------------- against the reference
@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    from rectools.models.ranking.candidate_ranking import Reranker

    yield Reranker
    stage_reference.remove_from_path(added)


def _pairs_frame(n_users, per_user, rng, ties):
    import pandas as pd

    users = np.repeat(np.arange(n_users) * 3 + 11, per_user)
    perm = rng.permutation(len(users))
    scores = rng.random(len(users))
    if ties:
        scores = np.round(scores * 20) / 20
    else:
        scores = rng.permutation(len(users)).astype(np.float64) / len(users)  # distinct
    return pd.DataFrame({"user_id": users[perm], "item_id": rng.integers(0, 10_000, len(users)), "score": scores,
                         "feat": rng.random(len(users)).astype(np.float32)})


@needs_ref
@pytest.mark.parametrize("k", [1, 10, 150])
def test_reranker_recommend_equals_the_reference_without_ties(ref, k):
    import pandas as pd
    from rectools_b200 import reranker_recommend

    df = _pairs_frame(300, 100, np.random.default_rng(k), ties=False)
    df.loc[::17, "user_id"] = None  # NA users: dropped
    for add_rank_col in (True, False):
        pd.testing.assert_frame_equal(reranker_recommend(df, k, add_rank_col), ref.recommend(df, k, add_rank_col))


@needs_ref
def test_reranker_recommend_with_ties(ref):
    import pandas as pd
    from rectools_b200 import reranker_recommend

    df = _pairs_frame(50, 5000, np.random.default_rng(4), ties=True)  # groups large enough for quicksort to reorder ties
    k = 300
    got = reranker_recommend(df, k)
    expected = ref.recommend(df, k)
    pd.testing.assert_frame_equal(got, reranker_recommend_np(df, k))
    # the reference's tie order is implementation-defined: equal as multisets within each (user, score) run
    pd.testing.assert_frame_equal(got[["user_id", "score", "rank"]], expected[["user_id", "score", "rank"]])
    key = ["user_id", "score"]
    cols = ["user_id", "score", "item_id", "feat"]
    # the k-th place cuts a tied run: compare the runs that both sides return whole
    last = got.groupby("user_id", sort=False)["score"].transform("last")
    whole = got["score"] != last
    a = got[whole][cols].sort_values(cols).reset_index(drop=True)
    b = expected[whole.to_numpy()][cols].sort_values(cols).reset_index(drop=True)
    pd.testing.assert_frame_equal(a, b)
    assert got.groupby(key, sort=False).size().equals(expected.groupby(key, sort=False).size())


def _two_stage_dataset(rng):
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset

    n_users, n_items, n = 400, 300, 12_000
    df = pd.DataFrame({
        Columns.User: rng.integers(0, n_users, n) * 5 + 1,
        Columns.Item: rng.zipf(1.3, n) % n_items,
        Columns.Weight: 1.0,
        Columns.Datetime: pd.Timestamp("2024-01-01") + pd.to_timedelta(rng.integers(0, 14, n), unit="D"),
    }).drop_duplicates([Columns.User, Columns.Item])
    return Dataset.construct(df)


@needs_ref
def test_candidate_ranking_model_end_to_end(ref):
    import pandas as pd
    import rectools_b200 as rb
    from rectools.model_selection import TimeRangeSplitter
    from rectools.models import PopularModel, PureSVDModel
    from rectools.models.ranking import CandidateGenerator, CandidateRankingModel, PerUserNegativeSampler, Reranker
    from sklearn.ensemble import GradientBoostingClassifier

    dataset = _two_stage_dataset(np.random.default_rng(0))
    model = CandidateRankingModel(
        candidate_generators=[CandidateGenerator(PopularModel(), 30, True, True, scores_fillna_value=-1.0, ranks_fillna_value=31),
                              CandidateGenerator(PureSVDModel(factors=8, random_state=32), 30, True, True, scores_fillna_value=-1.0,
                                                 ranks_fillna_value=31)],
        splitter=TimeRangeSplitter("2D", n_splits=1),
        sampler=PerUserNegativeSampler(3, 32),
        reranker=Reranker(GradientBoostingClassifier(random_state=123)),
    )
    model.fit(dataset)
    users = dataset.user_id_map.external_ids[:200]
    original = Reranker.__dict__["recommend"]
    seen = {}

    def recording(name, method):
        def recommend(cls, scored_pairs, k, add_rank_col=True):
            seen[name] = (scored_pairs.copy(), k, add_rank_col)
            out = method.__get__(None, cls)(scored_pairs, k, add_rank_col)
            seen[name + "_out"] = out.copy()
            return out

        return classmethod(recommend)

    try:
        # both runs rank the first stage on the engine, so the reranker gets the same scored pairs and is the only
        # difference between them (the stock first stage may round a candidate's score differently)
        rb.install()
        assert Reranker.__dict__["recommend"] is original
        Reranker.recommend = recording("stock", original)
        stock = model.recommend(users, dataset, k=10, filter_viewed=True)
        Reranker.recommend = original
        rb.uninstall()
        rb.install(rerank=True)
        rebound = Reranker.__dict__["recommend"]
        assert rebound is not original
        Reranker.recommend = recording("got", rebound)
        got = model.recommend(users, dataset, k=10, filter_viewed=True)
        Reranker.recommend = rebound
    finally:
        rb.uninstall()
    assert Reranker.__dict__["recommend"] is original
    pairs, k, add_rank_col = seen["got"]
    pd.testing.assert_frame_equal(pairs, seen["stock"][0])
    assert len(pairs) > 10 * 150 and (k, add_rank_col) == (10, True)
    # exactly the stable restatement of the position tie rule
    pd.testing.assert_frame_equal(seen["got_out"], reranker_recommend_np(pairs, k, add_rank_col))
    pd.testing.assert_frame_equal(got, seen["got_out"])
    # against stock: the same users, scores and ranks; within a tied score run the same items as a multiset (the stock
    # order of tied pairs is numpy quicksort's)
    pd.testing.assert_frame_equal(got[["user_id", "score", "rank"]], stock[["user_id", "score", "rank"]])
    key = lambda f: sorted(zip(f["user_id"], f["score"], f["item_id"]))  # noqa: E731
    last = got.groupby("user_id", sort=False)["score"].transform("last")
    whole = (got["score"] != last).to_numpy()
    assert key(got[whole]) == key(stock[whole])

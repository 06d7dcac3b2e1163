"""GPU: the radix selection of paths 2 and 3 for k > 1024 and k = None (`filter_mask_kernel` + `large_k_select_kernel`,
rectools_b200/csrc/large_k_select.cuh).

Every comparison is of the full padded arrays -- ids, scores, counts and every unfilled slot (-1 / -FLT_MAX) -- against the
fp64 oracle with no tie tolerance, or bit for bit against the streaming passes (B200_SELECT=0), which the radix selection
must reproduce exactly.  The catalogues have integer-valued factors (tests/exact_cases.py), so large tie blocks straddle
the k-th score of every row, and k runs across the shared-memory capacity S of the survivors' sort."""
import numpy as np
import pytest
from scipy import sparse

from tests import exact_cases as ec

pytestmark = pytest.mark.gpu

S = 12288  # LK_SMEM_PAIRS (rectools_b200/csrc/sizes.h)


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


def _same(got, exp, name):
    ids, sc, cnt = got
    eids, esc, ecnt = exp
    assert ids.shape == eids.shape, f"{name}: shape {ids.shape} vs {eids.shape}"
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, eids, err_msg=f"{name}: ids")
    np.testing.assert_array_equal(sc, esc, err_msg=f"{name}: scores")


def _bits_same(got, ref, name):
    for a, b, what in zip(got, ref, ("ids", "scores", "counts")):
        np.testing.assert_array_equal(np.ascontiguousarray(a).view(np.int32), np.ascontiguousarray(b).view(np.int32),
                                      err_msg=f"{name}: {what}")


def _prefix(exp, k):
    ids, sc, cnt = exp
    return ids[:, :k], sc[:, :k], np.minimum(cnt, k)


def _sparse_rows(rng, n_rows, d, max_nnz=60):
    nnz = rng.integers(0, max_nnz, n_rows)
    indptr = np.r_[0, np.cumsum(nnz)].astype(np.int64)
    indices = rng.integers(0, d, int(indptr[-1])).astype(np.int32)
    data = (rng.choice([-3, -2, -1, 1, 2, 3], int(indptr[-1])) / 2).astype(np.float32)
    return sparse.csr_matrix((data, indices, indptr), shape=(n_rows, d))


def _filter(rng, n, n_rows, n_keep=1_500):
    """Random filter rows with ids >= N; row 3 filters everything, row 4 all but n_keep objects."""
    rows = [rng.integers(0, n + 500, rng.integers(0, 3_000)) for _ in range(n_rows)]
    rows[3] = np.arange(n)
    rows[4] = np.delete(np.arange(n), rng.choice(n, n_keep, replace=False))
    return ec.csr_from_rows(rows, n)


def _with_select(monkeypatch, value, fn):
    monkeypatch.setenv("B200_SELECT", str(value))
    try:
        return fn()
    finally:
        monkeypatch.delenv("B200_SELECT")


# ------------------------------------------------------------------------------------------------ 1. against the oracle
@pytest.fixture(scope="module")
def dense_cases():
    rng = np.random.default_rng(3)
    n, d = 40_000, 6
    out = {"dot": (ec.int_matrix(rng, n, d), ec.int_matrix(rng, 48, d)),
           "cosine": (ec.pooled_matrix(rng, n, d, 500), ec.int_matrix(rng, 48, d))}
    for _, sub in out.values():
        sub[7] = 0  # every score +-0: one tie over the whole row
    return out


@pytest.mark.parametrize("with_wl", [False, True])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_dense_k_across_the_sort_capacity(lib, dense_cases, distance, with_wl):
    """Path 3, k = 1025, S - 1, S, S + 1, 2 S + 7, n_pos and n_pos + 5 (the whole catalogue), filter and whitelist."""
    from rectools_b200 import Engine

    objects, subjects = dense_cases[distance]
    n = len(objects)
    rng = np.random.default_rng(5)
    wl = np.sort(rng.choice(n, 30_000, replace=False)).astype(np.int32) if with_wl else None
    n_pos = n if wl is None else len(wl)
    filt = _filter(rng, n, len(subjects))
    exp = ec.expected_padded(distance, subjects, objects, np.arange(len(subjects)), None, filt, wl)
    assert exp[2][3] == 0 and exp[2][4] <= 1_500
    eng = Engine(objects, cosine=distance == "cosine")
    for k in (1025, S - 1, S, S + 1, 2 * S + 7, n_pos, n_pos + 5):
        got = eng.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, whitelist=wl)
        assert eng.last_stats["path"] == 3, eng.last_stats
        _same(got, _prefix(exp, min(k, n_pos)), f"{distance} wl={with_wl} k={k}")
    eng.close()


@pytest.mark.parametrize("with_wl", [False, True])
@pytest.mark.parametrize("shape", [(3_000, 3_000), (13_000, 32)])
def test_sparse_subjects(lib, shape, with_wl):
    """Path 2: an EASE-shaped problem (objects = items x items weights) and one with n_pos > S, k up to None."""
    import rectools_b200 as rb

    n, d = shape
    rng = np.random.default_rng(n)
    objects = ec.int_matrix(rng, n, d)
    csr = _sparse_rows(rng, 40, d)
    wl = np.sort(rng.choice(n, n - 700, replace=False)) if with_wl else None
    filt = _filter(rng, n, 40, n_keep=1_100)
    ranker = rb.B200Ranker("dot", csr, objects)
    sids = np.arange(40)
    exp = ec.expected_padded("dot", csr, objects, sids, None, filt, wl)
    n_pos = n if wl is None else len(wl)
    for k in (1025, 2048, S + 1, None):
        if k is not None and k > n_pos:
            continue
        _, ids, sc, cnt = ranker.rank_padded(sids, k, filt, wl)
        assert ranker.last_stats["path"] == 2, ranker.last_stats
        _same((ids, sc, cnt), _prefix(exp, n_pos if k is None else k), f"sparse {shape} wl={with_wl} k={k}")


def test_ties_across_the_select_digits(lib, monkeypatch):
    """d = 1, subject 1: the scores are the objects, drawn from consecutive floats around digit boundaries of the order key
    (keys differing only in the last 1, 2 or 3 bytes) with hundreds of exact copies each; k lands inside tie blocks."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(9)
    bases = np.array([0x3F800000, 0x3F7FFF00, 0x3F80FFF0, 0x3EFFFFFF, 0xBF800000, 0x407FFFFE], np.uint32)
    vals = np.concatenate([(b + np.arange(-3, 4, dtype=np.int64)).astype(np.uint32) for b in bases]).view(np.float32)
    objects = rng.choice(vals, size=(20_000, 1)).astype(np.float32)
    subjects = np.array([[1.0], [-1.0], [2.0]], np.float32)
    exp = ec.expected_padded("dot", subjects, objects, np.arange(3), None)
    eng = Engine(objects, cosine=False)
    top = np.unique(objects, return_counts=True)[1][::-1].cumsum()  # ranks where the tie blocks of row 0 end
    ks = sorted({1025, 2000, int(top[20]), int(top[20]) + 1, S, 15_000, 20_000})
    for k in ks:
        got = eng.topk(k, subjects=subjects)
        assert eng.last_stats["path"] == 3
        _same(got, _prefix(exp, k), f"digit ties k={k}")
        _bits_same(got, _with_select(monkeypatch, 0, lambda: eng.topk(k, subjects=subjects)), f"digit ties vs passes k={k}")
    eng.close()


def test_special_scores(lib, monkeypatch):
    """+-0 (tied, ordered by id), -inf and NaN (never returned), real -FLT_MAX (returned by the kernels), +inf, subnormals:
    bit-identical to the passes, counts = the scores > -inf, ties in id order."""
    from rectools_b200 import Engine

    fmax = np.float32(np.finfo(np.float32).max)
    vals = np.array([-fmax, -1, -0.0, 0.0, 1, np.nan, np.inf, -np.inf, fmax, 1e-45, -1e-45, 2, -2], np.float32)
    rng = np.random.default_rng(13)
    objects = rng.choice(vals, size=(3_000, 1)).astype(np.float32)
    subjects = np.array([[1.0], [-1.0], [0.0], [2.0], [0.5]], np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        scores = (subjects.astype(np.float64) @ objects.astype(np.float64).T).astype(np.float32)
    eng = Engine(objects, cosine=False)
    for k in (1025, 2_000, 3_000):
        ids, sc, cnt = eng.topk(k, subjects=subjects)
        assert eng.last_stats["path"] == 3
        _bits_same((ids, sc, cnt), _with_select(monkeypatch, 0, lambda: eng.topk(k, subjects=subjects)), f"special k={k}")
        np.testing.assert_array_equal(cnt, np.minimum(k, (scores > -np.inf).sum(axis=1)))
        for r in range(len(subjects)):
            s, i = sc[r, : cnt[r]], ids[r, : cnt[r]]
            assert not np.isnan(s).any() and (s > -np.inf).all()
            assert ((s[:-1] > s[1:]) | ((s[:-1] == s[1:]) & (i[:-1] < i[1:]))).all()
            np.testing.assert_array_equal(s, scores[r, i])
        assert (sc[2, : cnt[2]] == 0).all()  # 0 x (-1) and 0 x 1: one tie, in id order
    eng.close()


# ------------------------------------------------------------------------------------------------ 2. the call shapes
def test_row_chunks_row_map_filters_offset_host_and_device(lib, monkeypatch):
    """300 000 objects: three path-3 chunks at k = 1025 (864 rows each) and at k = S + 5 (sort scratch: 768 rows each);
    resident subjects through a row map with repeats, filters with out-of-range ids, a nonzero id offset, host and device
    inputs and outputs.  Bit-identical to the passes; the first rows against the oracle."""
    import torch

    from rectools_b200 import Engine

    rng = np.random.default_rng(17)
    n, d, off = 300_000, 8, 1_000
    objects = ec.int_matrix(rng, n, d)
    subjects = ec.int_matrix(rng, 1_500, d)
    sids = np.r_[rng.permutation(1_500), rng.integers(0, 1_500, 600)].astype(np.int64)
    rows = [rng.integers(off - 50, off + n + 100, rng.integers(0, 400)) for _ in sids]
    filt = ec.csr_from_rows(rows, off + n)
    eng = Engine(objects, cosine=False, id_offset=off)
    eng.set_subjects(subjects)
    local = sparse.csr_matrix(filt[:, off:off + n])
    exp = ec.expected_padded("dot", subjects, objects, sids[:64], S + 5, local[:64])
    dev = torch.device("cuda:0")
    d_sids = torch.from_numpy(sids).to(dev)
    d_ip = torch.from_numpy(filt.indptr.astype(np.int64)).to(dev)
    d_ix = torch.from_numpy(filt.indices.astype(np.int32)).to(dev)
    for k in (1025, S + 5):
        got = eng.topk(k, subject_ids=sids, indptr=filt.indptr, indices=filt.indices)
        assert eng.last_stats["path"] == 3
        ref = _with_select(monkeypatch, 0, lambda: eng.topk(k, subject_ids=sids, indptr=filt.indptr, indices=filt.indices))
        _bits_same(got, ref, f"chunks host k={k}")
        e_ids, e_sc, e_cnt = _prefix(exp, k)
        _same((got[0][:64], got[1][:64], got[2][:64]), (np.where(e_ids >= 0, e_ids + off, -1), e_sc, e_cnt), f"oracle k={k}")
        o_ids = torch.full((len(sids), k), 7, dtype=torch.int32, device=dev)
        o_sc = torch.full((len(sids), k), 3.0, dtype=torch.float32, device=dev)
        o_cnt = torch.full((len(sids),), -2, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        st = eng.topk_ptrs(len(sids), k, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE,
                           subject_ids=d_sids.data_ptr(), indptr=d_ip.data_ptr(), indices=d_ix.data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert st["path"] == 3
        _bits_same((o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy()), ref, f"chunks device k={k}")
    eng.close()


# ------------------------------------------------------------------------------------------------ 3. cross-checks
def test_radix_equals_passes_for_k_1025_to_2048(lib, monkeypatch):
    from rectools_b200 import Engine

    rng = np.random.default_rng(19)
    n, d = 5_000, 4
    objects = ec.int_matrix(rng, n, d)
    subjects = ec.int_matrix(rng, 33, d)
    filt = _filter(rng, n, 33, n_keep=1_300)
    wl = np.sort(rng.choice(n, 4_000, replace=False)).astype(np.int32)
    eng = Engine(objects, cosine=False)
    for k in (1025, 1056, 1300, 1301, 1537, 2048):
        for w in (None, wl):
            call = lambda: eng.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, whitelist=w)  # noqa: E731
            _bits_same(call(), _with_select(monkeypatch, 0, call), f"k={k} wl={w is not None}")
    eng.close()


@pytest.mark.parametrize("path", [2, 3])
def test_radix_at_small_k_equals_the_passes(lib, monkeypatch, path):
    """B200_SELECT=2: the radix selection at k = 33, 128, 129, 1000 on paths 2 and 3 against the default (the passes)."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(23 + path)
    n = 6_000
    d = 64
    objects = ec.int_matrix(rng, n, d)
    filt = _filter(rng, n, 40, n_keep=100)
    eng = Engine(objects, cosine=False)
    if path == 2:
        kw = dict(sparse_subjects=_sparse_rows(rng, 40, d))
    else:
        kw = dict(subjects=ec.int_matrix(rng, 40, d), flags=lib.Q_FORCE_EXACT)
    for k in (33, 128, 129, 1000):
        if path == 3 and k <= 128:
            continue
        ref = eng.topk(k, indptr=filt.indptr, indices=filt.indices, **kw)
        assert eng.last_stats["path"] == path
        got = _with_select(monkeypatch, 2, lambda: eng.topk(k, indptr=filt.indptr, indices=filt.indices, **kw))
        assert eng.last_stats["path"] == path
        _bits_same(got, ref, f"path {path} k={k}")
    eng.close()


def test_launches_do_not_grow_with_k(lib):
    from rectools_b200 import Engine

    rng = np.random.default_rng(29)
    n, d = 20_000, 8
    objects = ec.int_matrix(rng, n, d)
    subjects = ec.int_matrix(rng, 50, d)
    filt = _filter(rng, n, 50)
    eng = Engine(objects, cosine=False)
    launches = set()
    for k in (1025, 4096, S + 1, n):
        eng.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices)
        assert eng.last_stats["path"] == 3
        launches.add(eng.last_stats["n_launches"])
    assert len(launches) == 1, launches
    eng.close()


# ------------------------------------------------------------------------------------------------ 4. the Python API
@pytest.fixture(scope="module")
def ref():
    from oracle import stage_reference

    if not stage_reference.available():
        pytest.skip("reference package not staged (oracle/_ref)")
    added = stage_reference.add_to_path()
    import rectools  # noqa: F401

    yield
    import rectools_b200

    rectools_b200.uninstall()
    stage_reference.remove_from_path(added)


@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_ranker_k_none_against_the_reference(ref, distance):
    from rectools.models.rank import Distance, ImplicitRanker

    import rectools_b200 as rb
    from tests.helpers import assert_same_ranking

    rng = np.random.default_rng(31)
    u = rng.standard_normal((300, 32)).astype(np.float32)
    i = rng.standard_normal((3_000, 32)).astype(np.float32)
    filt = _filter(rng, 3_000, 200)
    wl = np.sort(rng.choice(3_000, 2_500, replace=False))
    sids = rng.permutation(300)[:200]
    dist = Distance.DOT if distance == "dot" else Distance.COSINE
    for w in (None, wl):
        exp = ImplicitRanker(dist, u, i, use_gpu=False).rank(sids, k=None, filter_pairs_csr=filt, sorted_object_whitelist=w)
        ranker = rb.B200Ranker(dist, u, i)
        got = ranker.rank(sids, k=None, filter_pairs_csr=filt, sorted_object_whitelist=w)
        assert ranker.last_stats["path"] == 3 and ranker.last_stats["k_out"] > 1024, ranker.last_stats
        np.testing.assert_array_equal(got[0], exp[0])
        assert_same_ranking(got[1], got[2], exp[1], exp[2], rtol=3e-5, atol=3e-6, tie_tol=3e-6, msg=f"{distance} wl={w is not None}")


def test_ease_recommend_all_items_through_install(ref):
    from rectools.models import EASEModel

    import rectools_b200
    from rectools_b200 import integration
    from tests.helpers import assert_same_ranking
    from tests.ref_models import synthetic_dataset

    dataset = synthetic_dataset(1_500, 1_400, 20, seed=6)
    model = EASEModel(regularization=200.0).fit(dataset)
    users = dataset.user_id_map.external_ids[::3]
    n_items = dataset.item_id_map.size
    exp = model.recommend(users, dataset, k=n_items, filter_viewed=True)
    rectools_b200.install(device=0)
    try:
        got = model.recommend(users, dataset, k=n_items, filter_viewed=True)
        stats = [e.last_stats for e in integration._ENGINE_CACHE.values()]  # pylint: disable=protected-access
    finally:
        rectools_b200.uninstall()
    assert any(s.get("path") == 2 and s.get("k_out") == n_items for s in stats), stats
    assert list(exp.columns) == list(got.columns)
    np.testing.assert_array_equal(exp["user_id"].to_numpy(), got["user_id"].to_numpy())
    assert_same_ranking(got["item_id"].to_numpy(), got["score"].to_numpy(), exp["item_id"].to_numpy(), exp["score"].to_numpy(),
                        rtol=3e-5, atol=3e-6, tie_tol=1e-5)


def test_vector_model_recommend_all_items_through_install(ref):
    """`VectorModel` (an injected ALS model) after `install()`: `recommend(k=n_items)` and the bound ranker's
    `rank(k=None)` reach path 3 with the radix selection and agree with the stock reference path."""
    import rectools.models.vector as vector
    from rectools.models.rank import Distance

    import rectools_b200
    from rectools_b200 import integration
    from tests.helpers import assert_same_ranking
    from tests.ref_models import injected_als, synthetic_dataset

    rng = np.random.default_rng(37)
    n_users, n_items = 1_500, 1_400
    dataset = synthetic_dataset(n_users, n_items, 20, seed=7)
    u = (rng.standard_normal((n_users, 32)) / np.sqrt(32)).astype(np.float32)
    i = (rng.standard_normal((n_items, 32)) / np.sqrt(32)).astype(np.float32)
    model = injected_als(u, i)
    users = dataset.user_id_map.external_ids[::3]
    exp = model.recommend(users, dataset, k=n_items, filter_viewed=True)
    sids = np.arange(0, n_users, 5)
    filt = _filter(rng, n_items, len(sids), n_keep=1_100)
    stock = vector.ImplicitRanker
    exp_rank = stock(Distance.DOT, u, i).rank(sids, k=None, filter_pairs_csr=filt)
    rectools_b200.install(device=0)
    try:
        got = model.recommend(users, dataset, k=n_items, filter_viewed=True)
        stats = [e.last_stats for e in integration._ENGINE_CACHE.values()]  # pylint: disable=protected-access
        ranker = vector.ImplicitRanker(Distance.DOT, u, i)
        assert isinstance(ranker, rectools_b200.B200ImplicitRanker)
        got_rank = ranker.rank(sids, k=None, filter_pairs_csr=filt)
        rank_stats = dict(ranker.last_stats)
    finally:
        rectools_b200.uninstall()
    assert any(s.get("path") == 3 and s.get("k_out") == n_items for s in stats), stats
    assert rank_stats["path"] == 3 and rank_stats["k_out"] == n_items, rank_stats
    assert list(exp.columns) == list(got.columns)
    np.testing.assert_array_equal(exp["user_id"].to_numpy(), got["user_id"].to_numpy())
    assert_same_ranking(got["item_id"].to_numpy(), got["score"].to_numpy(), exp["item_id"].to_numpy(), exp["score"].to_numpy(),
                        rtol=3e-5, atol=3e-6, tie_tol=3e-6, msg="recommend")
    np.testing.assert_array_equal(got_rank[0], exp_rank[0])
    assert_same_ranking(got_rank[1], got_rank[2], exp_rank[1], exp_rank[2], rtol=3e-5, atol=3e-6, tie_tol=3e-6, msg="rank")

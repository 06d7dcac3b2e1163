"""GPU: candidate sets (engine path 5, `b200_rank_topk_candidates`, `B200Ranker.rank_candidates`), every row of every call
checked against the rounding-interval oracle (`tests/score_interval.check_topk`) with no tolerance beyond the ambiguous
entries it reports.  A row's allow-list C_r is expressed there as a complement filter: everything outside C_r, plus the
row's own filter, is ineligible.

Covered: DOT / COSINE / EUCLIDEAN; fp32 objects and fp16 / bf16 objects kept at 16 bits; d = 1, 24, 65, 128, 256; rows of
0, 1, k-1, k, S-1, S, S+1 and 50 000 candidates (S = LK_SMEM_PAIRS, the shared-memory sort's capacity); k = 1, 10, 1024,
1025 and None; filters overlapping the lists, fully filtered rows; +-0, +-inf, NaN, +-FLT_MAX and subnormal scores; ties
on integer catalogues; three and more row chunks; resident and explicit subjects with subject_ids; bit-identity with
`rank_padded` when C_r is the whole catalogue on integer catalogues; every refusal with its outputs untouched; and the
ANN classes of `rectools_b200.ann` on the engine against the unmodified reference classes on the nmslib stand-in."""
import os
import pickle
import sys

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests.exact_cases import int_matrix
from tests.score_interval import check_topk

pytestmark = pytest.mark.gpu

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
S = 12288  # LK_SMEM_PAIRS
FMAX = np.finfo(np.float32).max


def _engine(objects, cosine=False, dtype="f32"):
    import torch

    from rectools_b200 import _lib
    from rectools_b200.ranker import Engine

    if dtype == "f32":
        return Engine(objects, cosine=cosine), objects
    t = torch.from_numpy(np.asarray(objects, np.float32)).to("cuda", torch.float16 if dtype == "f16" else torch.bfloat16)
    dt = _lib.DT_F16 if dtype == "f16" else _lib.DT_BF16
    eng = Engine(None, cosine=cosine, objects_device_ptr=t.data_ptr(), shape=tuple(t.shape), objects_dtype=dt, keep_16bit=True)
    eng._keep_tensor = t  # pylint: disable=protected-access  (read in place for the engine's life)
    return eng, t.cpu()


def _lists(rng, n_obj, lens):
    rows = [np.sort(rng.choice(n_obj, n, replace=False)).astype(np.int32) for n in lens]
    indptr = np.zeros(len(lens) + 1, np.int64)
    np.cumsum([len(r) for r in rows], out=indptr[1:])
    return indptr, (np.concatenate(rows) if rows else np.empty(0, np.int32)).astype(np.int32)


def _complement_filter(n_obj, cand_indptr, cand_indices, f_indptr=None, f_indices=None):
    rows = []
    for r in range(len(cand_indptr) - 1):
        banned = np.setdiff1d(np.arange(n_obj), cand_indices[cand_indptr[r] : cand_indptr[r + 1]])
        if f_indptr is not None:
            banned = np.union1d(banned, f_indices[f_indptr[r] : f_indptr[r + 1]])
        rows.append(banned)
    indptr = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(x) for x in rows], out=indptr[1:])
    return indptr, (np.concatenate(rows) if rows else np.empty(0)).astype(np.int64)


def _filter(rng, cand_indptr, cand_indices, n_obj, full_rows=()):
    """A filter that overlaps the lists (half of each row's candidates plus random others); rows in `full_rows` lose
    every candidate."""
    rows = []
    for r in range(len(cand_indptr) - 1):
        c = cand_indices[cand_indptr[r] : cand_indptr[r + 1]]
        take = c if r in full_rows else c[rng.random(len(c)) < 0.5]
        rows.append(np.unique(np.concatenate([take, rng.choice(n_obj, 5)])).astype(np.int32))
    indptr = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(x) for x in rows], out=indptr[1:])
    return indptr, np.concatenate(rows).astype(np.int32)


def _check(eng, objects, subjects, k, cand, filt=None, cosine=False, name="", **kw):
    cand_indptr, cand_indices = cand
    f_indptr, f_indices = filt if filt is not None else (None, None)
    got = eng.topk_candidates(k, cand_indptr, cand_indices, subjects=subjects, indptr=f_indptr, indices=f_indices, **kw)
    assert eng.last_stats["path"] == 5
    comp = _complement_filter(objects.shape[0], cand_indptr, cand_indices, f_indptr, f_indices)
    # A row that returns its whole list makes every one of its scores a checked, returned entry, so the share of ambiguous
    # entries (a score the interval oracle cannot pin to one fp32 value: ~2e-4 of them at d = 256) is that of single
    # scores here, not of the far rarer entries near a top-k cut that the checker's default share is sized for.
    check_topk(got, subjects, objects, k, cosine=cosine, filter_csr=comp, name=name, max_ambiguous=1e-3)
    return got


LENS = [0, 1, 9, 10, 1023, 1024, 1025, S - 1, S, S + 1, 50_000]


@pytest.mark.parametrize("k", [1, 10, 1024, 1025, None])
@pytest.mark.parametrize("cosine", [False, True])
def test_row_lengths_and_k(k, cosine):
    rng = np.random.default_rng(1)
    n_obj, d = 60_000, 24
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    subjects = rng.standard_normal((len(LENS), d)).astype(np.float32)
    eng, _ = _engine(objects, cosine)
    cand = _lists(rng, n_obj, LENS)
    kk = max(LENS) if k is None else k
    _check(eng, objects, subjects, kk, cand, cosine=cosine, name=f"lens k={k}")
    filt = _filter(rng, *cand, n_obj, full_rows=(3, 8))
    got = _check(eng, objects, subjects, kk, cand, filt, cosine=cosine, name=f"lens+filter k={k}")
    assert got[2][3] == 0 and got[2][8] == 0 and got[2][0] == 0
    # B200_Q_FORCE_EXACT changes nothing
    from rectools_b200 import _lib

    again = eng.topk_candidates(kk, *cand, subjects=subjects, indptr=filt[0], indices=filt[1], flags=_lib.Q_FORCE_EXACT)
    for a, b in zip(got, again):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("d", [1, 24, 65, 128, 256])
@pytest.mark.parametrize("cosine", [False, True])
def test_object_types_and_widths(dtype, d, cosine):
    rng = np.random.default_rng(d)
    n_obj = 20_000
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    subjects = rng.standard_normal((40, d)).astype(np.float32)
    eng, obj_seen = _engine(objects, cosine, dtype)
    cand = _lists(rng, n_obj, rng.integers(0, 3000, 40))
    filt = _filter(rng, *cand, n_obj, full_rows=(5,))
    for k in (10, 1025):
        _check(eng, obj_seen, subjects, k, cand, filt, cosine=cosine, name=f"{dtype} d={d} k={k}")


def test_euclidean_through_the_ranker():
    from rectools_b200.ranker import B200Ranker, prepare_factors, Distance

    rng = np.random.default_rng(5)
    n_obj, n_sub, d = 30_000, 64, 32
    items = rng.standard_normal((n_obj, d)).astype(np.float32)
    users = rng.standard_normal((n_sub, d)).astype(np.float32)
    ranker = B200Ranker("euclidean", users, items)
    sub_aug, obj_aug, _, _ = prepare_factors(Distance.EUCLIDEAN, users, items)
    sids = rng.permutation(n_sub)[:50]
    ip, ix = _lists(rng, n_obj, rng.integers(0, 5000, len(sids)))
    cands = sparse.csr_matrix((np.ones(len(ix)), ix, ip), shape=(len(sids), n_obj))
    _, ids, sc, cnt = ranker.rank_candidates_padded(sids, cands, 100)
    check_topk((ids, sc, cnt), sub_aug[sids], obj_aug, 100, filter_csr=_complement_filter(n_obj, ip, ix), name="euclidean")
    # the flat triplet: the padded rows with `rank`'s post-scaling
    s_flat, i_flat, d_flat = ranker.rank_candidates(sids, cands, 100)
    mask = np.arange(ids.shape[1])[None, :] < cnt[:, None]
    np.testing.assert_array_equal(i_flat, ids[mask])
    want = np.sqrt(np.maximum(ranker.subjects_dots[s_flat] - sc[mask], 0)).astype(np.float32)
    np.testing.assert_array_equal(d_flat, want)


def test_special_scores():
    """d = 1, subject 1: each score is the object value itself (a -0 object scores +0)."""
    tiny = np.float32(1e-45)
    vals = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, FMAX, -FMAX, tiny, -tiny, 1.0, -1.0, 0.0, np.nan, np.inf], np.float32)
    objects = vals.reshape(-1, 1)
    eng, _ = _engine(objects)
    n = len(vals)
    cand_indptr = np.array([0, n, n + 5, n + 5 + 3])
    cand_indices = np.concatenate([np.arange(n), [3, 4, 12, 2, 13], [0, 1, 11]]).astype(np.int32)
    cand_indices[n : n + 5] = np.sort(cand_indices[n : n + 5])
    ids, sc, cnt = eng.topk_candidates(20, cand_indptr, cand_indices, subjects=np.ones((3, 1), np.float32))
    for r in range(3):
        c = cand_indices[cand_indptr[r] : cand_indptr[r + 1]]
        kept = [i for i in c if vals[i] > -np.inf]  # -inf and NaN never rank
        want = sorted(kept, key=lambda i: (-float(vals[i]) + 0.0, i))  # +-0 tie, by id
        assert cnt[r] == len(want)
        assert ids[r, : cnt[r]].tolist() == want
        # the fp64 sum starts at +0, so a -0 object scores +0 (as on every route); every other score is the value itself
        want_bits = np.where(vals[want] == 0, np.float32(0.0), vals[want]).astype(np.float32)
        np.testing.assert_array_equal(sc[r, : cnt[r]].view(np.uint32), want_bits.view(np.uint32))
        assert (ids[r, cnt[r] :] == -1).all() and (sc[r, cnt[r] :] == -FMAX).all()


@pytest.mark.parametrize("cosine", [False, True])
def test_integer_ties_and_bit_identity_with_rank(cosine):
    rng = np.random.default_rng(3)
    n_obj, n_sub, d = 40_000, 96, 8
    objects = int_matrix(rng, n_obj, d, -2, 2).astype(np.float32)
    subjects = int_matrix(rng, n_sub, d, -2, 2).astype(np.float32)
    eng, _ = _engine(objects, cosine)
    f_indptr, f_indices = _filter(rng, *_lists(rng, n_obj, rng.integers(0, 200, n_sub)), n_obj)
    whole = (np.arange(n_sub + 1, dtype=np.int64) * n_obj, np.tile(np.arange(n_obj, dtype=np.int32), n_sub))
    for k in (1, 10, 100, 1024, 1025, 20_000):
        got = eng.topk_candidates(k, *whole, subjects=subjects, indptr=f_indptr, indices=f_indices)
        ref = eng.topk(k, subjects=subjects, indptr=f_indptr, indices=f_indices)
        for a, b in zip(got, ref):
            np.testing.assert_array_equal(a.view(np.uint32) if a.dtype == np.float32 else a, b.view(np.uint32) if b.dtype == np.float32 else b)
        assert got[0].shape == (n_sub, k)
    # ties inside short lists, checked against the intervals (exact here: no ambiguity allowed)
    cand = _lists(rng, n_obj, rng.integers(0, 4000, n_sub))
    rep = _check(eng, objects, subjects, 50, cand, (f_indptr, f_indices), cosine=cosine, name="int ties")
    assert rep is not None


def test_row_chunks_and_subject_ids(monkeypatch):
    rng = np.random.default_rng(9)
    n_obj, n_sub, d = 30_000, 2_000, 65
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    subjects = rng.standard_normal((n_sub, d)).astype(np.float32)
    eng, _ = _engine(objects)
    eng.set_subjects(subjects)
    sids = rng.integers(0, n_sub, 900)
    cand = _lists(rng, n_obj, rng.integers(0, 400, len(sids)))
    filt = _filter(rng, *cand, n_obj, full_rows=(0, 300))
    whole = eng.topk_candidates(30, *cand, subject_ids=sids, indptr=filt[0], indices=filt[1])
    assert eng.last_stats["n_chunks"] == 1
    monkeypatch.setenv("B200_CHUNK_ROWS", "256")
    got = eng.topk_candidates(30, *cand, subject_ids=sids, indptr=filt[0], indices=filt[1])
    assert eng.last_stats["n_chunks"] == 4
    for a, b in zip(whole, got):
        np.testing.assert_array_equal(a, b)
    comp = _complement_filter(n_obj, *cand, *filt)
    check_topk(got, subjects[sids], objects, 30, filter_csr=comp, name="chunks, resident subjects")
    # an explicit matrix indexed by subject_ids gives the same rows
    exp = eng.topk_candidates(30, *cand, subjects=subjects, subject_ids=sids, indptr=filt[0], indices=filt[1])
    for a, b in zip(exp, got):
        np.testing.assert_array_equal(a, b)
    st = eng.last_stats
    assert st["path"] == 5 and st["ms_main"] > 0 and st["ms_select"] > 0 and st["ms_total"] >= st["ms_main"]


def test_refusals_leave_outputs_untouched():
    import torch

    from rectools_b200 import _lib
    from rectools_b200.ranker import Engine

    rng = np.random.default_rng(0)
    n_obj, d = 1_000, 16
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    subjects = rng.standard_normal((4, d)).astype(np.float32)
    eng = Engine(objects, cosine=False)
    ip, ix = _lists(rng, n_obj, [3, 0, 5, 2])

    def out():
        return np.full((4, 10), 7, np.int32), np.full((4, 10), 3.5, np.float32), np.full(4, 9, np.int32)

    def refused(exc, match, k=10, ip=ip, ix=ix, **kw):
        o = out()
        with pytest.raises(exc, match=match):
            eng.topk_candidates(k, ip, ix, out=o, **{"subjects": subjects, **kw})
        assert (o[0] == 7).all() and (o[1] == 3.5).all() and (o[2] == 9).all()

    bad = ip.copy()
    bad[2] = 0
    refused(ValueError, "not monotone", ip=bad)
    refused(ValueError, "not an object", ix=np.where(ix == ix[0], n_obj, ix).astype(np.int32))
    swapped = ix.copy()
    swapped[[3, 4]] = swapped[[4, 3]]
    refused(ValueError, "strictly ascending", ix=swapped)
    for flag in (_lib.Q_INPUTS_ON_DEVICE, _lib.Q_OUTPUTS_ON_DEVICE, _lib.Q_SHARED_THRESHOLDS, _lib.Q_FORCE_TC):
        refused(NotImplementedError, "b200_rank_topk_candidates", flags=flag)
    refused(NotImplementedError, "whitelist", whitelist=np.arange(10))
    refused(NotImplementedError, "object_rows", subjects=None, object_rows=np.arange(4))
    refused(NotImplementedError, "sub_", subjects=None, sparse_subjects=sparse.csr_matrix(subjects))
    dev = torch.from_numpy(subjects).cuda()
    eng.set_subjects_device(dev.data_ptr(), 4)
    refused(NotImplementedError, "device memory", subjects=None, subject_ids=np.arange(4))
    eng.set_subjects(subjects)
    refused(ValueError, "out of range", subjects=None, subject_ids=np.array([0, 1, 2, 4]))
    off = Engine(objects, cosine=False, id_offset=100)
    o = out()
    with pytest.raises(NotImplementedError, match="id offset"):
        off.topk_candidates(10, ip, ix, subjects=subjects, out=o)
    assert (o[0] == 7).all()


def test_group_ranker_is_refused():
    from rectools_b200.ranker import B200Ranker

    rng = np.random.default_rng(0)
    r = B200Ranker("dot", rng.standard_normal((5, 8)), rng.standard_normal((100, 8)), device=[0])
    with pytest.raises(NotImplementedError, match="engine group"):
        r.rank_candidates([0, 1], sparse.csr_matrix((2, 100)), 5)


def test_ranker_normalises_and_keeps_the_caller_matrix():
    from rectools_b200.ranker import B200Ranker

    rng = np.random.default_rng(2)
    users, items = rng.standard_normal((20, 8)).astype(np.float32), rng.standard_normal((500, 8)).astype(np.float32)
    ranker = B200Ranker("cosine", users, items)
    data, ind, ptr = np.ones(6), np.array([40, 3, 40, 7, 2, 2]), np.array([0, 3, 3, 6])
    m = sparse.csr_matrix((data, ind, ptr), shape=(3, 500))
    keep = (m.indices.copy(), m.indptr.copy())
    s, i, sc = ranker.rank_candidates([4, 5, 6], m, None, sorted_object_whitelist=np.array([2, 3, 7, 40]))
    np.testing.assert_array_equal(m.indices, keep[0])
    np.testing.assert_array_equal(m.indptr, keep[1])
    assert sorted(i[s == 4].tolist()) == [3, 40] and len(i[s == 5]) == 0 and sorted(i[s == 6].tolist()) == [2, 7]
    # the same pairs get the same scores as `rank`
    s2, i2, sc2 = ranker.rank([4], None)
    ref = dict(zip(i2.tolist(), sc2.tolist()))
    for obj, score in zip(i[s == 4].tolist(), sc[s == 4].tolist()):
        assert ref[obj] == score
    with pytest.raises(ValueError, match="Number of rows"):
        ranker.rank_candidates([1, 2], m)
    with pytest.raises(ValueError, match="must be in"):
        ranker.rank_candidates([1, 2, 3], sparse.csr_matrix((np.ones(1), [600], [0, 1, 1, 1]), shape=(3, 700)))


# ----------------------------------------------------------------------------------------- ANN classes against the reference
@pytest.fixture(scope="module")
def ref_ann():
    if not stage_reference.available():
        pytest.skip("reference package neither staged nor checked out")
    added = stage_reference.add_to_path()
    stub = os.path.join(ROOT, "oracle", "nmslib_stub")
    sys.path.insert(0, stub)
    from rectools.tools import ann

    yield ann
    sys.path.remove(stub)
    sys.modules.pop("nmslib", None)
    stage_reference.remove_from_path(added)


@pytest.mark.parametrize("space", ["cosinesimil", "negdotprod", "l2"])
@pytest.mark.parametrize("kind", ["u2i", "i2i"])
def test_ann_classes_on_the_engine(ref_ann, space, kind):
    from rectools_b200 import ann as b200_ann

    rng = np.random.default_rng(11)
    n_items, n_users, d = 2_000, 60, 16
    if space == "cosinesimil":  # continuous factors: no ties to break
        items, users = rng.standard_normal((n_items, d)), rng.standard_normal((n_users, d))
    else:  # integer factors: every distance exact on both sides, ties by id on both
        items, users = int_matrix(rng, n_items, d, -3, 3), int_matrix(rng, n_users, d, -3, 3)
    items, users = items.astype(np.float32), users.astype(np.float32)
    imap = {f"i{i}": i for i in range(n_items)}
    params = {"method": "hnsw", "space": space}
    if kind == "u2i":
        umap = {f"u{i}": i for i in range(n_users)}
        ref = ref_ann.UserToItemAnnRecommender(users, items, umap, imap, index_top_k=n_items, index_init_params=params).fit()
        got = b200_ann.B200UserToItemAnnRecommender(users, items, umap, imap, index_init_params=params).fit()
        targets, call = [f"u{i}" for i in range(n_users)], "get_item_list_for_user_batch"
    else:
        ref = ref_ann.ItemToItemAnnRecommender(items, imap, index_top_k=n_items, index_init_params=params).fit()
        got = b200_ann.B200ItemToItemAnnRecommender(items, imap, index_init_params=params).fit()
        targets, call = [f"i{i}" for i in rng.choice(n_items, 40, replace=False)], "get_item_list_for_item_batch"
    lists = [[f"i{x}" for x in rng.choice(n_items, rng.integers(0, 400), replace=True)] for _ in targets]
    vec = users if kind == "u2i" else items
    rows = [int(t[1:]) for t in targets]

    def same(a, b):
        """Equal lists; for COSINE (continuous factors) an fp32 near-tie may swap two neighbours, so there the fp64
        cosine of each position must agree to 1e-6 instead."""
        assert [len(x) for x in a] == [len(x) for x in b]
        if space != "cosinesimil":
            assert [list(x) for x in a] == [list(x) for x in b]
            return
        for r, x, y in zip(rows, a, b):
            q = vec[r].astype(np.float64)
            cos = lambda ids: [q @ items[int(i[1:])] / np.linalg.norm(items[int(i[1:])].astype(np.float64)) for i in ids]
            np.testing.assert_allclose(cos(x), cos(y), rtol=0, atol=1e-6 * np.linalg.norm(q))

    for top_n in (1, 10, 100):
        for arg in (lists, None):
            same(getattr(got, call)(targets, top_n, arg), getattr(ref, call)(targets, top_n, arg))
    restored = pickle.loads(pickle.dumps(got))
    same(getattr(restored, call)(targets, 10, lists), getattr(ref, call)(targets, 10, lists))

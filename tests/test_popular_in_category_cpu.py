"""CPU: per-category lists mixed (engine path 8, `b200_rank_topk_list_mix`, `rectools_b200.popular`) up to where a GPU is
needed.

- the export is declared, exported and bound, the ABI stays 6 and the engine-group exports are unchanged;
- tests/list_mix_plan_driver.cpp prints `plan_list_mix` (rectools_b200/csrc/list_mix_plan.h): entry slots, the scratch
  route, chunk bounds within the byte budget, the B200_LIST_CHUNK_ROWS cap, and every refusal;
- the numpy restatement (tests/popular_mix_oracle.py) against the unmodified reference's
  `PopularInCategoryModel._recommend_u2i`, with its stock category models;
- the host logic with the library replaced by a stand-in backed by the restatement: the arguments handed over, the
  dtypes, each case handed to the stock method, `install(popular_in_category=True)` / `uninstall()`, and
  `PopularInCategoryModel.recommend` frames equal to the stock method's."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile
import warnings

import numpy as np
import pytest

from oracle import stage_reference
from tests.popular_mix_oracle import rank_list_mix_np, recommend_in_category_u2i_np
from tests.popular_oracle import rank_list_np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_export_declared_exported_and_bound():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    assert re.search(r"\bint b200_rank_topk_list_mix\s*\(", header)
    assert re.search(r"8 = per-category lists minus viewed ids, mixed \(b200_rank_topk_list_mix\)", header)
    assert "#define B200_MIX_ROTATE 0" in header and "#define B200_MIX_GROUP 1" in header
    assert (_lib.MIX_ROTATE, _lib.MIX_GROUP) == (0, 1)
    assert "b200_rank_topk_list_mix" in _lib.EXPORTS
    assert "#define B200_RANK_ABI_VERSION 6" in header and _lib.ABI_VERSION == 6
    assert sorted(e for e in _lib.EXPORTS if e.startswith("b200_rank_group_")) == [
        "b200_rank_group_create", "b200_rank_group_create_ex", "b200_rank_group_destroy", "b200_rank_group_get_info",
        "b200_rank_group_set_subjects", "b200_rank_group_topk"]
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    assert C.CDLL(_lib.LIB_PATH).b200_rank_topk_list_mix is not None
    assert _lib.load().b200_rank_topk_list_mix.argtypes is not None


def test_host_refusals_leave_outputs_untouched():
    """Refusals are decided before the device is touched, so they run here (the library needs no GPU to load)."""
    from rectools_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = _lib.load()
    offs = np.array([0, 2, 4], np.int64)
    ids = np.array([4, 2, 7, 4], np.int32)
    quota = np.array([1, 1], np.int32)

    def call(**kw):
        a = dict(n_lists=2, offs=offs, ids=ids, q=quota, mixing=0, k=2)
        a.update(kw)
        pos = np.full((2, 2), 77, np.int32)
        cnt = np.full(2, 77, np.int32)
        p = [x.ctypes.data if x is not None else None for x in (a["offs"], a["ids"], a["q"])]
        rc = lib.b200_rank_topk_list_mix(0, a["n_lists"], *p, a["mixing"], 2, None, None, a["k"], pos.ctypes.data,
                                         cnt.ctypes.data, None)
        assert (pos == 77).all() and (cnt == 77).all()
        return rc, lib.b200_rank_last_error().decode()

    assert call(mixing=5) == (_lib.E_INVALID, "b200_rank_topk_list_mix: unknown mixing 5")
    assert call(q=np.array([2, 1], np.int32))[1].endswith("the quotas sum to 3, more than k")
    assert call(ids=np.array([4, 2, -7, 4], np.int32))[0] == _lib.E_INVALID
    assert call(k=0)[0] == _lib.E_INVALID


# ----------------------------------------------------------------------------------------------------------------- plan
@pytest.fixture(scope="module")
def driver():
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    env = dict(os.environ)
    env.pop("CC", None)  # (as in rectools_b200/build.py: the image's CC/CXX may point at an unusable gcc)
    env.pop("CXX", None)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "list_mix_plan_driver")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "list_mix_plan_driver.cpp")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(cases):
            lines = []
            for c in cases:
                c = dict(c)
                for key in ("lists", "ids", "quota", "lens", "offsets"):
                    if key in c and not isinstance(c[key], str):
                        c[key] = ",".join(str(x) for x in c[key])
                lines.append(" ".join(f"{k}={v}" for k, v in c.items()))
            out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
            plans = []
            for ln in out.splitlines():
                head, _, message = ln.partition(" message=")
                p = {}
                for w in head.split():
                    k, v = w.split("=")
                    p[k] = [int(x) for x in v.split(",")] if k in ("bounds", "slots") and v else ([] if k in ("bounds", "slots") else int(v))
                p["message"] = message
                plans.append(p)
            return plans

        yield run


def row_bytes(m, k_out, scratch=0):
    return 8 + 4 * m + 4 * k_out + 4 + scratch


def scratch(slots, n_lists):
    p2 = 1
    while p2 < max(slots, 1):
        p2 *= 2
    return -(-(8 * p2 + 8 * slots + 4 * (2 * n_lists + 1)) // 16) * 16


def test_plan_rows_slots_and_scratch(driver):
    (p, q, r, s, t) = driver([
        dict(lists=[30, 4, 0, 12], quota=[4, 3, 0, 3], k=10, lens=[3, 0, 5]),
        dict(lists=[5], k=10, lens=[1]),
        dict(lists=[30, 4], k=10, lens="-", n_rows=0),
        dict(lists=[0, 0], k=10, lens=[2]),
        dict(lists=[], k=10, lens=[2, 1]),
    ])
    assert (p["error"], p["k_out"], p["n_total"], p["slots"]) == (0, 10, 46, [0, 10, 14, 14, 24])
    assert (p["bounds"], p["max_chunk_rows"], p["max_chunk_nnz"]) == ([0, 3], 3, 8)
    assert p["row_scratch"] == scratch(24, 4) and p["smem"] == 1
    assert (q["k_out"], q["slots"], q["bounds"]) == (5, [0, 5], [0, 1])
    for x in (r, s, t):  # no row, only empty lists, no list: nothing to rank
        assert (x["error"], x["n_chunks"]) == (0, 0)
    assert (s["k_out"], t["k_out"]) == (0, 0)


def test_plan_global_scratch_and_chunks(driver):
    lens = [4, 1, 9, 0, 2, 7]
    sc = scratch(20, 2)
    budget = row_bytes(4, 10, sc) + row_bytes(1, 10, sc)  # the first two rows fit exactly
    (p, q) = driver([dict(lists=[10, 10], k=10, lens=lens, smem=64, budget=budget),
                     dict(lists=[10, 10], k=10, lens=lens, budget=budget)])
    assert p["error"] == 0 and p["smem"] == 0 and p["row_scratch"] == sc
    b = p["bounds"]
    assert b[0] == 0 and b[-1] == len(lens) and b[1] == 2
    for lo, hi in zip(b[:-1], b[1:]):
        assert sum(row_bytes(m, 10, sc) for m in lens[lo:hi]) <= budget
        if hi < len(lens):
            assert sum(row_bytes(m, 10, sc) for m in lens[lo : hi + 1]) > budget
    assert q["smem"] == 1 and q["bounds"] == [0, len(lens)]  # in shared memory the scratch costs no chunk bytes
    # 200 lists x k = 1000: more scratch than shared memory holds
    (big,) = driver([dict(lists=[2000] * 200, k=1000, lens=[3])])
    assert big["smem"] == 0 and big["row_scratch"] == scratch(200_000, 200) and big["error"] == 0


def test_plan_row_cap_hook(driver):
    plans = driver([
        dict(lists=[50], k=5, lens=[1] * 10, B200_LIST_CHUNK_ROWS=3),
        dict(lists=[50], k=5, lens=[1] * 10, B200_LIST_CHUNK_ROWS=1),
        dict(lists=[50], k=5, lens=[1] * 10),
    ])
    assert plans[0]["bounds"] == [0, 3, 6, 9, 10] and plans[0]["max_chunk_rows"] == 3
    assert plans[1]["bounds"] == list(range(11))
    assert plans[2]["bounds"] == [0, 10]


def test_plan_refusals(driver):
    cases = [
        (dict(lists=[5], k=1, lens=[1], n_lists=-1), -1, "n_lists and n_rows must be >= 0"),
        (dict(lists=[5], k=1, lens=[1], n_rows=-1), -1, "n_lists and n_rows must be >= 0"),
        (dict(lists=[5], k=0, lens=[1]), -1, "k must be >= 1"),
        (dict(lists=[5], k=1, lens=[1], mixing=2), -1, "unknown mixing 2"),
        (dict(lists=[5], k=1, lens=[1], null_offsets=1), -1, "list_offsets is NULL"),
        (dict(lists=[5], k=1, lens=[1], null_quota=1), -1, "quota is NULL"),
        (dict(offsets=[1, 5], k=1, lens=[1]), -1, "list_offsets[0] = 1, not 0"),
        (dict(offsets=[0, 5, 3], k=1, lens=[1]), -1, "list_offsets is not monotone at list 1"),
        (dict(offsets=[0, 2**31], k=1, lens=[1]), -1, "more than 2^31 - 1 ids"),
        (dict(lists=[5], k=1, lens=[1], null_ids=1), -1, "list_ids is NULL"),
        (dict(lists=[3], ids=[0, -4, 2], k=1, lens=[1]), -1, "list_ids[1] = -4 is negative"),
        (dict(lists=[3, 3], quota=[1, -1], k=1, lens=[1]), -1, "quota[1] = -1 is negative"),
        (dict(lists=[3, 3], quota=[2, 1], k=2, lens=[1]), -1, "the quotas sum to 3, more than k"),
        (dict(lists=[5], k=1, lens=[1], null_counts=1), -1, "out_counts is NULL"),
        (dict(lists=[5], k=1, lens=[1], null_pos=1), -1, "out_pos is NULL"),
        (dict(lists=[5], k=1, lens=[1, 2], base=3), -1, "csr_indptr[0] = 3, not 0"),
        (dict(lists=[5], k=1, lens=[1, -1, 2]), -1, "csr_indptr is not monotone at row 1"),
        (dict(lists=[5], k=1, lens=[1, 2], null_indices=1), -1, "csr_indices is NULL"),
        (dict(lists=[5, 5], k=3, lens=[1, 40, 2], budget=row_bytes(39, 3)), -3, "row 1 (40 viewed ids, 6 entry slots) needs"),
    ]
    plans = driver([c for c, _, _ in cases])
    for (c, code, msg), p in zip(cases, plans):
        assert p["error"] == code, (c, p)
        assert p["message"].startswith("b200_rank_topk_list_mix: ") and msg in p["message"], (c, p)
        assert p["bounds"] == [] and p["slots"] == []
    # not refused: no list at all with NULL arrays, quotas summing below k, an empty list's NULL ids
    ok = driver([dict(lists=[], k=1, lens=[1], null_offsets=1, null_quota=1, null_ids=1, null_pos=1),
                 dict(lists=[3, 3], quota=[0, 1], k=4, lens=[1]),
                 dict(lists=[0], k=1, lens=[0], null_ids=1, null_pos=1, null_indices=1)])
    assert [p["error"] for p in ok] == [0, 0, 0]


# ------------------------------------------------------------------------------------------- the restatement vs reference
@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    from rectools.models import PopularInCategoryModel

    yield PopularInCategoryModel
    stage_reference.remove_from_path(added)


def _fit(model, ds):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # n_categories above the category count
        return model.fit(ds)


@needs_ref
@pytest.mark.parametrize("n_categories", [1, 2, 5, 40])
def test_restatement_matches_reference_u2i(ref, n_categories):
    from tests.popular_in_category_cases import category_dataset, in_category_settings

    ds = category_dataset(n_users=25, n_items=45, n_categories=n_categories, seed=n_categories, idle_users=2)
    users = np.arange(ds.user_id_map.size)  # the idle users (nothing viewed) and the heavy ones (everything viewed)
    csr = ds.get_user_item_matrix(include_weights=False)
    for i, kw in enumerate(in_category_settings(n_categories)):
        model = _fit(ref(**kw), ds)
        cases = [(1, True, None), (7, True, None), (45, True, None), (60, False, None), (4, True, np.arange(0, 45, 2)),
                 (9, False, np.arange(0, 45, 3))]
        for k, fv, wl in cases[i % 2 :: 2] if i % 3 else cases:
            expected = model._recommend_u2i(users, ds, k, fv, wl)  # pylint: disable=protected-access
            got = recommend_in_category_u2i_np(model, users, csr, k, fv, wl)
            for e, g in zip(expected, got):
                np.testing.assert_array_equal(np.asarray(e), g, err_msg=f"{kw} k={k} filter_viewed={fv}")


# ---------------------------------------------------------------------------------------------- host logic (stand-in lib)
class RecordingLib:
    """`b200_rank_topk_list_mix` and `b200_rank_topk_list` computed by the numpy restatements; records the arguments of
    the mixing calls."""

    def __init__(self):
        self.calls = []
        self.list_calls = 0

    @staticmethod
    def _arr(p, ctype, n, dtype):
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(ctype)), (n,)).copy() if n and p else np.zeros(0, dtype)

    def b200_rank_topk_list_mix(self, device, n_lists, offs_p, ids_p, quota_p, mixing, n_rows, indptr_p, indices_p, k,
                                out_pos, out_counts, stats):
        offs = self._arr(offs_p, C.c_int64, n_lists + 1, np.int64)
        ids = self._arr(ids_p, C.c_int32, int(offs[-1]) if n_lists else 0, np.int32)
        quota = self._arr(quota_p, C.c_int32, n_lists, np.int32)
        indptr = self._arr(indptr_p, C.c_int64, n_rows + 1, np.int64) if indptr_p else None
        indices = self._arr(indices_p, C.c_int32, int(indptr[-1]) if indptr is not None else 0, np.int32)
        lists = [ids[offs[c] : offs[c + 1]] for c in range(n_lists)]
        self.calls.append(dict(device=device, lists=lists, quota=quota, mixing=mixing, n_rows=n_rows, indptr=indptr,
                               indices=indices, k=k))
        pos, cnt = rank_list_mix_np(lists, quota, ("rotate", "group")[mixing], indptr, indices, n_rows, k)
        if pos.size:
            np.ctypeslib.as_array(C.cast(out_pos, C.POINTER(C.c_int32)), (pos.size,))[:] = pos.reshape(-1)
        if n_rows:
            np.ctypeslib.as_array(C.cast(out_counts, C.POINTER(C.c_int32)), (n_rows,))[:] = cnt
        stats._obj.path = 8  # pylint: disable=protected-access
        return 0

    def b200_rank_topk_list(self, device, n_list, list_p, n_rows, indptr_p, indices_p, k, out_pos, out_counts, stats):
        self.list_calls += 1
        lst = self._arr(list_p, C.c_int32, n_list, np.int32)
        indptr = self._arr(indptr_p, C.c_int64, n_rows + 1, np.int64) if indptr_p else None
        indices = self._arr(indices_p, C.c_int32, int(indptr[-1]) if indptr is not None else 0, np.int32)
        pos, cnt = rank_list_np(lst, indptr, indices, n_rows, k)
        if pos.size:
            np.ctypeslib.as_array(C.cast(out_pos, C.POINTER(C.c_int32)), (pos.size,))[:] = pos.reshape(-1)
        if n_rows:
            np.ctypeslib.as_array(C.cast(out_counts, C.POINTER(C.c_int32)), (n_rows,))[:] = cnt
        stats._obj.path = 7  # pylint: disable=protected-access
        return 0

    def b200_rank_last_error(self):
        return b""


@pytest.fixture()
def lib(monkeypatch):
    from rectools_b200 import _lib

    rec = RecordingLib()
    monkeypatch.setattr(_lib, "_LIB", rec)
    yield rec


def test_rank_list_mix_hands_over_and_pads(lib):
    from rectools_b200 import rank_list_mix
    from scipy import sparse

    viewed = sparse.csr_matrix((np.ones(3), ([0, 0, 1], [7, 2, 4])), shape=(2, 12))
    viewed.has_sorted_indices = False
    stats = {}
    pos, cnt = rank_list_mix([np.array([4, 2], np.int64), [7, 4]], [1, 1], "rotate", viewed, 2, device=3, stats=stats)
    (call,) = lib.calls
    assert (call["device"], call["mixing"], call["n_rows"], call["k"]) == (3, 0, 2, 2)
    np.testing.assert_array_equal(call["quota"], [1, 1])
    np.testing.assert_array_equal(call["indices"], [2, 7, 4])  # sorted within the rows on a copy
    assert pos.dtype == np.int32 and cnt.dtype == np.int32 and stats["path"] == 8
    np.testing.assert_array_equal(pos, [[0, -1], [1, 2]])
    np.testing.assert_array_equal(cnt, [1, 2])
    pos, cnt = rank_list_mix([[5, 6, 7]], [0], "group", None, 10**12, n_rows=2)
    assert lib.calls[-1]["k"] == 2**31 - 1 and lib.calls[-1]["mixing"] == 1 and lib.calls[-1]["indptr"] is None
    np.testing.assert_array_equal(pos, [[0, 1, 2], [0, 1, 2]])


def test_rank_list_mix_refuses_bad_arguments():
    from rectools_b200 import rank_list_mix

    with pytest.raises(ValueError, match="positive int"):
        rank_list_mix([[1]], [1], "rotate", None, 0, n_rows=1)
    with pytest.raises(ValueError, match="mixing"):
        rank_list_mix([[1]], [1], "shuffle", None, 1, n_rows=1)
    with pytest.raises(ValueError, match="quotas for"):
        rank_list_mix([[1], [2]], [1], "rotate", None, 1, n_rows=1)
    with pytest.raises(ValueError, match="sum to at most k"):
        rank_list_mix([[1], [2]], [1, 1], "rotate", None, 1, n_rows=1)
    with pytest.raises(ValueError, match=r"\[0, 2\^31 - 1\]"):
        rank_list_mix([[1, 2**31]], [1], "rotate", None, 1, n_rows=1)
    with pytest.raises(ValueError, match="sum to at most k"):  # k is capped at 2^31 - 1; the quota would wrap in int32
        rank_list_mix([[1]], [2**32 + 1], "rotate", None, 10**12, n_rows=1)
    with pytest.raises(TypeError, match="quota must be integers"):
        rank_list_mix([[1]], [0.5], "rotate", None, 1, n_rows=1)


@needs_ref
def test_recommend_u2i_hands_over_and_delegates(lib, ref):
    from rectools_b200.popular import popular_in_category_recommend_u2i
    from tests.popular_in_category_cases import category_dataset

    ds = category_dataset(n_users=30, n_categories=4, seed=3)
    model = _fit(ref(category_feature="category", mixing_strategy="group"), ds)
    users = np.array([9, 0, 21, 4], dtype=np.int64)
    expected = model._recommend_u2i(users, ds, 6, True, None)  # pylint: disable=protected-access
    got = popular_in_category_recommend_u2i(model, users, ds, 6, True, None, device=2)
    call = lib.calls[-1]
    assert (call["device"], call["k"], call["n_rows"], call["mixing"]) == (2, 6, 4, 1)
    np.testing.assert_array_equal(call["quota"], model._get_num_recs_for_each_category(6).values)  # pylint: disable=protected-access
    assert len(call["lists"]) == len(model.models)
    for e, g in zip(expected, got):
        np.testing.assert_array_equal(g, np.asarray(e))
    assert got[0].dtype == users.dtype and got[2].dtype == np.float64
    # filter_viewed=False: one row with nothing viewed, tiled
    got = popular_in_category_recommend_u2i(model, users, ds, 6, False, None)
    assert lib.calls[-1]["n_rows"] == 1 and lib.calls[-1]["indptr"] is None
    for e, g in zip(model._recommend_u2i(users, ds, 6, False, None), got):  # pylint: disable=protected-access
        np.testing.assert_array_equal(g, np.asarray(e))
    # handed to the stock method: repeated users, ids beyond int32, bad quotas, no category model
    n_calls = len(lib.calls)
    rep = np.array([3, 5, 3], dtype=np.int64)
    for e, g in zip(model._recommend_u2i(rep, ds, 4, True, None), popular_in_category_recommend_u2i(model, rep, ds, 4, True, None)):  # pylint: disable=protected-access
        np.testing.assert_array_equal(np.asarray(g), np.asarray(e))
    first = next(iter(model.models.values()))
    items, scores = first.popularity_list
    first.popularity_list = (np.concatenate(([2**33], items)), np.concatenate(([99.0], scores)))
    for e, g in zip(model._recommend_u2i(users, ds, 4, True, None), popular_in_category_recommend_u2i(model, users, ds, 4, True, None)):  # pylint: disable=protected-access
        np.testing.assert_array_equal(np.asarray(g), np.asarray(e))
    first.popularity_list = (items, scores)
    stock_quota = model._get_num_recs_for_each_category  # pylint: disable=protected-access
    for bad in (lambda k: stock_quota(k) * 2, lambda k: stock_quota(k) - 2, lambda k: stock_quota(k) + 0.5):
        model._get_num_recs_for_each_category = bad  # quotas summing above k, negative, not integers
        for e, g in zip(model._recommend_u2i(users, ds, 4, True, None), popular_in_category_recommend_u2i(model, users, ds, 4, True, None)):  # pylint: disable=protected-access
            np.testing.assert_array_equal(np.asarray(g), np.asarray(e))
    del model._get_num_recs_for_each_category
    assert len(lib.calls) == n_calls
    empty = _fit(ref(category_feature="category"), ds)
    empty.models, empty.category_scores = {}, empty.category_scores.iloc[:0]
    with pytest.raises(ValueError) as stock_error:
        empty._recommend_u2i(users, ds, 4, True, None)  # pylint: disable=protected-access
    with pytest.raises(ValueError, match=re.escape(str(stock_error.value))):
        popular_in_category_recommend_u2i(empty, users, ds, 4, True, None)
    assert len(lib.calls) == n_calls


@needs_ref
def test_install_rebinds_and_uninstall_restores(lib, ref):
    import pandas as pd
    import rectools_b200 as rb
    from tests.popular_in_category_cases import category_dataset

    original = ref.__dict__["_recommend_u2i"]
    ds = category_dataset(n_users=30, seed=4)
    model = _fit(ref(category_feature="category"), ds)
    users = ds.user_id_map.external_ids[:8]
    expected = model.recommend(users, ds, 5, True)
    try:
        for kw in ({}, {"popular": True}):  # neither touches PopularInCategoryModel
            rb.install(**kw)
            assert ref.__dict__["_recommend_u2i"] is original
            rb.uninstall()
        assert not lib.calls
        rb.install(device=[3, 1], popular_in_category=True)
        assert ref.__dict__["_recommend_u2i"] is not original
        pd.testing.assert_frame_equal(model.recommend(users, ds, 5, True), expected)
        assert lib.calls[-1]["device"] == 3  # the home device of a group
    finally:
        rb.uninstall()
    assert ref.__dict__["_recommend_u2i"] is original


@needs_ref
@pytest.mark.parametrize("n_categories", [1, 2, 5, 40])
def test_frames_equal_stock(lib, ref, n_categories):
    import pandas as pd
    import rectools_b200 as rb
    from tests.popular_in_category_cases import category_dataset, in_category_settings

    ds = category_dataset(n_users=40, n_items=50, n_categories=n_categories, seed=10 + n_categories, idle_users=2)
    ext_users, ext_items = ds.user_id_map.external_ids, ds.item_id_map.external_ids
    cases = []
    for fv in (True, False):
        cases += [(ext_users, 5, fv, None), (np.concatenate((ext_users[9:2:-1], [999_999])), 1, fv, None),
                  (ext_users[:10], len(ext_items) + 5, fv, None), (ext_users, 4, fv, ext_items[::3]),
                  (ext_users[2:4], 3, fv, ext_items[:4]),  # heavy users among items they viewed: empty
                  (ext_users, 3, fv, ext_items[-3:])]  # items nobody viewed: every list empty unless add_cold
    for kw in in_category_settings(n_categories):
        model = _fit(ref(**kw), ds)
        expected = [model.recommend(u, ds, k, fv, items_to_recommend=wl) for u, k, fv, wl in cases]
        rb.install(popular_in_category=True)
        try:
            for (u, k, fv, wl), exp in zip(cases, expected):
                pd.testing.assert_frame_equal(model.recommend(u, ds, k, fv, items_to_recommend=wl), exp,
                                              obj=f"{kw} k={k} filter_viewed={fv}")
        finally:
            rb.uninstall()
    assert lib.calls

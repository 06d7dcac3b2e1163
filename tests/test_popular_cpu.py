"""CPU: popularity lists (engine path 7, `b200_rank_topk_list`, `rectools_b200.popular`) up to where a GPU is needed.

- the export is declared, exported and bound, and the ABI stays 6;
- tests/list_plan_driver.cpp prints `plan_list` (rectools_b200/csrc/list_plan.h): chunk bounds within the byte budget, the
  B200_LIST_CHUNK_ROWS cap, and every refusal;
- the numpy restatement (tests/popular_oracle.py) against the unmodified reference's `PopularModel._recommend_for_user`
  loop;
- the host logic with the library replaced by a recording stand-in: the arguments handed over, the flattening and the
  dtypes, `install(popular=True)` / `uninstall()`, and `PopularModel.recommend` / `PopularInCategoryModel.recommend`
  frames equal to the stock methods'."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests.popular_oracle import rank_list_np, recommend_u2i_np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_export_declared_exported_and_bound():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    assert re.search(r"\bint b200_rank_topk_list\s*\(", header)
    assert re.search(r"7 = a shared list minus viewed ids \(b200_rank_topk_list\)", header)
    assert "b200_rank_topk_list" in _lib.EXPORTS
    assert "#define B200_RANK_ABI_VERSION 6" in header and _lib.ABI_VERSION == 6
    assert not any(e.startswith("b200_rank_group_") and "list" in e for e in _lib.EXPORTS)
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = C.CDLL(_lib.LIB_PATH)
    assert lib.b200_rank_topk_list is not None
    assert _lib.load().b200_rank_topk_list.argtypes is not None


def test_host_refusals_leave_outputs_untouched():
    """Refusals are decided before the device is touched, so they run here (the library needs no GPU to load)."""
    from rectools_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = _lib.load()
    lst = np.array([4, 2, 7], np.int32)
    indptr = np.array([0, 2, 3], np.int64)
    indices = np.array([2, 7, 4], np.int32)

    def call(n_list=3, lst_=lst, n_rows=2, ip=indptr, ix=indices, k=2):
        pos = np.full((2, 2), 77, np.int32)
        cnt = np.full(2, 77, np.int32)
        rc = lib.b200_rank_topk_list(0, n_list, lst_.ctypes.data if lst_ is not None else None, n_rows,
                                     ip.ctypes.data if ip is not None else None, ix.ctypes.data if ix is not None else None, k,
                                     pos.ctypes.data, cnt.ctypes.data, None)
        assert (pos == 77).all() and (cnt == 77).all()
        return rc, lib.b200_rank_last_error().decode()

    assert call(n_list=-1)[0] == _lib.E_INVALID
    assert call(n_rows=-1)[0] == _lib.E_INVALID
    assert call(k=0)[0] == _lib.E_INVALID
    assert call(n_list=2**31)[0] == _lib.E_INVALID
    assert call(lst_=None)[0] == _lib.E_INVALID
    assert call(lst_=np.array([4, -2, 7], np.int32))[0] == _lib.E_INVALID
    assert call(ip=np.array([1, 2, 3], np.int64))[0] == _lib.E_INVALID
    assert call(ip=np.array([0, 3, 2], np.int64))[0] == _lib.E_INVALID
    assert call(ix=None)[0] == _lib.E_INVALID
    rc, msg = call(ix=np.array([7, 2, 4], np.int32))
    assert rc == _lib.E_INVALID and "row 0: viewed ids are not ascending" in msg


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
        exe = os.path.join(tmp, "list_plan_driver")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "list_plan_driver.cpp")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(cases):
            lines = []
            for c in cases:
                c = dict(c)
                for key in ("lens", "ids", "list"):
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
                    p[k] = [int(x) for x in v.split(",")] if k == "bounds" and v else ([] if k == "bounds" else int(v))
                p["message"] = message
                plans.append(p)
            return plans

        yield run


def row_bytes(m, k_out):
    return 8 + 4 * m + 4 * k_out + 4


def test_plan_one_chunk_and_k_out(driver):
    (p, q, r, s) = driver([
        dict(n_list=100, k=10, lens=[3, 0, 5]),
        dict(n_list=4, k=10, lens=[1, 1]),
        dict(n_list=100, k=10, lens="-", n_rows=5),
        dict(n_list=0, k=10, lens=[2]),
    ])
    assert (p["error"], p["k_out"], p["bounds"], p["max_chunk_rows"], p["max_chunk_nnz"]) == (0, 10, [0, 3], 3, 8)
    assert (q["k_out"], q["bounds"]) == (4, [0, 2])
    assert (r["error"], r["bounds"], r["max_chunk_nnz"]) == (0, [0, 5], 0)
    assert (s["error"], s["k_out"], s["n_chunks"]) == (0, 0, 0)  # an empty list: nothing to rank


def test_plan_chunks_within_the_budget(driver):
    lens = [4, 1, 9, 0, 2, 7]
    budget = row_bytes(4, 10) + row_bytes(1, 10)  # the first two rows fit exactly
    (p,) = driver([dict(n_list=100, k=10, lens=lens, budget=budget)])
    assert p["error"] == 0
    b = p["bounds"]
    assert b[0] == 0 and b[-1] == len(lens) and b[1] == 2
    for lo, hi in zip(b[:-1], b[1:]):
        assert sum(row_bytes(m, 10) for m in lens[lo:hi]) <= budget
        if hi < len(lens):  # a chunk closes only when the next row does not fit
            assert sum(row_bytes(m, 10) for m in lens[lo : hi + 1]) > budget
    assert p["max_chunk_nnz"] == max(sum(lens[lo:hi]) for lo, hi in zip(b[:-1], b[1:]))


def test_plan_row_cap_hook(driver):
    plans = driver([
        dict(n_list=50, k=5, lens=[1] * 10, B200_LIST_CHUNK_ROWS=3),
        dict(n_list=50, k=5, lens=[1] * 10, B200_LIST_CHUNK_ROWS=1),
        dict(n_list=50, k=5, lens=[1] * 10, B200_LIST_CHUNK_ROWS=0),
        dict(n_list=50, k=5, lens=[1] * 10),  # the hook of the previous lines is gone
    ])
    assert plans[0]["bounds"] == [0, 3, 6, 9, 10] and plans[0]["max_chunk_rows"] == 3
    assert plans[1]["bounds"] == list(range(11))
    assert plans[2]["bounds"] == [0, 10] and plans[3]["bounds"] == [0, 10]


def test_plan_refusals(driver):
    cases = [
        (dict(n_list=-1, k=1, lens=[1]), -1, "n_list and n_rows must be >= 0"),
        (dict(n_list=5, k=1, lens=[1], n_rows=-1), -1, "n_list and n_rows must be >= 0"),
        (dict(n_list=5, k=0, lens=[1]), -1, "k must be >= 1"),
        (dict(n_list=2**31, k=1, lens=[1]), -1, "n_list exceeds 2^31 - 1"),
        (dict(n_list=5, k=1, lens=[1], null_list=1), -1, "list_ids is NULL"),
        (dict(n_list=5, k=1, lens=[1], null_counts=1), -1, "out_counts is NULL"),
        (dict(n_list=5, k=1, lens=[1], null_pos=1), -1, "out_pos is NULL"),
        (dict(n_list=3, k=1, lens=[1], list=[0, -4, 2]), -1, "list_ids[1] = -4 is negative"),
        (dict(n_list=5, k=1, lens=[1, 2], base=3), -1, "csr_indptr[0] = 3, not 0"),
        (dict(n_list=5, k=1, lens=[1, -1, 2]), -1, "csr_indptr is not monotone at row 1"),
        (dict(n_list=5, k=1, lens=[1, 2], null_indices=1), -1, "csr_indices is NULL"),
        (dict(n_list=5, k=1, lens=[1, 3], ids=[9, 4, 2, 6]), -1, "row 1: viewed ids are not ascending"),
        (dict(n_list=5, k=3, lens=[1, 40, 2], budget=row_bytes(39, 3)), -3, "row 1 (40 viewed ids, k_out = 3) needs"),
    ]
    plans = driver([c for c, _, _ in cases])
    for (c, code, msg), p in zip(cases, plans):
        assert p["error"] == code, (c, p)
        assert p["message"].startswith("b200_rank_topk_list: ") and msg in p["message"], (c, p)
        assert p["bounds"] == []
    # not refused: NULL out_pos with k_out = 0, NULL indices with no entry, repeats and negative viewed ids
    ok = driver([
        dict(n_list=0, k=1, lens=[1], null_pos=1, null_list=1),
        dict(n_list=5, k=1, lens=[0, 0], null_indices=1),
        dict(n_list=5, k=1, lens=[4], ids=[-3, 1, 1, 9]),
        dict(n_list=5, k=1, lens=[], n_rows=0, null_counts=1, null_pos=1),
    ])
    assert [p["error"] for p in ok] == [0, 0, 0, 0]


# ------------------------------------------------------------------------------------------- the restatement vs reference
@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    from rectools.models.popular import PopularModel

    yield PopularModel
    stage_reference.remove_from_path(added)


def _reference_rows(PopularModel, list_ids, scores, rows, k):
    """The reference's per-user step, `_recommend_for_user`, for each viewed row (None: filter_viewed=False)."""
    out = []
    for viewed in rows:
        ids, sc = PopularModel._recommend_for_user(k, (list_ids, scores), viewed)  # pylint: disable=protected-access
        out.append((np.asarray(ids), np.asarray(sc)))
    return out


def _list_cases():
    rng = np.random.default_rng(5)
    base = rng.permutation(60).astype(np.int64)
    yield "plain", base, [np.sort(rng.choice(60, 7, replace=False)) for _ in range(6)], 5
    yield "inverse", base[::-1].copy(), [np.sort(rng.choice(60, 12, replace=False)) for _ in range(6)], 10
    yield "add_cold_tail", np.concatenate((base[:40], np.arange(60, 70))), [np.arange(0, 70, 2)], 20
    yield "whitelist", np.sort(base[base % 3 == 0])[::-1].copy(), [np.sort(rng.choice(60, 20, replace=False)) for _ in range(4)], 6
    yield "everything_viewed", base[:10], [np.sort(base[:10]), np.arange(60)], 4
    yield "viewed_outside_list", base[:10], [np.arange(100, 130), np.array([-5, 1000])], 3
    yield "k_above_list", base[:8], [np.sort(base[:3]), np.array([], np.int64)], 50
    yield "empty_list", base[:0], [np.array([1, 2]), np.array([], np.int64)], 3
    yield "no_views", base, [np.array([], np.int64)] * 3, 7
    yield "first_k_viewed", base, [np.sort(base[:5])], 5
    yield "repeated_viewed", base, [np.sort(np.repeat(base[:4], 3))], 5
    yield "repeated_list_ids", np.array([3, 3, 3, 8, 1, 3]), [np.array([3]), np.array([3, 3]), np.array([8])], 1


@needs_ref
def test_restatement_matches_reference_for_user(ref):
    for name, list_ids, rows, k in _list_cases():
        scores = np.linspace(9.0, 1.0, len(list_ids))
        indptr = np.concatenate(([0], np.cumsum([len(r) for r in rows]))).astype(np.int64)
        indices = np.concatenate(rows).astype(np.int64) if rows else np.zeros(0, np.int64)
        pos, cnt = rank_list_np(list_ids, indptr, indices, len(rows), k)
        assert pos.shape == (len(rows), min(k, len(list_ids))), name
        for r, (ids, sc) in enumerate(_reference_rows(ref, list_ids, scores, rows, k)):
            got = pos[r, : cnt[r]]
            assert (pos[r, cnt[r] :] == -1).all(), name
            np.testing.assert_array_equal(list_ids[got], ids, err_msg=name)
            np.testing.assert_array_equal(scores[got], sc, err_msg=name)
        # nothing viewed: the list's first k for every row
        pos, cnt = rank_list_np(list_ids, None, None, 2, k)
        for ids, _ in _reference_rows(ref, list_ids, scores, [None, None], k):
            np.testing.assert_array_equal(list_ids[pos[0, : cnt[0]]], ids, err_msg=name)


@needs_ref
def test_restatement_matches_reference_u2i(ref):
    from tests.popular_cases import popular_dataset, popular_settings

    ds = popular_dataset()
    users = ds.user_id_map.convert_to_internal(ds.user_id_map.external_ids)
    for kw in list(popular_settings())[:8]:
        model = ref(**kw).fit(ds)
        for k, fv, wl in ((5, True, None), (40, True, None), (3, False, None), (4, True, np.arange(0, 40, 3))):
            items, scores = model._get_filtered_popularity_list(wl)  # pylint: disable=protected-access
            expected = model._recommend_u2i(users, ds, k, fv, wl)  # pylint: disable=protected-access
            got = recommend_u2i_np(items, scores, users, ds.get_user_item_matrix(include_weights=False), k, fv)
            for e, g in zip(expected, got):
                np.testing.assert_array_equal(np.asarray(e), g)


# ---------------------------------------------------------------------------------------------- host logic (stand-in lib)
class RecordingLib:
    """`b200_rank_topk_list` computed by the numpy restatement; records the arguments it was handed."""

    def __init__(self):
        self.calls = []

    def b200_rank_topk_list(self, device, n_list, list_p, n_rows, indptr_p, indices_p, k, out_pos, out_counts, stats):
        def arr(p, ctype, n, dtype):
            return np.ctypeslib.as_array(C.cast(p, C.POINTER(ctype)), (n,)).copy() if n and p else np.zeros(0, dtype)

        lst = arr(list_p, C.c_int32, n_list, np.int32)
        indptr = arr(indptr_p, C.c_int64, n_rows + 1, np.int64) if indptr_p else None
        indices = arr(indices_p, C.c_int32, int(indptr[-1]) if indptr is not None else 0, np.int32)
        self.calls.append(dict(device=device, n_list=n_list, list=lst, n_rows=n_rows, indptr=indptr, indices=indices, k=k))
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


def test_rank_list_hands_over_and_pads(lib):
    from rectools_b200 import rank_list

    viewed = sparse.csr_matrix((np.ones(4), ([0, 0, 2, 2], [5, 3, 9, 1])), shape=(3, 12))
    viewed.has_sorted_indices = False
    stats = {}
    pos, cnt = rank_list(np.array([3, 9, 4, 1, 5], np.int64), viewed, 3, device=2, stats=stats)
    (call,) = lib.calls
    assert (call["device"], call["n_list"], call["n_rows"], call["k"]) == (2, 5, 3, 3)
    np.testing.assert_array_equal(call["list"], [3, 9, 4, 1, 5])
    np.testing.assert_array_equal(call["indptr"], [0, 2, 2, 4])
    np.testing.assert_array_equal(call["indices"], [3, 5, 1, 9])  # sorted within the rows on a copy
    assert pos.dtype == np.int32 and cnt.dtype == np.int32 and stats["path"] == 7
    np.testing.assert_array_equal(pos, [[1, 2, 3], [0, 1, 2], [0, 2, 4]])
    np.testing.assert_array_equal(cnt, [3, 3, 3])
    # a row slice of a larger CSR is rebased; None means nothing viewed; k is clamped to the list
    pos, cnt = rank_list([7, 8], (np.array([2, 3, 3]), np.array([0, 0, 8, 0])), 10**12)
    np.testing.assert_array_equal(lib.calls[-1]["indptr"], [0, 1, 1])
    np.testing.assert_array_equal(pos, [[0, -1], [0, 1]])
    assert lib.calls[-1]["k"] == 2**31 - 1
    pos, cnt = rank_list([7, 8], None, 1, n_rows=3)
    assert lib.calls[-1]["indptr"] is None and pos.shape == (3, 1) and (cnt == 1).all()


def test_rank_list_refuses_bad_arguments():
    from rectools_b200 import rank_list

    with pytest.raises(ValueError, match="positive int"):
        rank_list([1], None, 0, n_rows=1)
    with pytest.raises(ValueError, match="n_rows"):
        rank_list([1], None, 1)
    with pytest.raises(ValueError, match=r"\[0, 2\^31 - 1\]"):
        rank_list([1, 2**31], None, 1, n_rows=1)
    with pytest.raises(TypeError, match="integers"):
        rank_list([1.5], None, 1, n_rows=1)
    with pytest.raises(ValueError, match="fit int32"):
        rank_list([1], (np.array([0, 1]), np.array([2**40])), 1)


def _same_outcome(got_fn, expected_fn):
    """The same frame, or the same exception type and message."""
    import pandas as pd

    try:
        expected = expected_fn()
    except Exception as e:  # pylint: disable=broad-except
        with pytest.raises(type(e), match=re.escape(str(e))):
            got_fn()
        return None
    got = got_fn()
    pd.testing.assert_frame_equal(got, expected)
    return got


@needs_ref
def test_popular_recommend_u2i_flattening_and_dtypes(lib, ref):
    from rectools_b200.popular import popular_recommend_u2i
    from tests.popular_cases import popular_dataset

    ds = popular_dataset()
    model = ref(popularity="sum_weight").fit(ds)
    users = np.array([5, 0, 9, 5], dtype=np.int64)
    expected = model._recommend_u2i(users, ds, 6, True, None)  # pylint: disable=protected-access
    got = popular_recommend_u2i(model, users, ds, 6, True, None, device=1)
    assert lib.calls[-1]["device"] == 1 and lib.calls[-1]["k"] == 6 and lib.calls[-1]["n_rows"] == 4
    for e, g in zip(expected, got):
        e = np.asarray(e)
        assert isinstance(g, np.ndarray) and g.dtype == e.dtype
        np.testing.assert_array_equal(g, e)
    # filter_viewed=False: tiled on the host, no call
    n_calls = len(lib.calls)
    for e, g in zip(model._recommend_u2i(users, ds, 6, False, None), popular_recommend_u2i(model, users, ds, 6, False, None)):  # pylint: disable=protected-access
        np.testing.assert_array_equal(g, np.asarray(e))
        assert g.dtype == np.asarray(e).dtype
    assert len(lib.calls) == n_calls
    # an empty result is three empty lists, as the reference returns it
    heavy = np.array([0, 1], dtype=np.int64)
    assert model._recommend_u2i(heavy, ds, 3, True, np.arange(4)) == ([], [], [])  # pylint: disable=protected-access
    assert popular_recommend_u2i(model, heavy, ds, 3, True, np.arange(4)) == ([], [], [])
    assert popular_recommend_u2i(model, heavy[:0], ds, 3, True, None) == ([], [], [])
    assert popular_recommend_u2i(model, heavy[:0], ds, 3, False, None) == ([], [], [])


@needs_ref
def test_ids_beyond_int32_go_to_the_stock_method(lib, ref):
    from rectools_b200.popular import popular_recommend_u2i
    from tests.popular_cases import popular_dataset

    ds = popular_dataset()
    model = ref().fit(ds)
    items, scores = model.popularity_list
    model.popularity_list = (np.concatenate(([2**33], items)), np.concatenate(([99.0], scores)))
    users = np.arange(4, dtype=np.int64)
    expected = model._recommend_u2i(users, ds, 4, True, None)  # pylint: disable=protected-access
    got = popular_recommend_u2i(model, users, ds, 4, True, None)
    assert lib.calls == []
    for e, g in zip(expected, got):
        np.testing.assert_array_equal(np.asarray(g), np.asarray(e))


@needs_ref
def test_install_popular_rebinds_and_uninstall_restores(lib, ref):
    import rectools_b200 as rb
    from tests.popular_cases import popular_dataset

    original = ref.__dict__["_recommend_u2i"]
    ds = popular_dataset()
    model = ref().fit(ds)
    users = ds.user_id_map.external_ids[:6]
    expected = model.recommend(users, ds, 4, True)
    try:
        rb.install()  # the default leaves PopularModel alone
        assert ref.__dict__["_recommend_u2i"] is original
        rb.uninstall()
        rb.install(device=[3, 1], popular=True)
        assert ref.__dict__["_recommend_u2i"] is not original
        _same_outcome(lambda: model.recommend(users, ds, 4, True), lambda: expected)
        assert lib.calls[-1]["device"] == 3  # the home device of a group
    finally:
        rb.uninstall()
    assert ref.__dict__["_recommend_u2i"] is original


def _compare_models(make_models, ds, lib):
    """Every recommend case of tests/popular_cases.py: the stock frame, then the frame with install(popular=True)."""
    import rectools_b200 as rb
    from tests.popular_cases import recommend_cases

    cases = list(recommend_cases(ds))
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
                import pandas as pd

                pd.testing.assert_frame_equal(model.recommend(users, ds, k, fv, items_to_recommend=wl), exp,
                                              obj=f"{model.__class__.__name__} k={k} filter_viewed={fv}")
        finally:
            rb.uninstall()
    assert lib.calls  # the stand-in ranked the filtered calls


@needs_ref
def test_popular_model_frames_equal_stock(lib, ref):
    from tests.popular_cases import popular_dataset, popular_settings

    ds = popular_dataset()
    _compare_models(lambda: (ref(**kw) for kw in popular_settings()), ds, lib)


@needs_ref
def test_popular_in_category_frames_equal_stock(lib, ref):
    from rectools.models import PopularInCategoryModel
    from tests.popular_cases import category_settings, popular_dataset

    ds = popular_dataset(n_users=40, seed=1)
    _compare_models(lambda: (PopularInCategoryModel(**kw) for kw in category_settings()), ds, lib)
    # popularity kinds and add_cold / inverse through the category models
    _compare_models(lambda: (PopularInCategoryModel(category_feature="category", popularity=p, add_cold=True, inverse=True)
                             for p in ("n_interactions", "mean_weight")), ds, lib)


@needs_ref
def test_popular_in_category_empty_result_frames_equal_stock(lib, ref):
    """Every category model returns an empty triplet: the reference builds object columns from the empty lists."""
    import rectools_b200 as rb
    from rectools.models import PopularInCategoryModel
    from tests.popular_cases import popular_dataset

    ds = popular_dataset(n_users=20, seed=2)
    heavy = ds.user_id_map.external_ids[:2]
    wl = ds.item_id_map.external_ids[:4]
    for kw in ({}, {"mixing_strategy": "group", "ratio_strategy": "equal"}):
        model = PopularInCategoryModel(category_feature="category", **kw).fit(ds)
        expected = model.recommend(heavy, ds, 3, True, items_to_recommend=wl)
        assert len(expected) == 0
        rb.install(popular=True)
        try:
            _same_outcome(lambda: model.recommend(heavy, ds, 3, True, items_to_recommend=wl), lambda: expected)
        finally:
            rb.uninstall()

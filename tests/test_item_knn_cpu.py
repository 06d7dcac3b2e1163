"""CPU: ItemKNN (engine path 9, `b200_rank_topk_knn`, `rectools_b200.item_knn`) up to where a GPU is needed.

- the stub's `fit` + `recommend` (tests/knn_oracle.py), driven through the unmodified wrapper, against the known answers of
  the reference's own tests (tests/golden/item_knn_known_answers.json);
- the numpy definition against the unmodified wrapper on the stub: u2i frames equal, i2i frames equal on tie-free rows;
- the export is declared, exported and bound, and the ABI stays 6;
- tests/knn_plan_driver.cpp prints `plan_knn` (rectools_b200/csrc/knn_plan.h): chunk bounds, slots, the dense-route count
  and every refusal;
- host refusals leave the outputs untouched; without a GPU the call fails at its first CUDA call with its own name;
- `install(item_knn=True)` / `uninstall()` and every delegation case, with the library replaced by the numpy definition."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests import knn_oracle
from tests.pairs_oracle import rank_pairs_np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")
FIXTURE = os.path.join(ROOT, "tests", "golden", "item_knn_known_answers.json")


@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    with knn_oracle.stub_methods():
        yield
    stage_reference.remove_from_path(added)


def _dataset(pairs, weights=None):
    import pandas as pd
    from rectools import Columns
    from rectools.dataset import Dataset

    df = pd.DataFrame(pairs, columns=Columns.UserItem)
    df[Columns.Weight] = 1 if weights is None else weights
    df[Columns.Datetime] = "2021-09-09"
    return Dataset.construct(df)


def _random_dataset(seed, n_users=40, n_items=30, per_user=6, weighted=True):
    rng = np.random.default_rng(seed)
    pairs = {(u, int(i)) for u in range(n_users) for i in rng.choice(n_items, size=per_user, replace=False)}
    pairs = sorted(pairs)
    w = rng.integers(1, 9, size=len(pairs)).astype(float) * 0.5 if weighted else None
    return _dataset([[u + 100, i + 500] for u, i in pairs], w)


# ------------------------------------------------------------------------------------------------------ known answers
@needs_ref
def test_stub_reproduces_the_known_answers(ref):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    from implicit.nearest_neighbours import ItemItemRecommender, TFIDFRecommender
    from rectools import Columns
    from rectools.models import ImplicitItemKNNWrapperModel

    fx = json.load(open(FIXTURE))
    ds = _dataset(fx["interactions"])
    cases = [(ItemItemRecommender, fx["base_class"])] + [(TFIDFRecommender, c) for c in fx["basic"] + fx["with_whitelist"]]
    for cls, c in cases:
        model = ImplicitItemKNNWrapperModel(model=cls(K=c["K"])).fit(ds)
        wl = c.get("items_to_recommend")
        actual = model.recommend(users=np.array(c["users"]), dataset=ds, k=c["k"], filter_viewed=c["filter_viewed"],
                                 items_to_recommend=None if wl is None else np.array(wl))
        expected = pd.DataFrame(c["expected"]).astype({Columns.Score: np.float32})
        pd.testing.assert_frame_equal(actual, expected, atol=1e-3)
    ds = _dataset(fx["i2i_interactions"])
    for c in fx["i2i"]:
        model = ImplicitItemKNNWrapperModel(model=TFIDFRecommender(K=c["K"])).fit(ds)
        wl = c["items_to_recommend"]
        actual = model.recommend_to_items(target_items=np.array(c["targets"]), dataset=ds, k=c["k"], filter_itself=c["filter_itself"],
                                          items_to_recommend=None if wl is None else np.array(wl))
        pd.testing.assert_frame_equal(actual.drop(columns=Columns.Score), pd.DataFrame(c["expected"]))


# --------------------------------------------------------------------------------------- the definition vs the wrapper
def _fitted(cls_name, ds, K=8):
    import implicit.nearest_neighbours as nn
    from rectools.models import ImplicitItemKNNWrapperModel

    return ImplicitItemKNNWrapperModel(model=getattr(nn, cls_name)(K=K)).fit(ds)


@needs_ref
@pytest.mark.parametrize("cls_name", ["ItemItemRecommender", "CosineRecommender", "TFIDFRecommender", "BM25Recommender"])
@pytest.mark.parametrize("filter_viewed", [True, False])
@pytest.mark.parametrize("whitelist", [False, True])
def test_definition_equals_the_wrapper_u2i(ref, cls_name, filter_viewed, whitelist):  # pylint: disable=unused-argument,redefined-outer-name
    ds = _random_dataset(3)
    model = _fitted(cls_name, ds)
    user_ids = np.arange(ds.user_id_map.size)
    wl = np.arange(0, ds.item_id_map.size, 3) if whitelist else None
    ui = ds.get_user_item_matrix(include_weights=True)
    for k in (1, 4, 50):
        stock = model._recommend_u2i(user_ids, ds, k, filter_viewed, wl)  # pylint: disable=protected-access
        mine = knn_oracle.recommend_u2i_np(model.model.similarity, ui, user_ids, k, filter_viewed, wl)
        np.testing.assert_array_equal(np.asarray(stock[0]), mine[0])
        np.testing.assert_array_equal(np.asarray(stock[1]), mine[1])
        np.testing.assert_array_equal(np.asarray(stock[2], dtype=np.float64), mine[2])


@needs_ref
@pytest.mark.parametrize("whitelist", [False, True])
def test_definition_equals_the_wrapper_i2i_without_ties(ref, whitelist):  # pylint: disable=unused-argument,redefined-outer-name
    ds = _random_dataset(5)
    model = _fitted("ItemItemRecommender", ds, K=10)
    S = model.model.similarity.copy()
    S.data = np.random.default_rng(1).permutation(S.nnz).astype(np.float64) + 0.5  # distinct values: no tie group
    model.model.similarity = S
    targets = np.arange(ds.item_id_map.size)
    wl = np.arange(1, ds.item_id_map.size, 2) if whitelist else None
    stock = model._recommend_i2i(targets, ds, 4, wl)  # pylint: disable=protected-access
    mine = knn_oracle.recommend_i2i_np(S, targets, 4, wl)
    for a, b in zip(stock, mine):
        np.testing.assert_array_equal(np.asarray(a), b)


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_export_declared_exported_and_bound():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    assert re.search(r"\bint b200_rank_topk_knn\s*\(", header)
    assert "9 = ItemKNN user" in header
    assert "b200_rank_topk_knn" in _lib.EXPORTS
    assert "#define B200_RANK_ABI_VERSION 6" in header and _lib.ABI_VERSION == 6
    assert set(re.findall(r"\b(b200_rank_[a-z_]+)\s*\(", header)) == set(_lib.EXPORTS)
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    assert _lib.load().b200_rank_topk_knn.argtypes is not None


def _call(lib, S, U, k, F=None, wl=None, n_items=None, outs=None):
    from rectools_b200 import _lib

    n = U.shape[0]
    ids, sc, cnt = outs if outs is not None else (np.full((n, k), 77, np.int32), np.full((n, k), 7.0), np.full(n, 77, np.int32))
    keep = []

    def p(a, dtype=None):
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a.ctypes.data

    st = _lib.Stats()
    rc = lib.b200_rank_topk_knn(0, S.shape[0] if n_items is None else n_items, p(S.indptr, np.int64), p(S.indices, np.int32),
                                p(S.data, np.float64), n, p(U.indptr, np.int64), p(U.indices, np.int32), p(U.data, np.float32),
                                None if F is None else p(F.indptr, np.int64), None if F is None else p(F.indices, np.int32),
                                p(wl), -1 if wl is None else len(wl), k, p(ids), p(sc), p(cnt), C.byref(st))
    return rc, ids, sc, cnt


def _csr(dense, dtype):
    m = sparse.csr_matrix(np.asarray(dense, dtype=dtype))
    m.indptr = m.indptr.astype(np.int64)
    m.indices = m.indices.astype(np.int32)
    return m


def test_host_refusals_leave_outputs_untouched():
    from rectools_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = _lib.load()
    S = _csr([[1, 2, 0], [0, 1, 3], [4, 0, 1]], np.float64)
    U = _csr([[1, 0, 2], [0, 1, 0]], np.float32)
    bad_s = S.copy()
    bad_s.data[1] = np.inf
    bad_u = U.copy()
    bad_u.data[0] = np.nan
    oob = U.copy()
    oob.indices = oob.indices.copy()
    oob.indices[0] = 3
    F = _csr([[0, 0, 1], [1, 1, 0]], np.float32)
    F.indices = np.ascontiguousarray(F.indices[[0, 2, 1]])  # row 1 descending
    cases = [
        (dict(S=bad_s, U=U, k=2), "s_data"),
        (dict(S=S, U=bad_u, k=2), "u_data"),
        (dict(S=S, U=oob, k=2), "u_indices"),
        (dict(S=S, U=U, k=2, F=F), "filter ids are not ascending"),
        (dict(S=S, U=U, k=2, wl=np.array([2, 1], np.int32)), "whitelist is not strictly ascending"),
        (dict(S=S, U=U, k=2, wl=np.array([0, 3], np.int32)), "whitelist[1]"),
        (dict(S=S, U=U, k=0), "k must be"),
    ]
    for kw, needle in cases:
        k = max(kw["k"], 1)
        outs = (np.full((2, k), 77, np.int32), np.full((2, k), 7.0), np.full(2, 77, np.int32))
        rc, ids, sc, cnt = _call(lib, outs=outs, **kw)
        assert rc == _lib.E_INVALID, needle
        assert needle in lib.b200_rank_last_error().decode(), (needle, lib.b200_rank_last_error())
        assert (ids == 77).all() and (sc == 7.0).all() and (cnt == 77).all()
    rc, *_ = _call(lib, S, U.__class__((np.zeros(0, np.float32), np.zeros(0, np.int32), np.zeros(1, np.int64)), shape=(0, 3)), 2)
    assert rc == _lib.OK  # no row: nothing to do, no device touched


def test_reports_cuda_failure_without_gpu():
    import torch

    from rectools_b200 import _lib, build

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    build.build()
    lib = _lib.load()
    S = _csr([[1, 2, 0], [0, 1, 3], [4, 0, 1]], np.float64)
    U = _csr([[1, 0, 2], [0, 1, 0]], np.float32)
    rc, ids, sc, cnt = _call(lib, S, U, 2)
    msg = lib.b200_rank_last_error().decode()
    assert rc == _lib.E_CUDA, (rc, msg)
    assert msg.startswith("b200_rank_topk_knn: ") and "failed at line" in msg, msg
    assert (ids == 77).all() and (cnt == 77).all()


# ------------------------------------------------------------------------------------------------------------ the plan
@pytest.fixture(scope="module")
def plan_driver():
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    tmp = tempfile.mkdtemp()
    exe = os.path.join(tmp, "knn_plan_driver")
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "knn_plan_driver.cpp")], env=env,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr

    def run(cases):
        lines = [" ".join(f"{k}={','.join(map(str, v)) if isinstance(v, (list, tuple)) else v}" for k, v in c.items()) for c in cases]
        out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
        plans = []
        for ln in out.splitlines():
            head, _, message = ln.partition(" message=")
            p = {"message": message}
            for w in head.split():
                key, v = w.split("=")
                p[key] = int(v) if key in ("error", "dense") else [int(x) for x in v.split(",") if x]
            plans.append(p)
        return plans

    yield run
    shutil.rmtree(tmp, ignore_errors=True)


def _s_rows(lens):
    """s_indptr / s_indices of an S whose row i holds the first lens[i] items."""
    indptr = np.concatenate([[0], np.cumsum(lens)]).tolist()
    return indptr, [j for n in lens for j in range(n)]


def test_plan_bounds_slots_and_routes(plan_driver):  # pylint: disable=redefined-outer-name
    s_indptr, s_indices = _s_rows([3, 1, 2, 0])
    base = dict(n_items=4, s_indptr=s_indptr, s_indices=s_indices, u_indptr=[0, 2, 2, 3], u_indices=[0, 2, 1], k=2)
    p = plan_driver([base])[0]
    assert p["error"] == 0 and p["bounds"] == [0, 3] and p["bound"] == [5, 0, 1]
    assert p["slot"] == [0, 4, 4, 5]  # row 0: min(B = 5, n_items = 4)
    p = plan_driver([dict(base, wl=[1])])[0]
    assert p["slot"] == [0, 1, 1, 2]  # min(B, n_whitelist)
    p = plan_driver([dict(base, wl="-")])[0]
    assert p["slot"] == [0, 0, 0, 0]
    p = plan_driver([dict(base, max_rows=2)])[0]
    assert p["bounds"] == [0, 2, 3]
    # the byte budget: row bytes 16 + 8m + 4f + 36 slots + 52k + 8
    row0 = 16 + 8 * 2 + 36 * 4 + 52 * 2 + 8
    row1 = 16 + 52 * 2 + 8
    p = plan_driver([dict(base, budget=row0 + row1)])[0]
    assert p["bounds"] == [0, 2, 3]
    p = plan_driver([dict(base, budget=row0 - 1)])[0]
    assert p["error"] == -3 and "row 0" in p["message"]
    # the dense route: B_u above 3072
    big = 4000
    s_indptr, s_indices = _s_rows([big] + [1] * (big - 1))
    p = plan_driver([dict(n_items=big, s_indptr=s_indptr, s_indices=s_indices, u_indptr=[0, 1, 2], u_indices=[0, 1], k=3)])[0]
    assert p["error"] == 0 and p["bound"] == [big, 1] and p["dense"] == 1


def test_plan_refusals(plan_driver):  # pylint: disable=redefined-outer-name
    s_indptr, s_indices = _s_rows([2, 1, 1])
    base = dict(n_items=3, s_indptr=s_indptr, s_indices=s_indices, u_indptr=[0, 1, 2], u_indices=[0, 2], k=2)
    cases = [
        (dict(base, k=0), "k must be >= 1"),
        (dict(base, no_out=1), "NULL"),
        (dict(base, s_indptr=[1, 2, 3, 4]), "s_indptr[0] = 1"),
        (dict(base, s_indptr=[0, 2, 1, 4]), "s_indptr is not monotone at row 1"),
        (dict(base, s_indices=[0, 0, 1, 2]), "S row 0 holds item 0 twice"),
        (dict(base, s_indices=[0, 3, 1, 2]), "s_indices[1] = 3"),
        (dict(base, nan_s=1), "s_data[0] is not finite"),
        (dict(base, u_indptr=[0, 2, 1]), "u_indptr is not monotone at row 1"),
        (dict(base, u_indices=[0, -1]), "u_indices[1] = -1"),
        (dict(base, nan_u=1), "u_data[0] is not finite"),
        (dict(base, f_indptr=[0, 2, 2], f_indices=[2, 1]), "row 0: filter ids are not ascending"),
        (dict(base, wl=[1, 1]), "the whitelist is not strictly ascending"),
        (dict(base, wl=[0, 3]), "whitelist[1] = 3"),
    ]
    plans = plan_driver([c for c, _ in cases])
    for (c, needle), p in zip(cases, plans):
        assert p["error"] == -1, (c, p)
        assert needle in p["message"] and p["message"].startswith("b200_rank_topk_knn: "), (needle, p["message"])
        assert p["bounds"] == [] and p["slot"] == []
    ok = plan_driver([dict(base, f_indptr=[0, 2, 3], f_indices=[1, 1, -5])])[0]  # repeats and any int32 in a filter row
    assert ok["error"] == 0


# ------------------------------------------------------------------------------------------------ install and delegation
@pytest.fixture
def numpy_library(monkeypatch):
    """`rank_knn` and `rank_pairs` replaced by the numpy definitions, recording their calls."""
    from rectools_b200 import item_knn, rerank

    calls = []

    def fake_knn(similarity, user_rows, k, filter_rows=None, whitelist=None, device=0, stats=None):  # pylint: disable=unused-argument
        calls.append("knn")
        return knn_oracle.rank_knn_np(similarity, user_rows, k, filter_rows, whitelist)

    def fake_pairs(codes, scores, k, device=0, n_groups=None, stats=None):  # pylint: disable=unused-argument
        calls.append("pairs")
        return rank_pairs_np(codes, scores, k, n_groups)

    monkeypatch.setattr(item_knn, "rank_knn", fake_knn)
    monkeypatch.setattr(rerank, "rank_pairs", fake_pairs)
    return calls


@needs_ref
def test_install_serves_and_uninstall_restores(ref, numpy_library):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    from rectools.models import ImplicitItemKNNWrapperModel

    import rectools_b200 as rb

    ds = _random_dataset(11)
    model = _fitted("TFIDFRecommender", ds)
    users = ds.user_id_map.external_ids[:15]
    items = ds.item_id_map.external_ids
    stock_u = model.recommend(users, ds, k=5, filter_viewed=True)
    stock_wl = model.recommend(users, ds, k=5, filter_viewed=False, items_to_recommend=items[::2])
    stock_i = model.recommend_to_items(items[:10], ds, k=3)
    orig = {n: ImplicitItemKNNWrapperModel.__dict__[n] for n in ("_recommend_u2i", "_recommend_i2i")}
    rb.install(item_knn=True, fast_recommend=False)
    try:
        assert ImplicitItemKNNWrapperModel.__dict__["_recommend_u2i"] is not orig["_recommend_u2i"]
        pd.testing.assert_frame_equal(model.recommend(users, ds, k=5, filter_viewed=True), stock_u)
        pd.testing.assert_frame_equal(model.recommend(users, ds, k=5, filter_viewed=False, items_to_recommend=items[::2]), stock_wl)
        mine_i = model.recommend_to_items(items[:10], ds, k=3)
        key = ["target_item_id", "item_id"]
        pd.testing.assert_frame_equal(mine_i.sort_values(key).reset_index(drop=True), stock_i.sort_values(key).reset_index(drop=True))
        assert numpy_library.count("knn") == 2 and numpy_library.count("pairs") == 1
    finally:
        rb.uninstall()
    for n, f in orig.items():
        assert ImplicitItemKNNWrapperModel.__dict__[n] is f


@needs_ref
def test_delegation_cases(ref, numpy_library):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    from implicit.nearest_neighbours import ItemItemRecommender
    from rectools.models import ImplicitItemKNNWrapperModel

    import rectools_b200 as rb

    class CustomKNN(ItemItemRecommender):  # a bare subclass: served
        pass

    class OwnRecommend(ItemItemRecommender):  # overrides recommend: delegated
        def recommend(self, *args, **kwargs):  # pylint: disable=useless-parent-delegation
            return super().recommend(*args, **kwargs)

    ds = _random_dataset(13)
    users = ds.user_id_map.external_ids[:10]

    def run(model):
        numpy_library.clear()
        stock = model.recommend(users, ds, k=4, filter_viewed=True)
        rb.install(item_knn=True, fast_recommend=False)
        try:
            mine = model.recommend(users, ds, k=4, filter_viewed=True)
        finally:
            rb.uninstall()
        pd.testing.assert_frame_equal(mine, stock)
        return "knn" in numpy_library

    assert run(ImplicitItemKNNWrapperModel(model=CustomKNN(K=6)).fit(ds))
    assert not run(ImplicitItemKNNWrapperModel(model=OwnRecommend(K=6)).fit(ds))
    dense = ImplicitItemKNNWrapperModel(model=ItemItemRecommender(K=6)).fit(ds)
    dense.model.similarity = dense.model.similarity.tocoo()  # not a CSR
    assert not run(dense)
    nan = ImplicitItemKNNWrapperModel(model=ItemItemRecommender(K=6)).fit(ds)
    nan.model.similarity = nan.model.similarity.copy()
    nan.model.similarity.data[0] = np.nan
    numpy_library.clear()
    rb.install(item_knn=True, fast_recommend=False)
    try:
        assert rb.item_knn._served_similarity(nan) is None  # pylint: disable=protected-access
        ints = ImplicitItemKNNWrapperModel(model=ItemItemRecommender(K=6)).fit(ds)
        ints.model.similarity = ints.model.similarity.astype(np.int64)
        assert rb.item_knn._served_similarity(ints) is None  # pylint: disable=protected-access
        dup = ImplicitItemKNNWrapperModel(model=ItemItemRecommender(K=6)).fit(ds)
        S = dup.model.similarity
        dup.model.similarity = sparse.csr_matrix((np.r_[S.data[:1], S.data], np.r_[S.indices[:1], S.indices],
                                                  np.r_[0, S.indptr[1:] + 1]), shape=S.shape)
        assert rb.item_knn._served_similarity(dup) is None  # pylint: disable=protected-access
    finally:
        rb.uninstall()
    raw = ds.get_raw_interactions()
    weights = np.ones(len(raw))
    weights[3] = np.inf
    inf_ds = _dataset(raw[["user_id", "item_id"]].to_numpy().tolist(), weights)
    model = _fitted("ItemItemRecommender", ds, K=6)
    numpy_library.clear()
    rb.install(item_knn=True, fast_recommend=False)
    try:
        with np.errstate(all="ignore"):
            rb.item_knn.item_knn_recommend_u2i(model, np.arange(5), inf_ds, 3, True, None)
        assert "knn" not in numpy_library  # non-finite weights: the stock loop ranks them
    finally:
        rb.uninstall()

"""CPU: RecTools' `calc_metrics` on path 10 (`b200_rank_metrics`, `rectools_b200.metrics`) up to where a GPU is needed.

- the numpy definition of the device outputs (tests/metrics_oracle.py) against the stock pandas code on the staged
  reference: the confusion tables equal `calc_confusions(merge_reco(...), k)` exactly, the per-user NDCG / MRR / MAP
  values equal `calc_per_user_from_merged` / `calc_per_user_from_fitted` bit for bit and in the same order;
- `rectools_b200.calc_metrics` with the library replaced by that definition gives stock's dict (keys, order, `==`
  values) for mixes with the other metric families, and hands every delegation case to the stock function;
- the known answers of the reference's own metric tests (tests/golden/metrics_known_answers.json);
- tests/metrics_plan_driver.cpp pins `plan_metrics` (rectools_b200/csrc/metrics_plan.h): device bytes and every refusal;
- the export is declared, exported and bound, and the ABI stays 6; without a GPU the call fails at its first CUDA call
  with its own name;
- `install(metrics=True)` / `uninstall()` rebind and restore the three module attributes, and `cross_validate` scores
  through the rebound function."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess
import tempfile
import warnings

import numpy as np
import pytest

from oracle import stage_reference
from tests import metrics_cases, metrics_oracle

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
FIXTURE = os.path.join(ROOT, "tests", "golden", "metrics_known_answers.json")
pytestmark = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    yield
    stage_reference.remove_from_path(added)


@pytest.fixture()
def fake_device(monkeypatch, ref):  # pylint: disable=unused-argument,redefined-outer-name
    """`device_metrics` replaced by the numpy definition; returns the list of its calls."""
    from rectools_b200 import metrics

    calls = []

    def fake(*args, **kwargs):
        calls.append(args)
        return metrics_oracle.device_metrics_np(*args, **kwargs)

    monkeypatch.setattr(metrics, "device_metrics", fake)
    return calls


def _bits(a):
    return np.asarray(a, dtype=np.float64).view(np.int64)


def _assert_same_dict(actual, expected):
    assert list(actual) == list(expected)
    for k in expected:
        e, a = expected[k], actual[k]
        assert type(a) is type(e), (k, type(a), type(e))
        assert a == e or (e != e and a != a), (k, a, e)


CASES = [
    dict(seed=1),
    dict(seed=2, id_dtype=np.int32, max_test=20, hit_share=0.7, dup_share=0.3),
    dict(seed=3, id_dtype=np.uint32, k_reco=25, hit_share=0.6),
    dict(seed=4, shuffle=False, ragged=False),
    dict(seed=5, n_users=10, n_items=8, k_reco=8, max_test=30, hit_share=0.9, dup_share=0.4),  # many repeats per rank
    dict(seed=6, extra_test_users=20, extra_reco_users=30, hit_share=0.2),
]


def _oracle_outputs(reco, interactions, ks, ranking):
    from rectools_b200.metrics import ndcg_tables

    tables, specs = ndcg_tables(ranking)
    cols = [np.asarray(interactions[c], np.int64) for c in ("user_id", "item_id")] + \
        [np.asarray(reco[c], np.int64) for c in ("user_id", "item_id", "rank")]
    return metrics_oracle.device_metrics_np(*cols, ks, tables, len(ks) > 0), tables, specs


# ---------------------------------------------------------------------------------------------- the definition vs stock
def test_pairwise_sum_is_numpys_reduceat():
    rng = np.random.default_rng(0)
    for n in list(range(1, 300)) + [1000, 4099]:
        a = rng.random(n) * 10.0 ** rng.integers(-8, 8, size=n)
        assert np.add.reduceat(a, [0])[0] == a[0] + metrics_oracle.pairwise_sum(list(a[1:])), n


@pytest.mark.parametrize("case", CASES, ids=[str(c["seed"]) for c in CASES])
def test_definition_against_stock_per_user(ref, case):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    from rectools.metrics import MAP, MRR, NDCG
    from rectools.metrics.base import merge_reco
    from rectools.metrics.classification import calc_confusions

    from rectools_b200.metrics import confusion_df, ranking_per_user

    reco, interactions = metrics_cases.tables(**case)
    ks = [1, 3, 10, 40]  # 40: larger than any list
    ranking = {}
    for k in ks:
        ranking[f"map{k}"] = MAP(k=k)
        ranking[f"mapk{k}"] = MAP(k=k, divide_by_k=True)
        ranking[f"mrr{k}"] = MRR(k=k)
        for base in (2, 3, 10):
            for ach in (False, True):
                ranking[f"ndcg{k}_{base}_{ach}"] = NDCG(k=k, log_base=base, divide_by_achievable=ach)
    out, tables, specs = _oracle_outputs(reco, interactions, ks, ranking)
    users = out["users"].astype(interactions["user_id"].dtype)
    assert out["flags"] == 0
    assert not np.array_equal(out["first_order"], np.arange(len(users))) or not case.get("shuffle", True)
    merged = merge_reco(reco, interactions)
    for q, k in enumerate(ks):
        pd.testing.assert_frame_equal(confusion_df(users, out["liked"], out["tp"][q], k), calc_confusions(merged, k), check_exact=True)
    k_index = {k: q for q, k in enumerate(ks)}
    fitted = MAP.fit(merged, max(ks))
    for name, m in ranking.items():
        expected = m.calc_per_user_from_fitted(fitted) if type(m) is MAP else m.calc_per_user_from_merged(merged)
        mine = ranking_per_user(m, out, tables, specs, k_index)
        order = np.arange(len(users)) if type(m) is MAP else out["first_order"]
        np.testing.assert_array_equal(users[order], expected.index.to_numpy(), err_msg=name)
        np.testing.assert_array_equal(_bits(mine), _bits(expected.to_numpy()), err_msg=name)
        assert pd.Series(mine).mean() == expected.mean() or np.isnan(expected.mean()), name


def test_ndcg_compensated_sum_differs_from_a_plain_one(ref):  # pylint: disable=unused-argument,redefined-outer-name
    """A user with many hits past k: the exact 0.0 terms still move pandas' compensation, and its sum is not the plain
    one; the definition (and so the device) gives pandas' bits."""
    from rectools.metrics import NDCG
    from rectools.metrics.base import merge_reco

    reco, interactions = metrics_cases.tables(11, n_users=40, n_items=300, k_reco=200, max_test=150, hit_share=0.9, dup_share=0.2)
    found = False
    for k, base in ((50, 3), (120, 10), (200, 2)):
        m = NDCG(k=k, log_base=base)
        out, tables, specs = _oracle_outputs(reco, interactions, [k], {"n": m})
        T = tables[0]
        expected = m.calc_per_user_from_merged(merge_reco(reco, interactions))
        mine = out["ndcg"][0][out["first_order"]]
        np.testing.assert_array_equal(_bits(mine), _bits(expected.to_numpy()))
        order = np.argsort(np.unique(interactions["user_id"], return_inverse=True)[1], kind="stable")
        hit = merge_reco(reco, interactions)["rank"].to_numpy()
        inv = np.unique(interactions["user_id"], return_inverse=True)[1]
        for s in range(len(out["users"])):
            ranks = [int(r) for r in hit[order][inv[order] == s] if r == r]
            plain = 0.0
            for r in ranks:
                plain += float(T[r - 1]) if r <= k else 0.0
            found |= plain != out["ndcg"][0][s]
    assert found


def test_map_sums_past_128_distinct_ranks(ref):  # pylint: disable=unused-argument,redefined-outer-name
    """Users with hundreds of distinct hit ranks: scipy's row sum takes numpy's pairwise split, and so does the
    definition."""
    from rectools.metrics import MAP
    from rectools.metrics.base import merge_reco

    reco, interactions = metrics_cases.tables(12, n_users=6, n_items=900, k_reco=800, max_test=700, hit_share=0.95, dup_share=0.1)
    ks = [9, 130, 400, 800]
    out, _, _ = _oracle_outputs(reco, interactions, ks, {})
    merged = merge_reco(reco, interactions)
    fitted = MAP.fit(merged, 800)
    assert (np.diff(fitted.precision_at_k.indptr) > 300).any()
    for q, k in enumerate(ks):
        expected = MAP(k=k).calc_per_user_from_fitted(fitted).to_numpy()
        np.testing.assert_array_equal(_bits(out["map"][q] / out["liked"]), _bits(expected))


# ------------------------------------------------------------------------------------------------ calc_metrics, faked
def _other_metrics():
    import pandas as pd
    from rectools.metrics import (
        AvgRecPopularity, CatalogCoverage, Intersection, IntraListDiversity, MeanInvUserFreq, PairwiseHammingDistanceCalculator,
        Serendipity,
    )

    features = pd.DataFrame({"f1": np.arange(5000) % 3, "f2": np.arange(5000) % 7}, index=pd.Index(np.arange(5000), name="item_id"))
    # (the AUC family is mixed in by the known-answer call below: on these tables stock's PartialAUC / PAP raise under
    # pandas 3, in `outer_merge_reco`'s cumsum over an object column)
    return {"miuf@3": MeanInvUserFreq(k=3), "arp@3": AvgRecPopularity(k=3),
            "ild@3": IntraListDiversity(k=3, distance_calculator=PairwiseHammingDistanceCalculator(features)),
            "seren@3": Serendipity(k=3), "cov@3": CatalogCoverage(k=3), "inter@3": Intersection(k=3)}


@pytest.mark.parametrize("seed", [21, 22, 23])
def test_calc_metrics_equals_stock_with_other_families(fake_device, seed):  # pylint: disable=redefined-outer-name
    from rectools.metrics import calc_metrics as stock

    import rectools_b200

    reco, interactions = metrics_cases.tables(seed, id_dtype=(np.int64, np.int32, np.uint32)[seed % 3])
    prev = interactions.sample(frac=0.5, random_state=seed)
    catalog = np.unique(np.concatenate([reco["item_id"], interactions["item_id"]]))
    served = metrics_cases.served_metrics(ks=(1, 5, 12))
    others = _other_metrics()
    names = list(served) + list(others)
    order = np.random.default_rng(seed).permutation(len(names))
    metrics = {names[i]: {**served, **others}[names[i]] for i in order}
    ref_reco = {"half": reco.sample(frac=0.5, random_state=seed), "other": reco.sample(frac=0.7, random_state=seed + 1)}
    expected = stock(metrics, reco, interactions, prev, catalog, ref_reco)
    actual = rectools_b200.calc_metrics(metrics, reco, interactions, prev, catalog, ref_reco)
    _assert_same_dict(actual, expected)
    assert len(fake_device) == 1
    # one family alone, and the two families with nothing else
    for sub in ({k: v for k, v in served.items() if k.startswith("ndcg")}, metrics_cases.nine_metrics(5)):
        _assert_same_dict(rectools_b200.calc_metrics(sub, reco, interactions, catalog=catalog), stock(sub, reco, interactions, catalog=catalog))


def _delegation_cases():
    import pandas as pd
    from rectools.metrics import MCC, NDCG, Accuracy, DebiasConfig, Precision

    class MyPrecision(Precision):
        pass

    reco, inter = metrics_cases.tables(31)
    nine = metrics_cases.nine_metrics(3)
    dup = pd.concat([reco, reco.iloc[:1]], ignore_index=True)
    rank0 = reco.copy()
    rank0.loc[0, "rank"] = 0
    f_users = inter.astype({"user_id": np.float64})
    obj_items = reco.astype({"item_id": object})
    f_rank = reco.astype({"rank": np.float64})
    big = inter.astype({"user_id": np.uint64})
    big.loc[0, "user_id"] = np.uint64(2**63 + 5)
    u64 = inter.astype({"user_id": np.uint64})  # uint64 against int64: no common integer type
    nullable = inter.astype({"item_id": "Int64"})
    missing = inter.drop(columns=["item_id"])
    return {
        "no interactions": (nine, reco, None, list(range(9999)), "no call"),
        "no catalog with Accuracy": ({"acc": Accuracy(k=2), "p": Precision(k=2)}, reco, inter, None, "no call"),
        "no catalog with MCC": ({"mcc": MCC(k=2)}, reco, inter, None, "no call"),
        "debias": ({"p": Precision(k=2, debias_config=DebiasConfig(iqr_coef=1.5, random_state=3)), "n": NDCG(k=2)}, reco, inter, None, "no call"),
        "subclass": ({"p": MyPrecision(k=2), "n": NDCG(k=2)}, reco, inter, None, "no call"),
        "float user ids": (nine, reco, f_users, list(range(9999)), "no call"),
        "object item ids": (nine, obj_items, inter, list(range(9999)), "no call"),
        "float ranks": (nine, f_rank, inter, list(range(9999)), "no call"),
        "uint64 >= 2^63": (nine, reco, big, list(range(9999)), "no call"),
        "uint64 with int64": (nine, reco, u64, list(range(9999)), "no call"),
        "nullable ints": (nine, reco, nullable, list(range(9999)), "no call"),
        "missing column": ({"n": NDCG(k=2)}, reco, missing, None, "no call"),
        "empty interactions": (nine, reco, inter.iloc[:0], list(range(9999)), "no call"),
        "non-int k": ({"n": NDCG(k=2.0)}, reco, inter, None, "no call"),
        "log_base below 1": ({"n": NDCG(k=2, log_base=0.5)}, reco, inter, None, "no call"),
        "duplicate reco pair": (nine, dup, inter, list(range(9999)), "call"),
        "rank below 1": (nine, rank0, inter, list(range(9999)), "call"),
    }


@pytest.mark.parametrize("name", [
    "no interactions", "no catalog with Accuracy", "no catalog with MCC", "debias", "subclass", "float user ids", "object item ids",
    "float ranks", "uint64 >= 2^63", "uint64 with int64", "nullable ints", "missing column", "empty interactions", "non-int k",
    "log_base below 1", "duplicate reco pair", "rank below 1"])
def test_delegation(fake_device, name):  # pylint: disable=redefined-outer-name
    from rectools.metrics import calc_metrics as stock

    import rectools_b200

    metrics, reco, inter, catalog, call = _delegation_cases()[name]

    def run(f):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            try:
                return ("ok", f(metrics, reco, inter, catalog=catalog)), [str(x.message) for x in w]
            except Exception as e:  # pylint: disable=broad-except
                return ("raise", type(e), str(e)), [str(x.message) for x in w]

    expected, w_expected = run(stock)
    actual, w_actual = run(rectools_b200.calc_metrics)
    assert len(fake_device) == (1 if call == "call" else 0)
    assert w_actual == w_expected
    if expected[0] == "ok":
        assert actual[0] == "ok", actual
        _assert_same_dict(actual[1], expected[1])
    else:
        assert actual == expected
    if name in ("no interactions", "no catalog with Accuracy", "no catalog with MCC"):
        assert expected[0] == "raise" and expected[1] is ValueError


def test_refused_allocation_warns_and_returns_stock(monkeypatch, ref):  # pylint: disable=unused-argument,redefined-outer-name
    from rectools.metrics import calc_metrics as stock

    import rectools_b200
    from rectools_b200 import metrics

    def refuse(*args, **kwargs):
        raise MemoryError("b200_rank_metrics: cudaMalloc(&p, ...) failed at line 1: out of memory")

    monkeypatch.setattr(metrics, "device_metrics", refuse)
    reco, inter = metrics_cases.tables(41)
    nine = metrics_cases.nine_metrics(4)
    with pytest.warns(RuntimeWarning, match="refused an allocation"):
        actual = rectools_b200.calc_metrics(nine, reco, inter, catalog=list(range(9999)))
    _assert_same_dict(actual, stock(nine, reco, inter, catalog=list(range(9999))))


# --------------------------------------------------------------------------------------------------------- known answers
def _known_answer_frames(c):
    import pandas as pd

    return pd.DataFrame(c["reco"]), pd.DataFrame(c["interactions"])


def _metric(spec):
    import rectools.metrics as RM

    kw = {k: v for k, v in spec.items() if k != "class"}
    return getattr(RM, spec["class"])(**kw)


def test_known_answers_per_user(fake_device):  # pylint: disable=redefined-outer-name
    import pandas as pd
    from rectools.metrics import MAP, MRR, NDCG

    import rectools_b200
    from rectools_b200.metrics import confusion_df, ranking_per_user

    fx = json.load(open(FIXTURE))
    assert len(fx["per_user"]) >= 15
    for c in fx["per_user"]:
        reco, inter = _known_answer_frames(c)
        m = _metric(c["metric"])
        expected = pd.Series(c["expected"], index=pd.Index(c["users"], name="user_id"), dtype=float)
        if type(m) in (NDCG, MRR, MAP):
            ks = [m.k] if type(m) is MAP else []
            out, tables, specs = _oracle_outputs(reco, inter, ks, {"m": m})
            order = np.arange(len(out["users"])) if type(m) is MAP else out["first_order"]
            mine = pd.Series(ranking_per_user(m, out, tables, specs, {m.k: 0}), index=pd.Index(out["users"][order], name="user_id"))
        else:
            out, _, _ = _oracle_outputs(reco, inter, [m.k], {})
            conf = confusion_df(out["users"], out["liked"], out["tp"][0], m.k)
            args = (conf,) if c["catalog"] is None else (conf, c["catalog"])
            mine = m.calc_per_user_from_confusion_df(*args)
        pd.testing.assert_series_equal(mine, expected, check_names=False)
        value = rectools_b200.calc_metrics({"m": m}, reco, inter, catalog=c["catalog"])["m"]
        assert np.isclose(value, expected.mean()), (c["metric"], value, expected.mean())


def test_known_answers_of_the_scoring_call(fake_device):  # pylint: disable=redefined-outer-name
    import pandas as pd
    import rectools.metrics as RM
    from rectools.metrics.base import MetricAtK

    import rectools_b200

    fx = json.load(open(FIXTURE))["scoring_success"]
    features = pd.DataFrame(fx["features"]).set_index("item_id")
    calculator = RM.PairwiseHammingDistanceCalculator(features)
    metrics = {}
    # the AUC family is left out: stock's `_AUCMetric.fit` raises under pandas 3 (a groupby cumsum over an object
    # column), with and without this package
    auc = ("PartialAUC", "PAP")
    expected = {k: v for k, v in fx["expected"].items() if k not in {name for name, cls, _ in fx["metrics"] if cls in auc}}
    for name, cls, kw in (row for row in fx["metrics"] if row[1] not in auc):
        if cls == "MetricAtK":
            metrics[name] = MetricAtK(**kw)
        elif cls == "IntraListDiversity":
            metrics[name] = RM.IntraListDiversity(distance_calculator=calculator, **kw)
        else:
            metrics[name] = getattr(RM, cls)(**kw)
    ref_recos = {k: pd.DataFrame(v) for k, v in fx["ref_recos"].items()}
    args = (pd.DataFrame(fx["reco"]), pd.DataFrame(fx["interactions"]), pd.DataFrame(fx["prev_interactions"]), fx["catalog"], ref_recos)
    with pytest.warns(UserWarning, match="Custom metrics are not supported"):
        actual = rectools_b200.calc_metrics(metrics, *args)
    assert actual == expected  # the literal's values (its key order is not stock's)
    with pytest.warns(UserWarning, match="Custom metrics are not supported"):
        _assert_same_dict(actual, RM.calc_metrics(metrics, *args))
    assert len(fake_device) == 1


# ------------------------------------------------------------------------------------------------------------ the C ABI
def test_export_declared_exported_and_bound():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    assert re.search(r"\bint b200_rank_metrics\s*\(", header)
    assert "10 = classification and ranking metrics" in header
    assert "b200_rank_metrics" in _lib.EXPORTS
    assert "#define B200_RANK_ABI_VERSION 6" in header and _lib.ABI_VERSION == 6
    assert set(re.findall(r"\b(b200_rank_[a-z_]+)\s*\(", header)) == set(_lib.EXPORTS)
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    assert _lib.load().b200_rank_metrics.argtypes is not None


def _raw_call(lib, n_inter=3, ks=(1, 2), offsets=(0, 2), map_out=True, **null):
    from rectools_b200 import _lib

    keep = []

    def p(a, dtype=np.int64):
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a.ctypes.data

    n = max(n_inter, 1)
    outs = {name: np.full(n * max(len(ks), len(offsets), 1), 77, np.int64) for name in ("users", "first", "liked", "min", "tp")}
    fouts = {name: np.full(n * max(len(ks), len(offsets), 1), 7.0) for name in ("map", "ndcg")}
    n_users, flags = C.c_int64(-5), C.c_int32(-5)
    g = lambda name, v: None if null.get(name) else v  # noqa: E731
    rc = lib.b200_rank_metrics(
        0, None, n_inter, g("iu", p([1, 2, 1])), g("ii", p([5, 6, 7])), 2, g("ru", p([1, 2])), p([5, 6]), p([1, 1]),
        len(ks), g("ks", p(list(ks) or [0])), len(offsets) - 1 if offsets else 0, g("offsets", p(list(offsets) or [0])),
        g("terms", p([1.0, 0.5], np.float64)), C.byref(n_users), outs["users"].ctypes.data, outs["first"].ctypes.data,
        outs["liked"].ctypes.data, outs["min"].ctypes.data, g("tp", outs["tp"].ctypes.data),
        fouts["map"].ctypes.data if map_out else None, g("ndcg", fouts["ndcg"].ctypes.data), C.byref(flags), C.byref(_lib.Stats()),
    )
    untouched = all((a == 77).all() for a in outs.values()) and all((a == 7.0).all() for a in fouts.values())
    return rc, untouched and n_users.value == -5 and flags.value == -5


def test_host_refusals_leave_outputs_untouched():
    from rectools_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = _lib.load()
    cases = [
        (dict(ks=(2, 2)), "ks are not strictly ascending"),
        (dict(ks=(0, 2)), "ks[0] = 0"),
        (dict(offsets=(1, 2)), "ndcg_offsets[0] = 1"),
        (dict(offsets=(0, 0)), "NDCG table 0 has 0 terms"),
        (dict(ks=(), map_out=True), "out_map is given without a k"),
        (dict(iu=True), "inter_users / inter_items are NULL"),
        (dict(ru=True), "reco_users / reco_items / reco_ranks are NULL"),
        (dict(tp=True), "out_tp is NULL"),
        (dict(ndcg=True), "out_ndcg is NULL"),
        (dict(terms=True), "ndcg_terms is NULL"),
    ]
    for kw, needle in cases:
        null = {k: v for k, v in kw.items() if v is True}
        rest = {k: v for k, v in kw.items() if v is not True}
        rc, untouched = _raw_call(lib, **rest, **null)
        msg = lib.b200_rank_last_error().decode()
        assert rc == _lib.E_INVALID, (needle, rc, msg)
        assert needle in msg and msg.startswith("b200_rank_metrics: "), (needle, msg)
        assert untouched, needle


def test_reports_cuda_failure_without_gpu():
    import torch

    from rectools_b200 import _lib, build

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    build.build()
    lib = _lib.load()
    rc, untouched = _raw_call(lib)
    msg = lib.b200_rank_last_error().decode()
    assert rc == _lib.E_CUDA, (rc, msg)
    assert msg.startswith("b200_rank_metrics: ") and "failed at line" in msg, msg
    assert untouched
    rc, _ = _raw_call(lib, n_inter=0)  # no interaction row: nothing to do, no device touched
    assert rc == _lib.OK


# ------------------------------------------------------------------------------------------------------------- the plan
@pytest.fixture(scope="module")
def plan_driver():
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    tmp = tempfile.mkdtemp()
    exe = os.path.join(tmp, "metrics_plan_driver")
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "metrics_plan_driver.cpp")],
                         env=env, capture_output=True, text=True)
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
                p[key] = int(v)
            plans.append(p)
        return plans

    yield run
    shutil.rmtree(tmp, ignore_errors=True)


def _bytes(n, m, slots, n_k, n_ndcg, n_terms, with_map):
    per_row = 40 + (24 if with_map else 0)
    per_user = 56 + 8 * n_k + 8 * n_ndcg + (16 + 8 * n_k if with_map else 0)
    return n * (per_row + per_user) + 24 * m + 4 * slots + 8 * n_k + 8 * (n_ndcg + 1) + 8 * n_terms + 12


def test_plan_slots_and_bytes(plan_driver):  # pylint: disable=redefined-outer-name
    base = dict(n_inter=1000, n_reco=300, ks=[1, 5, 10], ndcg_offsets=[0, 10, 15])
    plans = plan_driver([base, dict(base, map=1), dict(base, n_reco=0), dict(base, n_reco=8), dict(base, n_reco=9),
                         dict(n_inter=5_400_000, n_reco=10_000_000, ks=[10], ndcg_offsets=[0, 10], map=1)])
    assert all(p["error"] == 0 for p in plans), plans
    assert [p["slots"] for p in plans] == [1024, 1024, 16, 16, 32, 2**25]
    assert plans[0]["k_max"] == 10 and plans[0]["n_terms"] == 15
    assert plans[0]["bytes"] == _bytes(1000, 300, 1024, 3, 2, 15, False)
    assert plans[1]["bytes"] == _bytes(1000, 300, 1024, 3, 2, 15, True)
    assert plans[5]["bytes"] == _bytes(5_400_000, 10_000_000, 2**25, 1, 1, 10, True)
    assert plans[5]["bytes"] < 2 * 2**30  # the measured shape: under 2 GiB of device memory


def test_plan_refusals(plan_driver):  # pylint: disable=redefined-outer-name
    base = dict(n_inter=10, n_reco=10, ks=[1, 5], ndcg_offsets=[0, 3])
    cases = [
        (dict(base, n_inter=-1), "n_inter and n_reco must be >= 0"),
        (dict(base, n_reco=2**31), "must be <= 2^31 - 1"),
        (dict(base, n_k=-1), "n_k and n_ndcg must be >= 0"),
        (dict(base, no_inter=1), "inter_users / inter_items are NULL"),
        (dict(base, no_reco=1), "reco_users / reco_items / reco_ranks are NULL"),
        (dict(base, no_ks=1), "ks is NULL"),
        (dict(base, ks=[0, 5]), "ks[0] = 0 lies outside"),
        (dict(base, ks=[1, 2**31]), "ks[1] = 2147483648 lies outside"),
        (dict(base, ks=[5, 5]), "ks are not strictly ascending"),
        (dict(base, ks=[], map=1), "out_map is given without a k"),
        (dict(base, no_offsets=1), "ndcg_offsets is NULL"),
        (dict(base, ndcg_offsets=[2, 3]), "ndcg_offsets[0] = 2, not 0"),
        (dict(base, ndcg_offsets=[0, 3, 3]), "NDCG table 1 has 0 terms"),
        (dict(base, no_terms=1), "ndcg_terms is NULL"),
        (dict(base, no_out=1), "out_n_users / out_users"),
        (dict(base, no_tp=1), "out_tp is NULL"),
        (dict(base, no_ndcg=1), "out_ndcg is NULL"),
    ]
    plans = plan_driver([c for c, _ in cases])
    for (_, needle), p in zip(cases, plans):
        assert p["error"] == -1, (needle, p)
        assert needle in p["message"] and p["message"].startswith("b200_rank_metrics: "), (needle, p["message"])
    ok = plan_driver([dict(n_inter=0, n_reco=0, no_inter=1, no_reco=1, no_out=1, no_tp=1, no_ndcg=1, ks=[3], ndcg_offsets=[0, 1])])[0]
    assert ok["error"] == 0, ok  # no rows: NULL arrays and outputs are accepted


# ----------------------------------------------------------------------------------------------------- install(metrics)
def test_install_rebinds_and_uninstall_restores(fake_device):  # pylint: disable=redefined-outer-name
    import importlib

    import rectools_b200

    mods = [importlib.import_module(m) for m in ("rectools.metrics.scoring", "rectools.metrics", "rectools.model_selection.cross_validate")]
    stock = [m.calc_metrics for m in mods]
    assert stock[0] is stock[1] is stock[2]
    rectools_b200.install(metrics=True, fast_recommend=False)
    try:
        bound = [m.calc_metrics for m in mods]
        assert bound[0] is bound[1] is bound[2] and bound[0] is not stock[0]
        reco, inter = metrics_cases.tables(51)
        nine = metrics_cases.nine_metrics(3)
        _assert_same_dict(mods[1].calc_metrics(nine, reco, inter, catalog=list(range(9999))),
                          stock[0](nine, reco, inter, catalog=list(range(9999))))
        assert len(fake_device) == 1
    finally:
        rectools_b200.uninstall()
    assert [m.calc_metrics for m in mods] == stock


def test_cross_validate_scores_through_the_rebound_function(fake_device):  # pylint: disable=redefined-outer-name
    import pandas as pd
    from rectools.dataset import Dataset
    from rectools.model_selection import TimeRangeSplitter, cross_validate
    from rectools.models import PopularModel

    import rectools_b200

    rng = np.random.default_rng(61)
    n = 3000
    df = pd.DataFrame({"user_id": rng.integers(0, 200, n), "item_id": rng.integers(0, 80, n), "weight": 1.0,
                       "datetime": pd.Timestamp("2021-01-01") + pd.to_timedelta(rng.integers(0, 30, n), unit="D")})
    dataset = Dataset.construct(df)
    splitter = TimeRangeSplitter(test_size="5D", n_splits=2, filter_already_seen=True)
    metrics = {**metrics_cases.nine_metrics(5), "ndcg_ach@10": __import__("rectools.metrics", fromlist=["NDCG"]).NDCG(k=10, divide_by_achievable=True)}
    kw = dict(dataset=dataset, splitter=splitter, metrics=metrics, models={"pop": PopularModel()}, k=10, filter_viewed=True)
    expected = cross_validate(**kw)
    rectools_b200.install(metrics=True, fast_recommend=False)
    try:
        actual = cross_validate(**kw)
    finally:
        rectools_b200.uninstall()
    assert len(fake_device) == 2  # one call per fold
    assert actual["metrics"] == expected["metrics"]

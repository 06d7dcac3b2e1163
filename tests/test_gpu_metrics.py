"""GPU: RecTools' `calc_metrics` on path 10 (`b200_rank_metrics`) against the stock function of the staged reference,
with `==` on every value (no tolerance), and the device's per-user arrays against the numpy definition of
tests/metrics_oracle.py."""
import json
import os

import numpy as np
import pytest

from oracle import stage_reference
from tests import metrics_cases, metrics_oracle

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")]
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
FIXTURE = os.path.join(ROOT, "tests", "golden", "metrics_known_answers.json")


@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    yield
    stage_reference.remove_from_path(added)


def _same(actual, expected):
    assert list(actual) == list(expected)
    for k, e in expected.items():
        a = actual[k]
        assert type(a) is type(e) and (a == e or (e != e and a != a)), (k, a, e)


def _columns(reco, interactions):
    return ([np.ascontiguousarray(interactions[c], dtype=np.int64) for c in ("user_id", "item_id")]
            + [np.ascontiguousarray(reco[c], dtype=np.int64) for c in ("user_id", "item_id", "rank")])


CASES = [
    dict(seed=1),
    dict(seed=2, id_dtype=np.int32, max_test=20, hit_share=0.7, dup_share=0.3),
    dict(seed=3, id_dtype=np.uint32, k_reco=25, hit_share=0.6),
    dict(seed=4, shuffle=False, ragged=False),
    dict(seed=5, n_users=10, n_items=8, k_reco=8, max_test=30, hit_share=0.9, dup_share=0.4),
    dict(seed=6, extra_test_users=20, extra_reco_users=30, hit_share=0.2),
    dict(seed=11, n_users=40, n_items=300, k_reco=200, max_test=150, hit_share=0.9, dup_share=0.2),
    dict(seed=12, n_users=6, n_items=900, k_reco=800, max_test=700, hit_share=0.95, dup_share=0.1),
]


@pytest.mark.parametrize("case", CASES, ids=[str(c["seed"]) for c in CASES])
def test_seeded_cases(ref, case):  # pylint: disable=unused-argument,redefined-outer-name
    from rectools.metrics import calc_metrics as stock

    import rectools_b200
    from rectools_b200.metrics import device_metrics, ndcg_tables

    reco, interactions = metrics_cases.tables(**case)
    ks = (1, 3, 10, 40, 129, 800) if case.get("k_reco", 10) > 100 else (1, 3, 10, 40)
    metrics = metrics_cases.served_metrics(ks=ks)
    catalog = list(range(50_000))
    stats = {}
    _same(rectools_b200.calc_metrics(metrics, reco, interactions, catalog=catalog, stats=stats), stock(metrics, reco, interactions, catalog=catalog))
    assert stats["path"] == 10
    # the per-user arrays themselves, against the definition
    tables, _ = ndcg_tables(metrics)
    cols = _columns(reco, interactions)
    got = device_metrics(*cols, list(ks), tables, True)
    want = metrics_oracle.device_metrics_np(*cols, list(ks), tables, True)
    for key in ("users", "first_order", "liked", "min_rank", "tp"):
        np.testing.assert_array_equal(got[key], want[key], err_msg=key)
    for key in ("map", "ndcg"):
        np.testing.assert_array_equal(got[key].view(np.int64), want[key].view(np.int64), err_msg=key)
    assert got["flags"] == 0


@pytest.mark.parametrize("n_users", [10_000, 100_000, 1_000_000])
def test_random_tables_at_scale(ref, n_users):  # pylint: disable=unused-argument,redefined-outer-name
    from rectools.metrics import MAP, NDCG, calc_metrics as stock

    import rectools_b200

    reco, interactions = metrics_cases.large_tables(n_users, seed=n_users % 97)
    if n_users < 1_000_000:
        metrics = metrics_cases.served_metrics(ks=(1, 5, 10), log_bases=(2, 10))
    else:
        metrics = {**metrics_cases.nine_metrics(10), "map_k@5": MAP(k=5, divide_by_k=True),
                   "ndcg_ach@10": NDCG(k=10, log_base=3, divide_by_achievable=True)}
    catalog = np.arange(30_000)
    _same(rectools_b200.calc_metrics(metrics, reco, interactions, catalog=catalog), stock(metrics, reco, interactions, catalog=catalog))


def test_k_1000_and_a_user_with_1e5_rows(ref):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    from rectools.metrics import MAP, MRR, NDCG, Precision, Recall, calc_metrics as stock

    import rectools_b200

    rng = np.random.default_rng(7)
    n_users, k = 300, 1000
    users = np.arange(n_users, dtype=np.int64) * 5 + 1
    items = np.stack([rng.permutation(5000)[:k] for _ in range(n_users)])
    reco = pd.DataFrame({"user_id": np.repeat(users, k), "item_id": items.reshape(-1).astype(np.int64),
                         "rank": np.tile(np.arange(1, k + 1, dtype=np.int64), n_users)})
    big = 100_000  # user 0: 10^5 test rows, most of them repeats of its reco items
    rows_u = np.concatenate([np.zeros(big, np.int64), rng.integers(0, n_users, 20_000)])
    rows_i = np.where(rng.random(len(rows_u)) < 0.6, items[rows_u, rng.integers(0, k, len(rows_u))], rng.integers(0, 5000, len(rows_u)))
    p = rng.permutation(len(rows_u))
    interactions = pd.DataFrame({"user_id": users[rows_u[p]], "item_id": rows_i[p].astype(np.int64)})
    metrics = {}
    for kk in (1, 9, 129, 500, 1000):
        metrics.update({f"ndcg@{kk}": NDCG(k=kk), f"ndcg3a@{kk}": NDCG(k=kk, log_base=3, divide_by_achievable=True),
                        f"map@{kk}": MAP(k=kk), f"mapk@{kk}": MAP(k=kk, divide_by_k=True), f"mrr@{kk}": MRR(k=kk),
                        f"p@{kk}": Precision(k=kk), f"r@{kk}": Recall(k=kk)})
    _same(rectools_b200.calc_metrics(metrics, reco, interactions), stock(metrics, reco, interactions))


def test_duplicate_reco_pair_is_delegated(ref):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    from rectools.metrics import calc_metrics as stock

    import rectools_b200
    from rectools_b200.metrics import device_metrics

    reco, interactions = metrics_cases.tables(21)
    dup = pd.concat([reco, reco.iloc[[3]]], ignore_index=True)
    out = device_metrics(*_columns(dup, interactions), [3], [], False)
    assert out["flags"] == 1 and len(out["users"]) == 0
    rank0 = reco.copy()
    rank0.loc[5, "rank"] = 0
    assert device_metrics(*_columns(rank0, interactions), [3], [], False)["flags"] == 2
    nine = metrics_cases.nine_metrics(3)
    for table in (dup, rank0):
        _same(rectools_b200.calc_metrics(nine, table, interactions, catalog=list(range(5000))),
              stock(nine, table, interactions, catalog=list(range(5000))))


def test_known_answers(ref):  # pylint: disable=unused-argument,redefined-outer-name
    import pandas as pd
    import rectools.metrics as RM

    import rectools_b200

    fx = json.load(open(FIXTURE))
    for c in fx["per_user"]:
        spec = dict(c["metric"])
        m = getattr(RM, spec.pop("class"))(**spec)
        reco, inter = pd.DataFrame(c["reco"]), pd.DataFrame(c["interactions"])
        got = rectools_b200.calc_metrics({"m": m}, reco, inter, catalog=c["catalog"])
        assert np.isclose(got["m"], np.mean(c["expected"])), (c["metric"], got)
        _same(got, RM.calc_metrics({"m": m}, reco, inter, catalog=c["catalog"]))


def test_cross_validate_popular_and_als(ref, monkeypatch):  # pylint: disable=unused-argument,redefined-outer-name
    """`cross_validate` with a PopularModel and an ALS model (the stub's solver replaced by seeded factors), stock
    against `install(metrics=True)`: the same metrics for every fold and model."""
    import pandas as pd
    from implicit.cpu.als import AlternatingLeastSquares
    from rectools.dataset import Dataset
    from rectools.metrics import NDCG
    from rectools.model_selection import TimeRangeSplitter, cross_validate
    from rectools.models import ImplicitALSWrapperModel, PopularModel

    import rectools_b200

    def fit(self, user_items, show_progress=False, callback=None):  # pylint: disable=unused-argument
        rng = np.random.default_rng(self.random_state or 0)
        self.item_factors = rng.standard_normal((user_items.shape[1], self.factors)).astype(np.float32)
        self.user_factors = np.asarray(user_items @ self.item_factors, dtype=np.float32)

    monkeypatch.setattr(AlternatingLeastSquares, "fit", fit, raising=False)
    rng = np.random.default_rng(5)
    n = 60_000
    df = pd.DataFrame({"user_id": rng.integers(0, 3000, n), "item_id": rng.integers(0, 800, n), "weight": 1.0,
                       "datetime": pd.Timestamp("2021-01-01") + pd.to_timedelta(rng.integers(0, 60, n), unit="D")})
    dataset = Dataset.construct(df)
    splitter = TimeRangeSplitter(test_size="7D", n_splits=3, filter_already_seen=True)
    metrics = {**metrics_cases.nine_metrics(10), "ndcg_ach@5": NDCG(k=5, divide_by_achievable=True)}
    models = {"pop": PopularModel(), "als": ImplicitALSWrapperModel(AlternatingLeastSquares(factors=16, random_state=3))}
    kw = dict(dataset=dataset, splitter=splitter, metrics=metrics, models=models, k=10, filter_viewed=True)
    expected = cross_validate(**kw)
    rectools_b200.install(device=0, metrics=True)
    try:
        actual = cross_validate(**kw)
    finally:
        rectools_b200.uninstall()
    assert len(expected["metrics"]) == 6
    assert actual["metrics"] == expected["metrics"]

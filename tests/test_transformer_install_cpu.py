"""CPU: `install(transformers=True)` -- the module-level `TorchRanker` of the transformer similarity module (u2i) and of the
lightning module (item-to-item) rebound, with an oracle-backed stand-in (`OracleTorchRanker`) as the ranker, under the
UNMODIFIED SASRec / BERT4Rec / HSTU fitted through the `pytorch_lightning` stand-in (tests/lightning_stub).  The frames
must equal the stock frames (the stock scorer is the reference's own `TorchRanker`); near-ties of its fp32 arithmetic may
swap neighbours.  The GPU twin with the real engine is tests/test_gpu_transformer_install.py."""
import sys

import numpy as np
import pytest

from oracle import stage_reference
from tests import lightning_stub
from tests.helpers import OracleTorchRanker, assert_same_ranking

pytestmark = pytest.mark.skipif(not stage_reference.available(), reason="reference package not available")

SIM = "rectools.models.nn.transformers.similarity"
LIT = "rectools.models.nn.transformers.lightning"


@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    stub = lightning_stub.add_to_path()
    yield
    import rectools_b200

    rectools_b200.uninstall()
    lightning_stub.remove_from_path(stub)
    stage_reference.remove_from_path(added)


@pytest.fixture(scope="module")
def fitted(ref):
    from tests.transformer_cases import MODELS, build_model, dataset

    ds = dataset()
    return ds, {name: build_model(name).fit(ds) for name in MODELS}


def _stock():
    import importlib

    from rectools.models.rank import TorchRanker

    return TorchRanker, [importlib.import_module(m) for m in (SIM, LIT)]


def test_install_rebinds_both_names_and_uninstall_restores_them(ref):
    import rectools_b200

    stock, mods = _stock()
    rectools_b200.install()
    try:
        assert all(m.TorchRanker is stock for m in mods), "install() without transformers=True must leave both names stock"
    finally:
        rectools_b200.uninstall()
    rectools_b200.install(transformers=True)
    try:
        bound = [m.TorchRanker for m in mods]
        assert all(b is not stock for b in bound) and bound[0] is bound[1]
        rectools_b200.install(transformers=True)  # twice: uninstall still restores the stock class
    finally:
        rectools_b200.uninstall()
    assert all(m.TorchRanker is stock for m in mods)


def test_install_import_error_is_atomic(ref, monkeypatch):
    """Without `pytorch_lightning` the lightning module cannot be imported: the ImportError names the package and nothing
    (transformer names, `ImplicitRanker`s, methods) is rebound."""
    import rectools_b200
    from rectools.models import ease, vector
    from rectools.models.ease import EASEModel

    from rectools_b200 import integration

    stock, mods = _stock()
    before = (vector.ImplicitRanker, ease.ImplicitRanker, EASEModel.__dict__["_recommend_i2i"])
    monkeypatch.setitem(sys.modules, "pytorch_lightning", None)
    monkeypatch.delitem(sys.modules, LIT)
    with pytest.raises(ImportError, match="pytorch_lightning"):
        rectools_b200.install(transformers=True)
    assert (vector.ImplicitRanker, ease.ImplicitRanker, EASEModel.__dict__["_recommend_i2i"]) == before
    assert mods[0].TorchRanker is stock and mods[1].TorchRanker is stock
    assert not integration._ORIGINALS  # pylint: disable=protected-access


def _same_frames(exp, got, target_col):
    assert list(exp.columns) == list(got.columns)
    np.testing.assert_array_equal(exp[target_col].to_numpy(), got[target_col].to_numpy())
    np.testing.assert_array_equal(exp["rank"].to_numpy(), got["rank"].to_numpy())
    assert_same_ranking(got["item_id"].to_numpy(), got["score"].to_numpy(), exp["item_id"].to_numpy(), exp["score"].to_numpy(),
                        rtol=3e-5, atol=3e-6, tie_tol=3e-6)


def _calls(ds):
    items = ds.item_id_map.external_ids
    users = np.concatenate([[1], ds.user_id_map.external_ids[::3]])  # user 1 has viewed every item
    wl = items[::4]
    n_items = len(items)
    u2i = [dict(k=7, filter_viewed=True), dict(k=7, filter_viewed=False), dict(k=5, filter_viewed=True, items_to_recommend=wl),
           dict(k=n_items + 10, filter_viewed=True), dict(k=n_items + 10, filter_viewed=False, items_to_recommend=wl)]
    i2i = [dict(k=6, filter_itself=True), dict(k=6, filter_itself=False), dict(k=4, items_to_recommend=wl),
           dict(k=n_items + 10, filter_itself=False)]
    return users, items[::5], u2i, i2i


@pytest.mark.parametrize("name", ["sasrec", "bert4rec", "hstu"])
def test_installed_frames_equal_stock(fitted, name):
    import rectools_b200

    ds, models = fitted
    model = models[name]
    users, targets, u2i, i2i = _calls(ds)
    exp_u = [model.recommend(users, ds, **kw) for kw in u2i]
    exp_i = [model.recommend_to_items(targets, ds, **kw) for kw in i2i]
    rectools_b200.install(transformers=True, ranker_factory=OracleTorchRanker)
    try:
        got_u = [model.recommend(users, ds, **kw) for kw in u2i]
        got_i = [model.recommend_to_items(targets, ds, **kw) for kw in i2i]
    finally:
        rectools_b200.uninstall()
    for kw, e, g in zip(u2i, exp_u, got_u):
        assert len(e), kw
        _same_frames(e, g, "user_id")
        if kw["filter_viewed"]:
            assert not (g["user_id"] == 1).any(), "the user who viewed every item gets no rows"
    for e, g in zip(exp_i, got_i):
        assert len(e)
        _same_frames(e, g, "target_item_id")


@pytest.mark.parametrize("name", ["sasrec", "hstu"])
def test_config_round_trips_while_installed(fitted, name):
    """The stock similarity module ranks on the engine while installed, so the config stays that of the stock model."""
    import rectools_b200
    from rectools.models.nn.transformers.similarity import DistanceSimilarityModule

    _, models = fitted
    model = models[name]
    rectools_b200.install(transformers=True, ranker_factory=OracleTorchRanker)
    try:
        cfg = model.get_config(simple_types=True)
        assert cfg["similarity_module_type"] == "rectools.models.nn.transformers.similarity.DistanceSimilarityModule"
        again = type(model).from_config(cfg)
        assert again.get_config(simple_types=True) == cfg
        assert again.similarity_module_type is DistanceSimilarityModule
    finally:
        rectools_b200.uninstall()


def test_transformer_ranker_device_choice(ref):
    """Host factors rank on the installed device (only passed on when it is not the default); device tensors on their own
    device, or on the installed group when it contains that device."""
    from rectools_b200 import integration

    seen = []

    def factory(distance, device, subjects_factors, objects_factors, **kw):  # pylint: disable=unused-argument
        seen.append(kw.get("devices"))

    make = integration.transformer_ranker(factory)
    x = np.zeros((3, 2), np.float32)
    saved = integration.B200ImplicitRanker.default_device
    try:
        for installed, device, want in ((0, "cpu", None), (2, "cpu", 2), ((0, 1), "cpu", (0, 1)), ((0, 1), "cuda:1", (0, 1)),
                                        ((0, 1), "cuda:2", None), (1, "cuda:1", None), ((0, 0), "cuda", (0, 0))):
            integration.B200ImplicitRanker.default_device = installed
            seen.clear()
            make("dot", device, x, x)
            assert seen == [want], (installed, device)
    finally:
        integration.B200ImplicitRanker.default_device = saved

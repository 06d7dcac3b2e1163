"""GPU: SASRec / BERT4Rec / HSTU ranked on the engine through `install(transformers=True)` -- u2i through the stock
`DistanceSimilarityModule`, item-to-item through `TransformerLightningModule._recommend_i2i`, which passes one tensor as
both factors (the identity route of `B200TorchRanker`: no copy of the catalogue, the target rows gathered per call).

* the models end to end against stock `TorchRanker`, every engine row held to the rounding-interval oracle
  (`tests/score_interval.check_topk`) with no tolerance;
* the identity route bit for bit equal to the explicit-copy route (`subjects_factors=item_embs.clone()`) over DOT / COSINE,
  fp32 / fp16 / bf16 catalogues and every path, with and without a whitelist;
* its peak device memory, an engine group on one device, and the premise of its COSINE norms: a row's fp64 norm does not
  depend on how many rows the tensor has."""
import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests import lightning_stub
from tests.helpers import assert_same_ranking
from tests.score_interval import check_topk

pytestmark = pytest.mark.gpu

DTYPES = ("float32", "float16", "bfloat16")


def _torch_dtype(name):
    import torch

    return getattr(torch, name)


# ------------------------------------------------------------------------------------------- the norm premise
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", [16, 64, 256, 1000])
def test_row_norm_does_not_depend_on_row_count(dtype, d):
    """The identity route computes COSINE norms over the gathered rows only, the explicit route over the whole matrix:
    both are `torch.linalg.vector_norm(x.double(), dim=1)`, so they agree bit for bit only if a row's fp64 norm does not
    depend on the number of rows in the tensor."""
    import torch

    from rectools_b200.ranker import _device_norms

    g = torch.Generator(device="cuda:0").manual_seed(d)
    n = 20000
    x = (torch.randn((n, d), generator=g, device="cuda:0") * torch.rand((n, 1), generator=g, device="cuda:0") * 4).to(_torch_dtype(dtype))
    full64 = torch.linalg.vector_norm(x.double(), dim=1)
    full32 = _device_norms(x.to(torch.float32))
    rng = np.random.default_rng(d)
    for rows in (1, 2, 3, 7, 31, 128, 1000, 4097, n):
        idx = torch.from_numpy(np.sort(rng.choice(n, rows, replace=False))).to("cuda:0")
        part = x.index_select(0, idx)
        np.testing.assert_array_equal(torch.linalg.vector_norm(part.double(), dim=1).cpu().numpy().view(np.int64),
                                      full64[idx].cpu().numpy().view(np.int64), err_msg=f"{rows} rows")
        np.testing.assert_array_equal(_device_norms(part).view(np.int32), full32[idx.cpu().numpy()].view(np.int32))


# ------------------------------------------------------------------------------------------- identity vs explicit copy
CASES = {  # name: (n_targets, k, env, expected stats path)
    "path0": (100, 10, {}, 0),
    "path1_narrow": (600, 10, {}, 1),
    "path1_wide": (600, 100, {}, 1),
    "path3_k1025": (600, 1025, {}, 3),
    "path3_none": (300, None, {}, 3),
    "path3_passes": (600, 200, {"B200_WIDE": "0"}, 3),
    "path3_radix": (600, 200, {"B200_WIDE": "0", "B200_SELECT": "2"}, 3),
}
N_ITEMS, D = 20000, 64


@pytest.fixture(scope="module")
def catalogues():
    import torch

    g = torch.Generator(device="cuda:0").manual_seed(5)
    x = torch.randn((N_ITEMS, D), generator=g, device="cuda:0") / np.sqrt(D)
    x[7] = 0.0  # a zero row: COSINE norm 1e-10
    return {name: x.to(_torch_dtype(name)) for name in DTYPES}


def _bits(a):
    return a.view(np.int32) if a.dtype == np.float32 else a


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("restrict", [False, True])
def test_identity_route_equals_explicit_copy(catalogues, monkeypatch, case, dtype, distance, restrict):
    from rectools_b200 import B200TorchRanker

    n_targets, k, env, path = CASES[case]
    for name, value in env.items():
        monkeypatch.setenv(name, value)
    items = catalogues[dtype]
    rng = np.random.default_rng(n_targets)
    targets = rng.choice(N_ITEMS, n_targets, replace=False)
    targets[:2] = [7, targets[2]]  # the zero row, and a repeated target
    wl = filt = None
    if restrict:
        wl = np.sort(rng.choice(N_ITEMS, N_ITEMS // 2, replace=False))
        filt = sparse.random(n_targets, N_ITEMS, density=0.002, format="csr", random_state=1)
        filt.data[:] = 1.0
    ident = B200TorchRanker(distance, items.device, items, items)
    copy = B200TorchRanker(distance, items.device, items.clone(), items)
    assert ident._identity is not None and copy._identity is None  # pylint: disable=protected-access
    assert ident.subjects_norms is None
    got = ident.rank_padded(targets, k, filt, wl)
    st = dict(ident.last_stats)
    exp = copy.rank_padded(targets, k, filt, wl)
    assert st["path"] == copy.last_stats["path"] == path, (st["path"], copy.last_stats["path"])
    flat, flat_exp = ident.rank(targets, k, filt, wl), copy.rank(targets, k, filt, wl)
    for a, b in zip(got + flat, exp + flat_exp):
        assert a.dtype == b.dtype and a.shape == b.shape
        np.testing.assert_array_equal(_bits(a), _bits(b))
    if case in ("path0", "path1_narrow", "path1_wide"):
        rows = items.float().cpu().numpy()
        check_topk(got[1:], rows[targets], items.float().cpu().numpy(), k, cosine=distance == "cosine", filter_csr=filt,
                   whitelist=wl, name=f"{case}/{dtype}/{distance}")


def test_identity_route_candidate_sets_make_subjects_resident(catalogues):
    """Candidate-set calls rank resident subjects by id: an identity ranker makes its catalogue resident first, and then
    answers as the explicit route does."""
    import torch

    from rectools_b200 import B200TorchRanker

    items = catalogues["bfloat16"]
    ident = B200TorchRanker("cosine", items.device, items, items)
    copy = B200TorchRanker("cosine", items.device, items.clone(), items)
    g = torch.Generator(device=items.device).manual_seed(3)
    cand = torch.randint(-1, N_ITEMS, (50, 300), generator=g, device=items.device)
    targets = np.arange(50) * 13
    for a, b in zip(ident.rank_candidates_device(targets, cand, 20), copy.rank_candidates_device(targets, cand, 20)):
        np.testing.assert_array_equal(a.cpu().numpy(), b.cpu().numpy())
    assert ident._identity is None  # pylint: disable=protected-access
    for a, b in zip(ident.rank(targets, 20), copy.rank(targets, 20)):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_identity_route_peak_memory_below_fp32_catalogue(distance):
    """A bf16 catalogue: the identity route allocates far less than the catalogue's fp32 size on the device (no copy of
    the catalogue), the explicit-copy route at least that much (its fp32 subjects)."""
    import torch

    from rectools_b200 import B200TorchRanker

    n, d = 200_000, 256
    items = (torch.randn((n, d), device="cuda:0") / 16).to(torch.bfloat16)
    fp32_bytes = n * d * 4
    targets = np.arange(0, n, 97)
    peaks = {}
    for route in ("identity", "explicit"):
        subjects = items if route == "identity" else items.clone()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        ranker = B200TorchRanker(distance, items.device, subjects, items)
        out = ranker.rank(targets, 20)
        torch.cuda.synchronize()
        peaks[route] = torch.cuda.max_memory_allocated() - base
        assert len(out[1]) == 20 * len(targets)
        del ranker, subjects
    print(f"{distance}: peak above baseline {peaks}, fp32 catalogue {fp32_bytes}")
    assert peaks["identity"] < fp32_bytes // 8
    assert peaks["explicit"] >= fp32_bytes


# ------------------------------------------------------------------------------------------- the models end to end
@pytest.fixture(scope="module")
def fitted():
    if not stage_reference.available():
        pytest.skip("reference package not staged (oracle/_ref)")
    added = stage_reference.add_to_path()
    stub = lightning_stub.add_to_path()
    from tests.transformer_cases import MODELS, build_model, dataset

    ds = dataset(n_users=400, n_items=3000, per_user=15)
    models = {name: build_model(name, n_factors=32, device=None).fit(ds) for name in MODELS}
    yield ds, models
    import rectools_b200

    rectools_b200.uninstall()
    lightning_stub.remove_from_path(stub)
    stage_reference.remove_from_path(added)


def _checked_ranker():
    """`B200TorchRanker` that holds every padded engine answer to the rounding-interval oracle before it answers."""
    import torch

    from rectools_b200 import B200TorchRanker

    seen = []

    class Checked(B200TorchRanker):
        def __init__(self, distance, device, subjects_factors, objects_factors, *args, **kwargs):
            super().__init__(distance, device, subjects_factors, objects_factors, *args, **kwargs)
            host = lambda t: t.detach().to(torch.float32).cpu().numpy() if hasattr(t, "detach") else np.asarray(t, np.float32)
            self._check = (host(subjects_factors), host(objects_factors), self._identity is not None)

        def rank(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None):
            sub, obj, identity = self._check
            filt = filter_pairs_csr
            if filt is not None:
                filt = filt.copy()
                filt.eliminate_zeros()
            _, ids, scores, counts = self.rank_padded(subject_ids, k, filt, sorted_object_whitelist)
            check_topk((ids, scores, counts), sub[np.asarray(subject_ids)], obj, k, cosine=self.distance.value == "cosine",
                             filter_csr=filt, whitelist=sorted_object_whitelist, verbose=False)
            seen.append((identity, type(self.engine).__name__))
            return super().rank(subject_ids, k, filter_pairs_csr, sorted_object_whitelist)

    return Checked, seen


def _calls(ds, model):
    items = ds.item_id_map.external_ids
    users = np.concatenate([[1], ds.user_id_map.external_ids[::2]])
    wl = items[::3]
    u2i = [dict(k=10, filter_viewed=True), dict(k=10, filter_viewed=False), dict(k=30, filter_viewed=True, items_to_recommend=wl),
           dict(k=len(items) + 5, filter_viewed=True)]
    i2i = [dict(k=10, filter_itself=True), dict(k=10, filter_itself=False), dict(k=40, items_to_recommend=wl)]
    known = model.data_preparator.get_known_item_ids()  # targets must be items of the model's sessions
    return users, known[::4], u2i, i2i


def _same_frames(exp, got, target_col):
    assert list(exp.columns) == list(got.columns)
    np.testing.assert_array_equal(exp[target_col].to_numpy(), got[target_col].to_numpy())
    np.testing.assert_array_equal(exp["rank"].to_numpy(), got["rank"].to_numpy())
    assert_same_ranking(got["item_id"].to_numpy(), got["score"].to_numpy(), exp["item_id"].to_numpy(), exp["score"].to_numpy(),
                        rtol=3e-5, atol=3e-6, tie_tol=3e-6)


@pytest.mark.parametrize("name", ["sasrec", "bert4rec", "hstu"])
def test_models_through_install_match_stock_torch_ranker(fitted, name):
    import rectools_b200

    ds, models = fitted
    model = models[name]
    users, targets, u2i, i2i = _calls(ds, model)
    exp_u = [model.recommend(users, ds, **kw) for kw in u2i]
    exp_i = [model.recommend_to_items(targets, ds, **kw) for kw in i2i]
    checked, seen = _checked_ranker()
    rectools_b200.install(transformers=True, ranker_factory=checked)
    try:
        got_u = [model.recommend(users, ds, **kw) for kw in u2i]
        got_i = [model.recommend_to_items(targets, ds, **kw) for kw in i2i]
        # the default factory (B200TorchRanker) gives the same frames as the checked one
        rectools_b200.install(transformers=True)
        again_u, again_i = model.recommend(users, ds, **u2i[0]), model.recommend_to_items(targets, ds, **i2i[0])
    finally:
        rectools_b200.uninstall()
    assert seen == [(False, "Engine")] * len(u2i) + [(True, "Engine")] * len(i2i), "u2i: two tensors; i2i: the identity route"
    for e, g in zip(exp_u, got_u):
        assert len(e)
        _same_frames(e, g, "user_id")
    for e, g in zip(exp_i, got_i):
        assert len(e)
        _same_frames(e, g, "target_item_id")
    assert again_u.equals(got_u[0]) and again_i.equals(got_i[0])


def test_engine_group_on_one_device_gives_the_same_frames(fitted):
    import rectools_b200

    ds, models = fitted
    frames = {}
    for device in (0, [0, 0]):
        checked, seen = _checked_ranker()
        rectools_b200.install(device=device, transformers=True, ranker_factory=checked)
        try:
            frames[str(device)] = []
            for model in models.values():
                users, targets, u2i, i2i = _calls(ds, model)
                frames[str(device)] += [model.recommend(users, ds, **u2i[2]), model.recommend_to_items(targets, ds, **i2i[2])]
        finally:
            rectools_b200.uninstall()
        assert {s[1] for s in seen} == {"Engine" if device == 0 else "EngineGroup"}
    for a, b in zip(frames["0"], frames["[0, 0]"]):
        assert len(a) and a.equals(b)

"""GPU: LightFM, BPR and DSSM ranked on the engine through `install()`, every engine row held to the rounding-interval
oracle with no tolerance (the case table and the checks: tests/vector_model_cases.py; its CPU twin with an oracle
ranker: tests/test_vector_models_cpu.py).  Each call prints its route: path, tensor-core launches, fallback and
exhaustive rows, and the ambiguous entries of the check.

* bias-folded LightFM (DOT d + 2, COSINE d + 1 at d = 30, 64, 318, 319: both sides of a 64-column block and of the
  tensor-core limit d_pad = 320), small and dominant user biases (exact fp32 ties across the cut), k = 1 ... 1025 and
  above the catalogue, filters, whitelists, `filter_itself`, features with hot / warm / cold targets;
* BPR (implicit's bias column), DSSM (EUCLIDEAN u2i and i2i);
* ALS with `recommend_use_gpu_ranking=True`: the unmodified `ImplicitRanker._rank_on_gpu` through `patch_implicit_gpu()`;
* the baseline shape: LightFM, 138 493 users x 26 744 items, 64 components, k = 10, sampled rows checked, the share of
  rows the certificate sent to the fallback printed."""
import subprocess

import numpy as np
import pytest

from oracle import stage_reference
from tests import lightfm_stub, lightning_stub
from tests.score_interval import check_topk

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not stage_reference.available(), reason="reference package not staged (oracle/_ref)")]


@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    stubs = (lightfm_stub.add_to_path(), lightning_stub.add_to_path())
    yield
    import rectools_b200

    rectools_b200.uninstall()
    lightning_stub.remove_from_path(stubs[1])
    lightfm_stub.remove_from_path(stubs[0])
    stage_reference.remove_from_path(added)


def _card():
    import torch

    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return f"{torch.cuda.get_device_name(0)}, power limit {power}"


@pytest.mark.parametrize("name", ["lightfm_30_small", "lightfm_30_dominant", "lightfm_64_small", "lightfm_64_dominant",
                                  "lightfm_318_small", "lightfm_318_dominant", "lightfm_319_small", "lightfm_319_dominant",
                                  "lightfm_features", "bpr", "dssm"])
def test_vector_models_through_install(ref, name):
    from rectools_b200 import integration
    from tests.vector_model_cases import run_case

    for line in run_case(name, "gpu", integration.B200ImplicitRanker):
        print(line)


def _factors(n, d, seed):
    return (np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32) / np.sqrt(d)).astype(np.float32)


def test_als_gpu_ranking_seam(ref):
    """`recommend_use_gpu_ranking=True`: the unmodified `ImplicitRanker` ranks through `implicit.gpu.KnnQuery` on the
    engine (`patch_implicit_gpu()`); every call it makes is checked.  Both seams rank on the engine with its own object
    norms, so the ids equal those of `install()`; the scores too wherever the reference's subject norm
    (`np.linalg.norm` in fp32) equals the engine ranker's (fp32 of the fp64 norm).  The rows where they differ are
    counted and printed."""
    import rectools_b200
    from rectools_b200 import implicit_gpu
    from tests.ref_models import injected_als, synthetic_dataset

    n_users, n_items, d = 3000, 6000, 64
    ds = synthetic_dataset(n_users, n_items, 30, seed=5)
    model = injected_als(_factors(n_users, d, 11), _factors(n_items, d, 12))
    model.recommend_use_gpu_ranking = True
    users = np.random.default_rng(1).permutation(ds.user_id_map.external_ids)[:2500]
    targets = ds.item_id_map.external_ids[::5]
    seen = []

    def backend(items, queries, k, item_norms, csr):
        out = implicit_gpu._engine_backend(items, queries, k, item_norms, csr)  # pylint: disable=protected-access
        rep = check_topk(out, queries, items, k, cosine=item_norms is not None, filter_csr=csr, verbose=False,
                         name=f"implicit.gpu seam k={k} cosine={item_norms is not None}")
        seen.append((item_norms is not None, csr is not None, len(queries), rep.n_ambiguous))
        return out

    implicit_gpu.patch_implicit_gpu(backend=backend)
    try:
        seam_u = model.recommend(users, ds, k=10, filter_viewed=True)
        seam_i = model.recommend_to_items(targets, ds, k=10)
    finally:
        implicit_gpu.unpatch_implicit_gpu()
    assert [s[:3] for s in seen] == [(False, True, len(users)), (True, False, len(targets))], seen
    print(f"implicit.gpu seam calls (cosine, filter, rows, ambiguous): {seen}")
    rectools_b200.install()
    try:
        ours_u = model.recommend(users, ds, k=10, filter_viewed=True)
        ours_i = model.recommend_to_items(targets, ds, k=10)
    finally:
        rectools_b200.uninstall()
    for seam, ours, col in ((seam_u, ours_u, "user_id"), (seam_i, ours_i, "target_item_id")):
        assert list(seam.columns) == list(ours.columns) and len(seam) == len(ours)
        np.testing.assert_array_equal(seam[col].to_numpy(), ours[col].to_numpy())
        np.testing.assert_array_equal(seam["item_id"].to_numpy(), ours["item_id"].to_numpy())
    np.testing.assert_array_equal(seam_u["score"].to_numpy().astype(np.float32), ours_u["score"].to_numpy().astype(np.float32))
    # i2i COSINE: the subject norms of the two seams, per target
    items32 = model.model.item_factors
    tid = ds.item_id_map.convert_to_internal(seam_i["target_item_id"].to_numpy())
    ref_norm = np.linalg.norm(items32, axis=1)
    eng_norm = np.sqrt(np.einsum("ij,ij->i", items32.astype(np.float64), items32.astype(np.float64))).astype(np.float32)
    agree = ref_norm[tid] == eng_norm[tid]
    a, b = seam_i["score"].to_numpy(), ours_i["score"].to_numpy()
    np.testing.assert_array_equal(np.asarray(a, np.float32)[agree], np.asarray(b, np.float32)[agree])
    t_all = ds.item_id_map.convert_to_internal(targets)
    n_diff = int((ref_norm[t_all] != eng_norm[t_all]).sum())
    n_score = int((np.asarray(a, np.float32) != np.asarray(b, np.float32)).sum())
    print(f"i2i COSINE: the two subject norms differ on {n_diff} of {len(targets)} targets; {n_score} of {len(a)} scores differ")
    assert n_score <= int((~agree).sum())


def test_baseline_shape(ref):
    """LightFM at the shape of BASELINE.md: 138 493 users x 26 744 items, 64 components (DOT d = 66), k = 10, no
    filter, heavy-tailed item norms and biases.  4096 sampled rows are held to the rounding-interval oracle; the share of
    rows the certificate sent to the fallback is printed (no timing)."""
    import rectools_b200
    from rectools_b200 import integration
    from tests.ref_models import injected_lightfm, synthetic_dataset
    from tests.vector_model_cases import _expected_vectors, recording_ranker

    n_users, n_items, nc, k = 138_493, 26_744, 64, 10
    ds = synthetic_dataset(n_users, n_items, 3, seed=7)
    rng = np.random.default_rng(8)
    ue = rng.standard_normal((n_users, nc)) / np.sqrt(nc) * rng.lognormal(0.0, 0.3, (n_users, 1))
    ie = rng.standard_normal((n_items, nc)) / np.sqrt(nc) * rng.lognormal(0.0, 0.8, (n_items, 1))
    ub, ib = 0.5 * rng.standard_t(3, n_users), 0.5 * rng.standard_t(3, n_items)
    model = injected_lightfm(ds, ue, ie, ub, ib)
    users = ds.user_id_map.external_ids
    log = []
    saved = integration.B200ImplicitRanker
    integration.B200ImplicitRanker = recording_ranker(saved, log)
    try:
        rectools_b200.install()
        frame = model.recommend(users, ds, k=k, filter_viewed=False)
    finally:
        rectools_b200.uninstall()
        integration.B200ImplicitRanker = saved
    assert len(log) == 1 and len(frame) == n_users * k
    rec = log[0]
    st = rec["stats"]
    assert rec["d_pad"] == 128 and st["path"] == 1, (rec["d_pad"], st)
    _, _, s_aug, o_aug = _expected_vectors(model, ds, "u2i")
    rows = np.sort(np.random.default_rng(9).choice(n_users, 4096, replace=False))
    rep = check_topk((rec["ids"][rows], rec["scores"][rows], rec["counts"][rows]), s_aug[rec["sids"][rows]], o_aug, k,
                     name="baseline shape, 4096 sampled rows")
    print(f"baseline shape on {_card()}: path {st['path']}, {st['n_tc_launches']} tensor-core launches, "
          f"{st['n_fallback_rows']} of {n_users} rows fell back ({st['n_fallback_rows'] / n_users:.4%}), "
          f"{st.get('n_exact_rows')} ranked exhaustively; ambiguous {rep.n_ambiguous}")

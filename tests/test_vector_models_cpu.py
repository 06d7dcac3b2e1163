"""CPU: the case table of tests/vector_model_cases.py -- the unmodified `LightFMWrapperModel` (bias-folded DOT / COSINE,
d = 30 ... 319 + the fold, small and dominant biases, features with hot / warm / cold targets), `ImplicitBPRWrapperModel`
(implicit's bias column) and `DSSMModel` (EUCLIDEAN) through `install()` -- with an oracle-backed ranker in place of the
engine (`OracleImplicitRanker`).  The GPU twin with the real engine is tests/test_gpu_vector_models.py.

The mutation test shows that the checks bite: a provider that swaps two tied ids, moves one score by one ulp, filters
with the next user's row or leaves out the COSINE subject-norm division must fail them."""
import numpy as np
import pytest

from oracle import stage_reference
from tests import lightfm_stub, lightning_stub

pytestmark = pytest.mark.skipif(not stage_reference.available(), reason="reference package not available")


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


CASES = ["lightfm_30_small", "lightfm_30_dominant", "lightfm_64_small", "lightfm_64_dominant", "lightfm_318_dominant",
         "lightfm_319_small", "lightfm_features", "bpr", "dssm"]


@pytest.mark.parametrize("name", CASES)
def test_vector_models_through_install(ref, name):
    from tests.vector_model_cases import OracleImplicitRanker, run_case

    for line in run_case(name, "cpu", OracleImplicitRanker):
        print(line)


def test_case_table_covers_the_issue_shapes(ref):
    """Every LightFM width and bias kind is in the table the GPU test runs, and the CPU runs one of each width."""
    from tests.vector_model_cases import LIGHTFM, MODELS

    assert {nc for nc, _ in LIGHTFM.values()} == {30, 64, 318, 319} and set(LIGHTFM) <= set(MODELS)
    assert {LIGHTFM[c][0] for c in CASES if c in LIGHTFM} == {30, 64, 318, 319}


@pytest.mark.parametrize("mutation, name, call", [
    ("swap_tied", "lightfm_30_dominant", 3),  # k = 129 without the filter: exact ties inside the rows
    ("ulp", "lightfm_30_small", 1),
    ("next_filter", "lightfm_30_small", 0),  # k = 1 with the filter
    ("no_norm", "lightfm_30_small", -3),  # i2i COSINE
])
def test_checks_catch_a_mutated_provider(ref, mutation, name, call):
    import rectools_b200
    from rectools_b200 import integration
    from tests.vector_model_cases import OracleImplicitRanker, build, calls, check_case, invoke, recording_ranker

    model, ds = build(name, "cpu")
    kind, kw = calls(name, ds)[call]
    if mutation == "next_filter":
        assert kind == "u2i" and kw["filter_viewed"]
    if mutation == "no_norm":
        assert kind == "i2i" and str(getattr(model.i2i_dist, "value", model.i2i_dist)) == "cosine"
    stock = invoke(model, ds, kind, kw)

    def ranked(mut):
        class Provider(OracleImplicitRanker):
            mutation = mut
            applied = [0]

        frames, logs = {}, {}
        for fast in (True, False):
            logs[fast] = []
            saved = integration.B200ImplicitRanker
            integration.B200ImplicitRanker = recording_ranker(Provider, logs[fast])
            try:
                rectools_b200.install(fast_recommend=fast)
                frames[fast] = invoke(model, ds, kind, kw)
            finally:
                rectools_b200.uninstall()
                integration.B200ImplicitRanker = saved
        return frames, logs, Provider.applied[0]

    frames, logs, _ = ranked(None)
    check_case(model, ds, kind, kw, stock, frames, logs, label="unmutated")  # the same call passes unmutated
    frames, logs, applied = ranked(mutation)
    assert applied > 0, f"{mutation} changed nothing"
    with pytest.raises(AssertionError):
        check_case(model, ds, kind, kw, stock, frames, logs, label=mutation)


def test_oracle_provider_matches_the_reference_ranker(ref):
    """The CPU provider is the engine's definition: its flat answers equal the unmodified `ImplicitRanker`'s (stub top-k)
    on integer-valued factors, where every score is exact (ties ordered by id on both sides)."""
    from rectools.models.rank import Distance, ImplicitRanker
    from scipy import sparse

    from tests.vector_model_cases import OracleImplicitRanker

    rng = np.random.default_rng(3)
    u = rng.integers(-4, 5, (50, 6)).astype(np.float32)
    i = rng.integers(-4, 5, (300, 6)).astype(np.float32)
    filt = sparse.random(50, 300, density=0.05, format="csr", random_state=2)
    filt.data[:] = 1
    wl = np.sort(rng.choice(300, 200, replace=False))
    for dist in (Distance.DOT, Distance.EUCLIDEAN):
        for f, w in ((None, None), (filt, wl)):
            exp = ImplicitRanker(dist, u, i).rank(np.arange(50), 7, f, w)
            got = OracleImplicitRanker(dist, u, i).rank(np.arange(50), 7, f, w)
            for a, b in zip(exp, got):
                np.testing.assert_array_equal(np.asarray(a), np.asarray(b))

"""CPU: scored pairs (engine path 6, `b200_rank_topk_pairs`, `rectools_b200.rerank`) up to where a GPU is needed.

- the export is declared, exported and bound, the ABI stays 6 and the engine-group exports are unchanged;
- the order key and the stable per-group top-k, restated in numpy (tests/pairs_oracle.py), against the unmodified
  reference `Reranker.recommend`: +-0 ties, NaN tails, -inf, NA users, string and float user ids, extra columns, an
  existing `rank` column, the empty frame;
- the host logic of `reranker_recommend` with the library replaced by a recording stand-in: what is delegated to the
  original method, the codes and offsets handed over, and `install(rerank=True)` / `uninstall()`."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from oracle import stage_reference
from tests.pairs_oracle import rank_pairs_np, reranker_recommend_np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
needs_ref = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_export_declared_exported_and_bound():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    assert re.search(r"\bint b200_rank_topk_pairs\s*\(", header)
    for name, value in (("F64", 0), ("F32", 1), ("I64", 2), ("I32", 3)):
        assert re.search(rf"#define B200_PAIRS_{name} {value}\b", header)
        assert getattr(_lib, f"PAIRS_{name}") == value
    assert "b200_rank_topk_pairs" in _lib.EXPORTS
    assert "#define B200_RANK_ABI_VERSION 6" in header and _lib.ABI_VERSION == 6
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = C.CDLL(_lib.LIB_PATH)
    assert lib.b200_rank_topk_pairs is not None
    assert lib.b200_rank_abi_version() == 6
    assert _lib.load().b200_rank_topk_pairs.argtypes is not None


def test_group_exports_unchanged():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    group = sorted(set(re.findall(r"\b(b200_rank_group_[a-z_]+)\s*\(", header)))
    assert group == sorted(
        ["b200_rank_group_create", "b200_rank_group_create_ex", "b200_rank_group_destroy", "b200_rank_group_get_info",
         "b200_rank_group_set_subjects", "b200_rank_group_topk"]
    )
    assert sorted(e for e in _lib.EXPORTS if e.startswith("b200_rank_group_")) == group


# ------------------------------------------------------------------------------------------- the restatement vs reference
@pytest.fixture(scope="module")
def ref():
    added = stage_reference.add_to_path()
    from rectools.models.ranking.candidate_ranking import Reranker

    yield Reranker
    stage_reference.remove_from_path(added)


def _frames():
    import pandas as pd

    nan, inf = np.nan, np.inf
    yield "special", pd.DataFrame({
        "user_id": [1, 1, 1, 1, 2, 2, 2, 3, 3, 3, 3],
        "item_id": np.arange(11),
        "score": [2.0, -inf, nan, nan, -0.0, 0.0, -1.0, inf, nan, 5.0, -inf],
    }), 3
    yield "na_users_float_ids", pd.DataFrame({
        "user_id": [1.5, np.nan, 1.5, None, 7.25, 7.25, 1.5],
        "item_id": np.arange(7),
        "score": [0.1, 9.0, 0.3, 8.0, -1.0, 1.0, 0.2],
    }), 2
    yield "string_ids_extra_cols_rank", pd.DataFrame({
        "user_id": ["b", "a", "b", "c", "a", "b", None],
        "item_id": ["x", "y", "z", "x", "w", "v", "u"],
        "score": np.array([3, -2, 5, 1, 7, 4, 9], dtype=np.int64),
        "feature": np.arange(7, dtype=np.float32),
        "rank": np.arange(7, dtype=np.int64) * 10,
    }), 2
    yield "fp32_scores", pd.DataFrame({
        "user_id": np.repeat(np.arange(4), 5),
        "item_id": np.arange(20),
        "score": np.random.default_rng(0).permutation(20).astype(np.float32) - np.float32(10),
    }), 4
    yield "int32_extremes", pd.DataFrame({
        "user_id": [0, 0, 0, 1, 1],
        "item_id": np.arange(5),
        "score": np.array([np.iinfo(np.int32).min, np.iinfo(np.int32).max, 0, -1, 1], dtype=np.int32),
    }), 2
    rng = np.random.default_rng(1)
    n = 3000
    yield "random", pd.DataFrame({
        "user_id": rng.integers(0, 200, n) * 7 + 3,
        "item_id": rng.integers(0, 1000, n),
        "score": rng.random(n),
    }), 10


@needs_ref
@pytest.mark.parametrize("add_rank_col", [True, False])
def test_restatement_matches_reference(ref, add_rank_col):
    import pandas as pd

    for name, df, k in _frames():
        expected = ref.recommend(df, k, add_rank_col)
        got = reranker_recommend_np(df, k, add_rank_col)
        pd.testing.assert_frame_equal(got, expected, obj=name)


@needs_ref
def test_restatement_matches_reference_on_the_empty_frame(ref):
    import pandas as pd

    df = pd.DataFrame({"user_id": np.array([], np.int64), "item_id": np.array([], np.int64), "score": np.array([], np.float64)})
    for add_rank_col in (True, False):
        pd.testing.assert_frame_equal(reranker_recommend_np(df, 5, add_rank_col), ref.recommend(df, 5, add_rank_col))


def test_restatement_orders_by_key_then_position():
    codes = np.array([0, 0, 0, 0, 0, -1, 1])
    scores = np.array([1.0, np.nan, 1.0, -np.inf, -0.0, 9.0, 0.0])
    pos, off = rank_pairs_np(codes, scores, 10, 2)
    np.testing.assert_array_equal(pos, [0, 2, 4, 3, 1, 6])
    np.testing.assert_array_equal(off, [0, 5, 6])
    ints = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, -1, 0], dtype=np.int64)
    pos, _ = rank_pairs_np(np.zeros(4, np.int64), ints, 4, 1)
    np.testing.assert_array_equal(pos, [1, 3, 2, 0])


# ---------------------------------------------------------------------------------------------- host logic (stand-in lib)
class RecordingLib:
    """`b200_rank_topk_pairs` computed by the numpy restatement; records the arguments it was handed."""

    def __init__(self):
        self.calls = []

    def b200_rank_topk_pairs(self, device, stream, n, codes_p, scores_p, stype, n_groups, k, flags, out_pos, out_offsets, stats):
        dt = {0: np.float64, 1: np.float32, 2: np.int64, 3: np.int32}[stype]
        codes = np.ctypeslib.as_array(C.cast(codes_p, C.POINTER(C.c_int64)), (n,)).copy() if n else np.zeros(0, np.int64)
        ctype = {np.float64: C.c_double, np.float32: C.c_float, np.int64: C.c_int64, np.int32: C.c_int32}[dt]
        scores = np.ctypeslib.as_array(C.cast(scores_p, C.POINTER(ctype)), (n,)).copy() if n else np.zeros(0, dt)
        self.calls.append(dict(device=device, n=n, codes=codes, scores=scores, stype=stype, n_groups=n_groups, k=k, flags=flags))
        pos, off = rank_pairs_np(codes, scores, k, n_groups)
        np.ctypeslib.as_array(C.cast(out_offsets, C.POINTER(C.c_int64)), (n_groups + 1,))[:] = off
        if len(pos):
            np.ctypeslib.as_array(C.cast(out_pos, C.POINTER(C.c_int64)), (len(pos),))[:] = pos
        stats._obj.path = 6  # pylint: disable=protected-access
        return 0

    def b200_rank_last_error(self):
        return b""


@pytest.fixture()
def lib(monkeypatch, ref):
    from rectools_b200 import _lib

    rec = RecordingLib()
    monkeypatch.setattr(_lib, "_LIB", rec)
    yield rec


@needs_ref
def test_codes_and_offsets_handed_over(lib, ref):
    import pandas as pd
    from rectools_b200 import reranker_recommend

    df = pd.DataFrame({"user_id": ["u2", "u1", None, "u2", "u3", "u1"], "item_id": np.arange(6),
                       "score": [0.5, 0.25, 1.0, 0.75, -1.0, 0.0]})
    stats = {}
    got = reranker_recommend(df, 1, device=3, stats=stats)
    pd.testing.assert_frame_equal(got, ref.recommend(df, 1))
    (call,) = lib.calls
    np.testing.assert_array_equal(call["codes"], [0, 1, -1, 0, 2, 1])
    np.testing.assert_array_equal(call["scores"], df["score"].to_numpy())
    assert (call["device"], call["n"], call["n_groups"], call["k"], call["flags"], call["stype"]) == (3, 6, 3, 1, 0, 0)
    assert stats["path"] == 6


@needs_ref
@pytest.mark.parametrize("dtype,stype", [(np.float64, 0), (np.float32, 1), (np.int64, 2), (np.int32, 3)])
def test_score_dtypes_are_handed_over_unchanged(lib, ref, dtype, stype):
    import pandas as pd
    from rectools_b200 import reranker_recommend

    df = pd.DataFrame({"user_id": [0, 0, 1, 0], "item_id": np.arange(4), "score": np.array([3, 1, 2, 3], dtype=dtype)})
    pd.testing.assert_frame_equal(reranker_recommend(df, 2), ref.recommend(df, 2))
    assert lib.calls[-1]["stype"] == stype and lib.calls[-1]["scores"].dtype == dtype


@needs_ref
def test_k_is_clamped_to_the_row_count(lib, ref):
    import pandas as pd
    from rectools_b200 import reranker_recommend

    df = pd.DataFrame({"user_id": [0, 1, 0], "item_id": np.arange(3), "score": [1.0, 2.0, 3.0]})
    pd.testing.assert_frame_equal(reranker_recommend(df, 10**12), ref.recommend(df, 10**12))
    assert lib.calls[-1]["k"] == 3


def _same_outcome(got_fn, expected_fn):
    """The same frame, or the same exception type and message."""
    import pandas as pd

    try:
        expected = expected_fn()
    except Exception as e:  # pylint: disable=broad-except
        with pytest.raises(type(e), match=re.escape(str(e))):
            got_fn()
        return
    pd.testing.assert_frame_equal(got_fn(), expected)


@needs_ref
def test_delegated_cases_go_to_the_original_method(lib, ref):
    import pandas as pd
    from rectools_b200 import reranker_recommend

    base = pd.DataFrame({"user_id": [0, 0, 1, 1, 0], "item_id": np.arange(5), "score": [0.5, 0.1, 0.3, 0.9, 0.7]})
    cases = [
        (base.assign(score=[True, False, True, True, False]), 2),
        (base.assign(score=pd.array([0.5, 0.1, None, 0.9, 0.7], dtype="Float64")), 2),
        (base.assign(score=pd.array([5, 1, 3, 9, 7], dtype="Int64")), 2),
        (base.assign(score=np.array([0.5, 0.1, 0.3, 0.9, 0.7], dtype=object)), 2),
        (base.assign(user_id=pd.Categorical([0, 0, 1, 1, 0])), 2),
        (base, 2.0),
        (base, True),
    ]
    for df, k in cases + [(base, 0), (base, -3)]:  # k < 1: the reference's own answer (head() of a negative count)
        _same_outcome(lambda: reranker_recommend(df, k), lambda: ref.recommend(df, k))
    assert lib.calls == []


@needs_ref
def test_install_rerank_rebinds_and_uninstall_restores(lib, ref):
    import pandas as pd
    import rectools_b200 as rb
    from rectools.models.ranking.candidate_ranking import Reranker

    original = Reranker.__dict__["recommend"]
    df = pd.DataFrame({"user_id": [5, 5, 6], "item_id": np.arange(3), "score": [0.1, 0.2, 0.3]})
    try:
        rb.install()  # the default leaves Reranker alone
        assert Reranker.__dict__["recommend"] is original
        rb.uninstall()
        rb.install(device=[2, 1], rerank=True)
        assert Reranker.__dict__["recommend"] is not original
        assert isinstance(Reranker.__dict__["recommend"], classmethod)
        got = Reranker.recommend(df, 1)
        pd.testing.assert_frame_equal(got, original.__get__(None, Reranker)(df, 1))
        assert lib.calls[-1]["device"] == 2  # the home device of a group
        # delegated calls reach the original, not the rebound method
        n_calls = len(lib.calls)
        _same_outcome(lambda: Reranker.recommend(df, 1.5), lambda: original.__get__(None, Reranker)(df, 1.5))
        assert len(lib.calls) == n_calls
    finally:
        rb.uninstall()
    assert Reranker.__dict__["recommend"] is original


def test_rank_pairs_refuses_bad_arguments():
    from rectools_b200 import rank_pairs

    with pytest.raises(ValueError, match="positive int"):
        rank_pairs(np.zeros(3, np.int64), np.zeros(3), 0)
    with pytest.raises(TypeError, match="float64, float32, int64 or int32"):
        rank_pairs(np.zeros(3, np.int64), np.zeros(3, np.float16), 1)
    with pytest.raises(ValueError, match="length"):
        rank_pairs(np.zeros(3, np.int64), np.zeros(4), 1)

"""CPU: candidate sets (engine path 5, `b200_rank_topk_candidates`) up to the point where a GPU is needed.

- the export is declared, exported and bound, and the ABI stays 6;
- tests/cand_plan_driver.cpp prints `plan_candidates` (rectools_b200/csrc/plan.h): row chunks by the candidates and k_out
  of their rows, the sort-scratch boundary at LK_SMEM_PAIRS, the row that fits no chunk, every refusal, and the check of
  the candidate ids;
- `normalize_candidates`: unsorted rows, repeated ids, empty rows, the whitelist, the caller's matrix left as it was, and
  the ValueErrors;
- `rectools_b200.ann` with an oracle-backed ranker against the unmodified `rectools.tools.ann` classes, which import here
  through the brute-force nmslib stand-in of oracle/nmslib_stub (skipped when the reference package is not staged)."""
import ctypes
import os
import pickle
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
NMSLIB_STUB = os.path.join(ROOT, "oracle", "nmslib_stub")

OK, INVALID, NOMEM, UNSUPPORTED = 0, -1, -3, -4
INPUTS_ON_DEVICE, OUTPUTS_ON_DEVICE, FORCE_EXACT, FORCE_TC, SHARED_THRESHOLDS = 1, 2, 4, 8, 16
S = 12288  # LK_SMEM_PAIRS, rectools_b200/csrc/sizes.h
GIB = 1 << 30


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_export_declared_exported_and_bound():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    assert re.search(r"\bint b200_rank_topk_candidates\s*\(", header)
    assert "b200_rank_topk_candidates" in _lib.EXPORTS
    assert "#define B200_RANK_ABI_VERSION 6" in header and _lib.ABI_VERSION == 6
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert lib.b200_rank_topk_candidates is not None
    assert lib.b200_rank_abi_version() == 6
    assert _lib.load().b200_rank_topk_candidates.argtypes is not None


def test_engine_group_refuses_candidate_sets():
    from rectools_b200.ranker import EngineGroup

    with pytest.raises(NotImplementedError, match="engine group"):
        EngineGroup.topk_candidates(object.__new__(EngineGroup), 10, np.zeros(1), np.zeros(0))


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
        exe = os.path.join(tmp, "cand_plan_driver")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cand_plan_driver.cpp")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(cases):
            lines = []
            for c in cases:
                c = {"n_objects": 1_000_000, "k": 100, "d": 128, **c}
                if "lens" in c and not isinstance(c["lens"], str):
                    c["n_rows"] = c.get("n_rows", len(c["lens"]))
                    c["lens"] = ",".join(str(x) for x in c["lens"])
                if "ids" in c:
                    c["ids"] = ",".join(str(x) for x in c["ids"])
                lines.append(" ".join(f"{k}={v}" for k, v in c.items()))
            out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
            plans = []
            for ln in out.splitlines():
                head, _, message = ln.partition(" message=")
                p = {}
                for w in head.split():
                    k, v = w.split("=")
                    p[k] = [int(x) for x in v.split(",") if x] if k == "bounds" else int(v)
                p["message"] = message
                plans.append(p)
            assert len(plans) == len(cases)
            return plans

        yield run


def plan(driver, **case):
    return driver([case])[0]


def row_bytes(n, k_out):
    return 4 * n + (16 * n if k_out > S else 0) + 8 * k_out


def test_one_chunk_for_small_calls(driver):
    p = plan(driver, lens=[1000] * 100, k=100)
    assert (p["error"], p["ids_error"], p["k_out"], p["n_chunks"], p["bounds"]) == (OK, OK, 100, 1, [0, 100])
    assert p["max_chunk_cands"] == 100_000 and p["max_chunk_rows"] == 100


def test_k_out_is_min_of_k_and_the_catalogue(driver):
    assert plan(driver, lens=[3], k=10, n_objects=5)["k_out"] == 5
    assert plan(driver, lens=[3], k=10**9, n_objects=1_000_000)["k_out"] == 1_000_000


def test_chunks_by_candidates_within_the_budget(driver):
    # 10 rows of 100 candidates, k_out = 10: 480 B per row; a budget of 1000 B holds two rows
    lens = [100] * 10
    p = plan(driver, lens=lens, k=10, budget=1000)
    assert row_bytes(100, 10) == 480
    assert p["bounds"] == [0, 2, 4, 6, 8, 10] and p["n_chunks"] == 5 and p["max_chunk_cands"] == 200
    # ragged rows: chunks close before the row that would overflow
    p = plan(driver, lens=[200, 10, 10, 200, 0, 0, 200], k=10, budget=1000)
    assert row_bytes(200, 10) == 880 and row_bytes(10, 10) == 120 and row_bytes(0, 10) == 80
    assert p["bounds"] == [0, 2, 4, 6, 7]  # 880 + 120 fill a chunk exactly; 80 + 80 + 880 do not
    assert p["max_chunk_cands"] == 210 and p["max_chunk_rows"] == 2
    # the engine's 1 GiB: 65 536 rows of 1000 candidates at k = 100 (4.8 KB per row) fit in one chunk
    p = plan(driver, lens="1000," * 65536, n_rows=65536, k=100)
    assert p["n_chunks"] == 1


def test_chunk_rows_hook(driver):
    p = plan(driver, lens=[5] * 1000, k=10, B200_CHUNK_ROWS=256)
    assert p["bounds"] == [0, 256, 512, 768, 1000] and p["max_chunk_rows"] == 256
    # (the hook is at least 256 rows)
    assert plan(driver, lens=[5] * 1000, k=10, B200_CHUNK_ROWS=10)["n_chunks"] == 4
    # and a budget still splits within it
    assert plan(driver, lens=[5] * 1000, k=10, B200_CHUNK_ROWS=256, budget=100 * row_bytes(5, 10))["max_chunk_rows"] == 100


@pytest.mark.parametrize("k_out", [S - 1, S, S + 1])
def test_sort_scratch_boundary(driver, k_out):
    n = 50_000
    p = plan(driver, lens=[n], k=k_out, budget=10**9)
    assert p["k_out"] == k_out and p["error"] == OK
    # the scratch is taken only above S: exactly one row's bytes as the budget fits, one byte less does not
    exact = row_bytes(n, k_out)
    assert (exact - 4 * n - 8 * k_out > 0) == (k_out > S)
    assert plan(driver, lens=[n, n], k=k_out, budget=exact)["bounds"] == [0, 1, 2]
    assert plan(driver, lens=[n], k=k_out, budget=exact - 1)["error"] == NOMEM


def test_a_row_longer_than_a_chunk_is_refused(driver):
    p = plan(driver, lens=[10, 300_000_000], k=10)  # 1.2 GB of scores
    assert p["error"] == NOMEM and "row 1" in p["message"] and "300000000 candidates" in p["message"]
    p = plan(driver, lens=[10, 60_000_000], k=20_000)  # 20 B per candidate above S: 1.2 GB
    assert p["error"] == NOMEM
    assert plan(driver, lens=[10, 60_000_000], k=100)["error"] == OK  # 240 MB without the scratch


@pytest.mark.parametrize(
    "case, code, words",
    [
        ({"flags": INPUTS_ON_DEVICE}, UNSUPPORTED, "host inputs"),
        ({"flags": OUTPUTS_ON_DEVICE}, UNSUPPORTED, "host inputs"),
        ({"res_device": 1}, UNSUPPORTED, "device memory"),
        ({"sparse": 1}, UNSUPPORTED, "sub_"),
        ({"rows": 1}, UNSUPPORTED, "object_rows"),
        ({"whitelist": 1}, UNSUPPORTED, "whitelist"),
        ({"flags": SHARED_THRESHOLDS}, UNSUPPORTED, "SHARED_THRESHOLDS"),
        ({"flags": FORCE_TC}, UNSUPPORTED, "FORCE_TC"),
        ({"id_offset": 1}, UNSUPPORTED, "id offset"),
        ({"d": 49153}, UNSUPPORTED, "d = 49153"),
        ({"lens": "-", "n_rows": 2}, INVALID, "cand_indptr is NULL"),
    ],
)
def test_refusals(driver, case, code, words):
    p = plan(driver, **{"lens": [3, 4], **case})
    assert p["error"] == code and words in p["message"], p


def test_refusals_come_before_the_rows(driver):
    # a refused call is refused whatever its rows hold, and before they are read
    assert plan(driver, lens="-", n_rows=2, flags=INPUTS_ON_DEVICE)["error"] == UNSUPPORTED
    # empty calls are no error
    assert plan(driver, lens=[], n_rows=0)["error"] == OK
    assert plan(driver, lens=[], n_rows=0)["n_chunks"] == 0


def test_force_exact_changes_nothing(driver):
    a, b = driver([{"lens": [3, 4, 5], "k": 2}, {"lens": [3, 4, 5], "k": 2, "flags": FORCE_EXACT}])
    assert a == b and a["error"] == OK


def test_candidate_ids_are_checked(driver):
    ok = plan(driver, lens=[3, 0, 2], ids=[0, 5, 99, 1, 2], n_objects=100)
    assert ok["error"] == OK and ok["ids_error"] == OK
    p = plan(driver, lens=[3, 2], ids=[0, 5, 5, 1, 2], n_objects=100)
    assert p["ids_error"] == INVALID and "row 0" in p["message"] and "strictly ascending" in p["message"]
    p = plan(driver, lens=[3, 2], ids=[0, 5, 6, 2, 1], n_objects=100)
    assert p["ids_error"] == INVALID and "row 1" in p["message"]
    p = plan(driver, lens=[1, 2], ids=[0, 5, 100], n_objects=100)
    assert p["ids_error"] == INVALID and "candidate 100" in p["message"]
    p = plan(driver, lens=[1, 2], ids=[-1, 5, 6], n_objects=100)
    assert p["ids_error"] == INVALID and "candidate -1" in p["message"]
    # ascending across rows is not required
    assert plan(driver, lens=[2, 2], ids=[5, 6, 0, 1], n_objects=100)["ids_error"] == OK


def test_indptr_must_be_monotone(driver):
    p = plan(driver, lens=[3, -1, 2], n_rows=3)
    assert p["error"] == INVALID and "not monotone at row 1" in p["message"]


def test_existing_plans_untouched():
    """`plan_call` / `plan_rows` are pinned by their own drivers and tests, which this feature leaves as they were."""
    src = open(os.path.join(ROOT, "rectools_b200", "csrc", "plan.h")).read()
    assert "inline CallPlan plan_call(const CallShape& s, const Hooks& h)" in src
    assert "inline CallPlan plan_rows(const CallShape& s, const Hooks& h)" in src


# -------------------------------------------------------------------------------------------------------- normalisation
def test_normalisation_sorts_deduplicates_and_keeps_the_caller_matrix():
    from rectools_b200.ranker import normalize_candidates

    indptr = np.array([0, 4, 4, 7, 8])
    indices = np.array([9, 2, 9, 0, 5, 1, 3, 7], dtype=np.int32)
    data = np.array([1, 0, 2, 3, 4, 5, 6, 0], dtype=np.float32)  # stored zeros still count: rows are structure
    m = sparse.csr_matrix((data, indices, indptr), shape=(4, 10))
    before = (m.indptr.copy(), m.indices.copy(), m.data.copy())
    ip, ix = normalize_candidates(m, 4, 10)
    assert ip.dtype == np.int64 and ix.dtype == np.int32
    assert ip.tolist() == [0, 3, 3, 6, 7]
    assert ix.tolist() == [0, 2, 9, 1, 3, 5, 7]
    for a, b in zip(before, (m.indptr, m.indices, m.data)):
        np.testing.assert_array_equal(a, b)
    # whitelist intersection
    ip, ix = normalize_candidates(m, 4, 10, np.array([1, 2, 7, 9]))
    assert ip.tolist() == [0, 2, 2, 3, 4] and ix.tolist() == [2, 9, 1, 7]
    # other sparse formats are taken by their structure as well
    ip2, ix2 = normalize_candidates(m.tocoo(), 4, 10)
    assert ip2.tolist() == [0, 3, 3, 6, 7] and ix2.tolist() == [0, 2, 9, 1, 3, 5, 7]


def test_normalisation_errors():
    from rectools_b200.ranker import normalize_candidates

    m = sparse.csr_matrix((np.ones(2), [1, 3], [0, 1, 2]), shape=(2, 20))
    with pytest.raises(ValueError, match=r"Number of rows in `candidates_csr` must be equal to `len\(subject_ids\)`"):
        normalize_candidates(m, 3, 20)
    with pytest.raises(ValueError, match=r"must be in \[0, 3\)"):
        normalize_candidates(m, 2, 3)
    ip, ix = normalize_candidates(sparse.csr_matrix((2, 0)), 2, 5)  # no candidates at all
    assert ip.tolist() == [0, 0, 0] and len(ix) == 0


# ------------------------------------------------------------------------------------------------- ANN classes vs reference
class OracleCandRanker:
    """CPU stand-in with the ranker surface `rectools_b200.ann` uses (`rank_padded`, `rank_candidates_padded`), backed by the
    fp64 oracle: a candidate set is the complement filter, as the GPU tests express it."""

    def __init__(self, distance, subjects_factors, objects_factors):
        self._dist = str(getattr(distance, "value", distance))
        self._u = np.asarray(subjects_factors, dtype=np.float32)
        self._i = np.asarray(objects_factors, dtype=np.float32)

    def _padded(self, subject_ids, k, allowed):
        from oracle.topk_oracle import rank_oracle

        n_obj = self._i.shape[0]
        k_out = min(k, n_obj)
        ids = np.full((len(subject_ids), k_out), -1, np.int32)
        scores = np.full((len(subject_ids), k_out), -np.finfo(np.float32).max, np.float32)
        counts = np.zeros(len(subject_ids), np.int32)
        for r, sid in enumerate(subject_ids):
            banned = np.setdiff1d(np.arange(n_obj), allowed[r])
            filt = sparse.csr_matrix((np.ones(len(banned)), banned, [0, len(banned)]), shape=(1, n_obj))
            _, oi, os_ = rank_oracle(self._dist, self._u, self._i, [sid], k, filt, accum="f64")
            counts[r] = len(oi)
            ids[r, : len(oi)], scores[r, : len(oi)] = oi, os_
        return np.asarray(subject_ids), ids, scores, counts

    def rank_padded(self, subject_ids, k=None, filter_pairs_csr=None):
        n_obj = self._i.shape[0]
        allowed = []
        for r in range(len(subject_ids)):
            banned = filter_pairs_csr[r].indices if filter_pairs_csr is not None else []
            allowed.append(np.setdiff1d(np.arange(n_obj), banned))
        return self._padded(subject_ids, k, allowed)

    def rank_candidates_padded(self, subject_ids, candidates_csr, k=None):
        from rectools_b200.ranker import normalize_candidates

        ip, ix = normalize_candidates(candidates_csr, len(subject_ids), self._i.shape[0])
        return self._padded(subject_ids, k, [ix[ip[r] : ip[r + 1]] for r in range(len(subject_ids))])


needs_reference = pytest.mark.skipif(not stage_reference.available(), reason="reference package neither staged nor checked out")


@pytest.fixture(scope="module")
def ref_ann():
    added = stage_reference.add_to_path()
    sys.path.insert(0, NMSLIB_STUB)
    from rectools.tools import ann  # the unmodified module, on the brute-force nmslib stand-in

    yield ann
    sys.path.remove(NMSLIB_STUB)
    sys.modules.pop("nmslib", None)
    stage_reference.remove_from_path(added)


def _as_lists(res):
    return [list(np.asarray(x).tolist()) for x in res]


FIXTURE_ITEMS = np.array([[1, 1, 1, 1, 1], [2, 2, 2, 2, 2], [1, 2, 3, 4, 5], [6, 7, 8, 9, 10], [11, 12, 13, 14, 15]])
FIXTURE_USERS = np.array([[0, 0, 0, 0, 1], [5, 4, 3, 2, 1], [1, 1, 1, 1, 1]])


def _pair(ref_ann, kind, space, users, items, index_top_k=None):
    from rectools_b200 import ann as b200_ann

    n_items = len(items)
    item_map = {str(i): i for i in range(n_items)}
    params = {"method": "hnsw", "space": space}
    ktop = n_items if index_top_k is None else index_top_k
    if kind == "u2i":
        user_map = {f"u{i}": i for i in range(len(users))}
        ref = ref_ann.UserToItemAnnRecommender(users, items, user_map, item_map, index_top_k=ktop, index_init_params=params).fit()
        got = b200_ann.B200UserToItemAnnRecommender(users, items, user_map, item_map, index_top_k=ktop, index_init_params=params,
                                                   ranker_factory=OracleCandRanker).fit()
    else:
        ref = ref_ann.ItemToItemAnnRecommender(items, item_map, index_top_k=ktop, index_init_params=params).fit()
        got = b200_ann.B200ItemToItemAnnRecommender(items, item_map, index_top_k=ktop, index_init_params=params,
                                                   ranker_factory=OracleCandRanker).fit()
    return ref, got


@needs_reference
@pytest.mark.parametrize("space", ["cosinesimil", "negdotprod", "l2"])
def test_fixture_i2i_matches_reference(ref_ann, space):
    ref, got = _pair(ref_ann, "i2i", space, None, FIXTURE_ITEMS)
    for top_n in (1, 2, 4, 10):
        assert list(got.get_item_list_for_item("0", top_n)) == list(ref.get_item_list_for_item("0", top_n))
        avail = ["1", "2", "4", "4"]
        assert list(got.get_item_list_for_item("3", top_n, avail)) == list(ref.get_item_list_for_item("3", top_n, avail))
        batch, lists = ["0", "1", "3"], [["1", "2", "3", "4"], ["0", "4"], ["2", "2"]]
        assert _as_lists(got.get_item_list_for_item_batch(batch, top_n, lists)) == _as_lists(ref.get_item_list_for_item_batch(batch, top_n, lists))
        assert _as_lists(got.get_item_list_for_item_batch(batch, top_n)) == _as_lists(ref.get_item_list_for_item_batch(batch, top_n))


@needs_reference
@pytest.mark.parametrize("space", ["cosinesimil", "negdotprod", "l2"])
def test_fixture_u2i_matches_reference(ref_ann, space):
    ref, got = _pair(ref_ann, "u2i", space, FIXTURE_USERS, FIXTURE_ITEMS)
    for top_n in (1, 2, 5, 8):
        assert list(got.get_item_list_for_user("u0", top_n)) == list(ref.get_item_list_for_user("u0", top_n))
        assert list(got.get_item_list_for_user("u1", top_n, ["4", "0", "0"])) == list(ref.get_item_list_for_user("u1", top_n, ["4", "0", "0"]))
        users, lists = ["u2", "u0", "u2"], [["0", "1", "2"], [], ["3", "4"]]
        assert _as_lists(got.get_item_list_for_user_batch(users, top_n, lists)) == _as_lists(ref.get_item_list_for_user_batch(users, top_n, lists))
        assert _as_lists(got.get_item_list_for_user_batch(users, top_n)) == _as_lists(ref.get_item_list_for_user_batch(users, top_n))


@needs_reference
@pytest.mark.parametrize("space", ["cosinesimil", "negdotprod", "l2"])
@pytest.mark.parametrize("kind", ["u2i", "i2i"])
def test_random_tie_free_inputs_match_reference(ref_ann, space, kind):
    rng = np.random.default_rng(7)
    n_items, n_users, d = 300, 40, 16
    items = rng.standard_normal((n_items, d)).astype(np.float32)
    users = rng.standard_normal((n_users, d)).astype(np.float32)
    ref, got = _pair(ref_ann, kind, space, users, items)
    targets = [f"u{i}" for i in range(n_users)] if kind == "u2i" else [str(i) for i in rng.choice(n_items, 25, replace=False)]
    lists = [[str(x) for x in rng.choice(n_items, rng.integers(0, 60), replace=True)] for _ in targets]
    call = "get_item_list_for_user_batch" if kind == "u2i" else "get_item_list_for_item_batch"
    for top_n in (1, 10, 50):
        assert _as_lists(getattr(got, call)(targets, top_n, lists)) == _as_lists(getattr(ref, call)(targets, top_n, lists))
        assert _as_lists(getattr(got, call)(targets, top_n)) == _as_lists(getattr(ref, call)(targets, top_n))


@needs_reference
def test_i2i_lists_exclude_every_target_of_the_batch(ref_ann):
    ref, got = _pair(ref_ann, "i2i", "cosinesimil", None, FIXTURE_ITEMS)
    lists = [["0", "1", "2", "3", "4"], ["0", "1", "2", "3", "4"]]
    want = [["4", "3"], ["4", "3"]]  # neither 0 nor 1, for either row (the reference's own fixture answer)
    assert _as_lists(ref.get_item_list_for_item_batch(["0", "1"], 2, lists)) == want
    assert _as_lists(got.get_item_list_for_item_batch(["0", "1"], 2, lists)) == want
    # without lists only the row's own item goes: row "0" gets "1" back
    assert list(got.get_item_list_for_item_batch(["0", "1"], 1)[0]) == ["1"]


@needs_reference
def test_short_lists_and_unknown_ids(ref_ann):
    ref, got = _pair(ref_ann, "u2i", "negdotprod", FIXTURE_USERS, FIXTURE_ITEMS)
    assert list(got.get_item_list_for_user("u0", 3, ["2"])) == ["2"]  # min(top_n, |allowed|)
    assert list(got.get_item_list_for_user("u0", 3, [])) == []
    with pytest.raises(KeyError):
        ref.get_item_list_for_user("nobody", 3)
    with pytest.raises(KeyError):
        got.get_item_list_for_user("nobody", 3)
    with pytest.raises(KeyError):
        got.get_item_list_for_user("u0", 3, ["no such item"])


@needs_reference
@pytest.mark.parametrize("kind", ["u2i", "i2i"])
def test_pickling(ref_ann, kind):
    ref, got = _pair(ref_ann, kind, "cosinesimil", FIXTURE_USERS, FIXTURE_ITEMS)
    call = (lambda r: r.get_item_list_for_user_batch(["u0", "u1"], 3, [["0", "3", "4"], ["1"]])) if kind == "u2i" else (
        lambda r: r.get_item_list_for_item_batch(["0", "2"], 3, [["1", "3", "4"], ["1"]]))
    before = _as_lists(call(got))
    state = got.__getstate__()
    assert state["_ranker"] is None  # the engine is not pickled
    loaded = pickle.loads(pickle.dumps(got))
    assert loaded._ranker is None  # pylint: disable=protected-access
    assert _as_lists(call(loaded)) == before == _as_lists(call(ref))
    assert loaded.index_top_k == got.index_top_k and loaded.distance == got.distance


@needs_reference
def test_constructor_refusals(ref_ann):  # pylint: disable=unused-argument
    from rectools_b200 import ann as b200_ann

    with pytest.raises(ValueError, match="space"):
        b200_ann.B200ItemToItemAnnRecommender(FIXTURE_ITEMS, {str(i): i for i in range(5)}, index_init_params={"space": "jaccard"})
    with pytest.raises(ValueError, match="index"):
        b200_ann.B200ItemToItemAnnRecommender(FIXTURE_ITEMS, {str(i): i for i in range(5)}, index=object())
    with pytest.raises(ValueError, match="shape mismatch"):
        b200_ann.B200UserToItemAnnRecommender(np.ones((2, 3)), FIXTURE_ITEMS, {"a": 0, "b": 1}, {str(i): i for i in range(5)})

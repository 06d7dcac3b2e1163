"""CPU: candidate sets from device memory (engine path 5, `b200_rank_topk_candidates_device`) up to where a GPU is needed.

- the export is declared, exported and bound, the ABI stays 6 and the engine-group exports are unchanged;
- tests/cand_device_plan_driver.cpp prints `plan_candidates_device` (rectools_b200/csrc/plan.h): chunk bounds against the
  byte rule for host and device outputs, rows around LK_SMEM_PAIRS (the preparation's and the selection's scratch), the
  B200_CHUNK_ROWS hook, a row above the budget, every refusal and refusals before the rows are read, any indptr base; and
  `plan_candidates` of the host route, which shares the chunk loop, still returns its plans;
- the Python argument handling that needs no GPU."""
import ctypes
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

OK, INVALID, NOMEM, UNSUPPORTED = 0, -1, -3, -4
INPUTS_ON_DEVICE, OUTPUTS_ON_DEVICE, FORCE_EXACT, FORCE_TC, SHARED_THRESHOLDS = 1, 2, 4, 8, 16
DEV = INPUTS_ON_DEVICE
S = 12288  # LK_SMEM_PAIRS, rectools_b200/csrc/sizes.h
GIB = 1 << 30


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_export_declared_exported_and_bound():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    assert re.search(r"\bint b200_rank_topk_candidates_device\s*\(", header)
    assert "b200_rank_topk_candidates_device" in _lib.EXPORTS
    assert "#define B200_RANK_ABI_VERSION 6" in header and _lib.ABI_VERSION == 6
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200rank.so is not built")
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert lib.b200_rank_topk_candidates_device is not None
    assert lib.b200_rank_abi_version() == 6
    assert _lib.load().b200_rank_topk_candidates_device.argtypes is not None


def test_group_exports_unchanged():
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    group = sorted(set(re.findall(r"\b(b200_rank_group_[a-z_]+)\s*\(", header)))
    assert group == sorted(
        ["b200_rank_group_create", "b200_rank_group_create_ex", "b200_rank_group_destroy", "b200_rank_group_get_info",
         "b200_rank_group_set_subjects", "b200_rank_group_topk"]
    )
    assert sorted(e for e in _lib.EXPORTS if e.startswith("b200_rank_group_")) == group


def test_engine_group_refuses_device_candidate_sets():
    from rectools_b200.ranker import EngineGroup

    with pytest.raises(NotImplementedError, match="engine group"):
        EngineGroup.topk_candidates_device(object.__new__(EngineGroup), 10, None, None)


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
        exe = os.path.join(tmp, "cand_device_plan_driver")
        src = os.path.join(ROOT, "tests", "cand_device_plan_driver.cpp")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, src], env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(cases):
            lines = []
            for c in cases:
                c = {"n_objects": 1_000_000, "k": 100, "d": 128, "flags": DEV, **c}
                if "lens" in c and not isinstance(c["lens"], str):
                    c["n_rows"] = c.get("n_rows", len(c["lens"]))
                    c["lens"] = ",".join(str(x) for x in c["lens"])
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


def dev_row_bytes(n, k_out, host_out):
    return 8 * n + (16 * n if n > S else 0) + (16 * n if k_out > S else 0) + (8 * k_out if host_out else 0)


def test_one_chunk_for_small_calls(driver):
    for flags in (DEV, DEV | OUTPUTS_ON_DEVICE):
        p = plan(driver, lens=[1000] * 100, k=100, flags=flags)
        assert (p["error"], p["k_out"], p["n_chunks"], p["bounds"]) == (OK, 100, 1, [0, 100])
        assert p["max_chunk_cands"] == 100_000 and p["max_chunk_rows"] == 100


@pytest.mark.parametrize("host_out", [True, False])
def test_chunks_follow_the_byte_rule(driver, host_out):
    flags = DEV if host_out else DEV | OUTPUTS_ON_DEVICE
    rng = np.random.default_rng(int(host_out))
    lens = [int(x) for x in rng.integers(0, 400, 60)]
    budget = 4000  # (a row of 399 entries takes 3272 B with host outputs)
    p = plan(driver, lens=lens, k=10, budget=budget, flags=flags)
    assert p["error"] == OK
    b = p["bounds"]
    assert b[0] == 0 and b[-1] == len(lens)
    for c0, c1 in zip(b[:-1], b[1:]):
        used = sum(dev_row_bytes(n, 10, host_out) for n in lens[c0:c1])
        assert used <= budget
        if c1 < len(lens):  # a chunk closes only before the row that would overflow it
            assert used + dev_row_bytes(lens[c1], 10, host_out) > budget
    assert p["max_chunk_cands"] == max(sum(lens[c0:c1]) for c0, c1 in zip(b[:-1], b[1:]))
    assert p["max_chunk_rows"] == max(c1 - c0 for c0, c1 in zip(b[:-1], b[1:]))


def test_host_outputs_add_their_staging(driver):
    # 10 rows of 100 entries, k_out = 10: 800 B per row with device outputs, 880 B with host outputs
    assert dev_row_bytes(100, 10, False) == 800 and dev_row_bytes(100, 10, True) == 880
    assert plan(driver, lens=[100] * 10, k=10, budget=1600, flags=DEV | OUTPUTS_ON_DEVICE)["bounds"] == [0, 2, 4, 6, 8, 10]
    assert plan(driver, lens=[100] * 10, k=10, budget=1600, flags=DEV)["bounds"] == list(range(11))
    # the engine's 1 GiB: 65 536 rows of 1000 entries at k = 100 fit in one chunk
    assert plan(driver, lens="1000," * 65536, n_rows=65536, k=100)["n_chunks"] == 1


@pytest.mark.parametrize("n", [S - 1, S, S + 1])
def test_preparation_scratch_boundary(driver, n):
    # rows longer than S sort in 16 B per entry of global scratch
    exact = dev_row_bytes(n, 10, False)
    assert (exact - 8 * n > 0) == (n > S)
    flags = DEV | OUTPUTS_ON_DEVICE
    assert plan(driver, lens=[n, n], k=10, budget=exact, flags=flags)["bounds"] == [0, 1, 2]
    assert plan(driver, lens=[n], k=10, budget=exact - 1, flags=flags)["error"] == NOMEM


@pytest.mark.parametrize("k_out", [S - 1, S, S + 1])
def test_selection_scratch_boundary(driver, k_out):
    n = 100
    exact = dev_row_bytes(n, k_out, True)
    assert (exact - 8 * n - 8 * k_out > 0) == (k_out > S)
    p = plan(driver, lens=[n, n], k=k_out, budget=exact)
    assert p["k_out"] == k_out and p["bounds"] == [0, 1, 2]
    assert plan(driver, lens=[n], k=k_out, budget=exact - 1)["error"] == NOMEM


def test_both_scratch_terms_add_up(driver):
    n, k_out = 20_000, S + 1
    exact = dev_row_bytes(n, k_out, False)
    assert exact == 8 * n + 16 * n + 16 * n
    flags = DEV | OUTPUTS_ON_DEVICE
    assert plan(driver, lens=[n], k=k_out, budget=exact, flags=flags)["error"] == OK
    assert plan(driver, lens=[n], k=k_out, budget=exact - 1, flags=flags)["error"] == NOMEM


def test_chunk_rows_hook(driver):
    p = plan(driver, lens=[5] * 1000, k=10, B200_CHUNK_ROWS=256)
    assert p["bounds"] == [0, 256, 512, 768, 1000] and p["max_chunk_rows"] == 256
    assert plan(driver, lens=[5] * 1000, k=10, B200_CHUNK_ROWS=10)["n_chunks"] == 4  # (at least 256 rows)
    assert plan(driver, lens=[5] * 1000, k=10, B200_CHUNK_ROWS=256, budget=100 * dev_row_bytes(5, 10, True))["max_chunk_rows"] == 100


def test_a_row_above_the_budget_is_refused(driver):
    p = plan(driver, lens=[10, 100_000_000], k=10)  # 8 B + 16 B per entry: 2.4 GB
    assert p["error"] == NOMEM and "row 1" in p["message"] and "100000000 candidates" in p["message"]
    assert p["message"].startswith("b200_rank_topk_candidates_device: ")
    assert plan(driver, lens=[10, 40_000_000], k=10)["error"] == OK  # 960 MB


def test_any_indptr_base(driver):
    a, b = driver([{"lens": [3, 0, 7], "base": 0}, {"lens": [3, 0, 7], "base": 12345}])
    assert a == b and a["error"] == OK
    p = plan(driver, lens=[3, 4], base=-1)
    assert p["error"] == INVALID and "cand_indptr[0] < 0" in p["message"]


@pytest.mark.parametrize(
    "case, code, words",
    [
        ({"flags": 0}, INVALID, "b200_rank_topk_candidates"),
        ({"flags": OUTPUTS_ON_DEVICE}, INVALID, "B200_Q_INPUTS_ON_DEVICE"),
        ({"sparse": 1}, UNSUPPORTED, "sub_"),
        ({"rows": 1}, UNSUPPORTED, "object_rows"),
        ({"whitelist": 1}, UNSUPPORTED, "whitelist"),
        ({"flags": DEV | SHARED_THRESHOLDS}, UNSUPPORTED, "SHARED_THRESHOLDS"),
        ({"flags": DEV | FORCE_TC}, UNSUPPORTED, "FORCE_TC"),
        ({"id_offset": 1}, UNSUPPORTED, "id offset"),
        ({"d": 49153}, UNSUPPORTED, "d = 49153"),
        ({"lens": "-", "n_rows": 2}, INVALID, "cand_indptr is NULL"),
        ({"lens": [3, -1]}, INVALID, "not monotone at row 1"),
    ],
)
def test_refusals(driver, case, code, words):
    p = plan(driver, **{"lens": [3, 4], **case})
    assert p["error"] == code and words in p["message"], p
    assert p["message"].startswith("b200_rank_topk_candidates_device: ")


def test_refusals_come_before_the_rows(driver):
    # a refused call is refused whatever its rows hold, and before they are read
    for case in ({"flags": 0}, {"whitelist": 1}, {"flags": DEV | FORCE_TC}, {"d": 49153}):
        assert plan(driver, lens="-", n_rows=2, **case)["error"] in (INVALID, UNSUPPORTED)
        assert "NULL" not in plan(driver, lens="-", n_rows=2, **case)["message"]
    # resident subjects in device memory are read here
    assert plan(driver, lens=[3, 4], res_device=1)["error"] == OK
    # empty calls are no error, and read no row
    assert plan(driver, lens="-", n_rows=0)["error"] == OK
    assert plan(driver, lens="-", n_rows=0)["n_chunks"] == 0
    assert plan(driver, lens="-", n_rows=3, n_objects=0)["error"] == OK


def test_force_exact_changes_nothing(driver):
    a, b = driver([{"lens": [3, 4, 5], "k": 2}, {"lens": [3, 4, 5], "k": 2, "flags": DEV | FORCE_EXACT}])
    assert a == b and a["error"] == OK


def test_host_plan_is_unchanged(driver):
    # plan_candidates shares the chunk loop: its plans, messages and refusals are those it always had
    def host(**c):
        return plan(driver, route="host", flags=0, **c)

    p = host(lens=[200, 10, 10, 200, 0, 0, 200], k=10, budget=1000)
    assert p["bounds"] == [0, 2, 4, 6, 7] and p["max_chunk_cands"] == 210 and p["max_chunk_rows"] == 2
    assert host(lens=[5] * 1000, k=10, B200_CHUNK_ROWS=256)["bounds"] == [0, 256, 512, 768, 1000]
    p = host(lens=[10, 300_000_000], k=10)
    assert p["error"] == NOMEM and p["message"].startswith("b200_rank_topk_candidates: row 1 (300000000 candidates, k_out = 10)")
    assert host(lens=[3, -1])["message"] == "b200_rank_topk_candidates: cand_indptr is not monotone at row 1"
    assert host(lens="-", n_rows=2)["message"] == "b200_rank_topk_candidates: cand_indptr is NULL"
    assert plan(driver, route="host", flags=INPUTS_ON_DEVICE, lens=[3])["error"] == UNSUPPORTED
    assert host(lens=[3], res_device=1)["error"] == UNSUPPORTED


# --------------------------------------------------------------------------------------------------------------- Python
def test_ranker_refusals_need_no_gpu():
    from rectools_b200.ranker import B200Ranker, EngineGroup

    r = object.__new__(B200Ranker)
    r._subjects_csr = object()  # pylint: disable=protected-access
    with pytest.raises(NotImplementedError, match="sparse"):
        r.rank_candidates_device(np.arange(2), None)
    r._subjects_csr = None  # pylint: disable=protected-access
    r.engine = object.__new__(EngineGroup)
    with pytest.raises(NotImplementedError, match="engine group"):
        r.rank_candidates_device(np.arange(2), None)


def test_ranker_takes_cuda_candidates_only():
    torch = pytest.importorskip("torch")
    from rectools_b200.ranker import B200Ranker, Engine

    r = object.__new__(B200Ranker)
    r._subjects_csr = None  # pylint: disable=protected-access
    r.engine = object.__new__(Engine)
    r.engine.device = 0
    with pytest.raises(TypeError, match="CUDA tensor"):
        r.rank_candidates_device(np.arange(2), torch.zeros((2, 3), dtype=torch.int32))
    with pytest.raises(TypeError, match="CUDA tensor"):
        r.rank_candidates_device(np.arange(2), np.zeros((2, 3), np.int32))


def test_engine_takes_cuda_inputs_only():
    torch = pytest.importorskip("torch")
    from rectools_b200.ranker import Engine

    e = object.__new__(Engine)
    e.device, e.n_objects, e.d = 0, 10, 4
    with pytest.raises(TypeError, match="cand_indptr"):
        e.topk_candidates_device(5, np.zeros(3, np.int64), np.zeros(4, np.int32), subjects=np.zeros((2, 4), np.float32))
    with pytest.raises(TypeError, match="cand_indptr"):
        e.topk_candidates_device(5, torch.zeros(3, dtype=torch.int64), torch.zeros(4, dtype=torch.int32))


def test_output_triplet_is_checked():
    torch = pytest.importorskip("torch")
    from rectools_b200.ranker import check_candidate_outputs

    dev = torch.device("cuda", 0)
    good = (np.zeros((4, 3), np.int32), np.zeros((4, 3), np.float32), np.zeros(4, np.int32))
    assert check_candidate_outputs(good, 4, 3, dev) is False
    with pytest.raises(ValueError, match="ids must have shape"):
        check_candidate_outputs((np.zeros((4, 2), np.int32),) + good[1:], 4, 3, dev)
    with pytest.raises(ValueError, match="counts must have shape"):
        check_candidate_outputs(good[:2] + (np.zeros(3, np.int32),), 4, 3, dev)
    with pytest.raises(TypeError, match="scores must be float32"):
        check_candidate_outputs((good[0], np.zeros((4, 3), np.float64), good[2]), 4, 3, dev)
    with pytest.raises(TypeError, match="ids must be int32"):
        check_candidate_outputs((np.zeros((4, 3), np.int64),) + good[1:], 4, 3, dev)
    with pytest.raises(ValueError, match="C-contiguous"):
        check_candidate_outputs((np.zeros((3, 4), np.int32).T,) + good[1:], 4, 3, dev)
    with pytest.raises(ValueError, match=r"\(ids, scores, counts\)"):
        check_candidate_outputs(good[:2], 4, 3, dev)
    # torch tensors: dtype and shape as for numpy, and they must be CUDA tensors on the engine's device
    t = (torch.zeros((4, 3), dtype=torch.int32), torch.zeros((4, 3)), torch.zeros(4, dtype=torch.int32))
    with pytest.raises(TypeError, match="CUDA tensors"):
        check_candidate_outputs(t, 4, 3, dev)
    with pytest.raises(TypeError, match="ids must be int32"):
        check_candidate_outputs((t[0].long(),) + t[1:], 4, 3, dev)
    with pytest.raises(ValueError, match="scores must have shape"):
        check_candidate_outputs((t[0], torch.zeros((4, 4)), t[2]), 4, 3, dev)
    with pytest.raises(TypeError, match="numpy array or a CUDA tensor"):
        check_candidate_outputs(([0] * 12,) + good[1:], 4, 3, dev)

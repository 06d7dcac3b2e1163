"""CPU: the plan of a ranking call (rectools_b200/csrc/plan.h) -- path, tensor-core mode, epilogue warps, K', append-list
size, row chunks and refusals -- pinned for an H100 engine (132 SMs: 66 CTA pairs, a wave of 16 896 subject rows).

tests/plan_driver.cpp is compiled with the system g++ and prints the plan of each case.  Every expected value below was
derived by hand from the decision code as it stood inline in b200_rank_topk before it moved into plan.h."""
import os
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

# B200_Q_* flags and B200_TC_* types of include/b200_rank.h
IN_DEV, FORCE_EXACT, FORCE_TC, SHARED = 1, 4, 8, 16
FP16, BF16 = 1, 2
PATH_EXACT, PATH_TC, PATH_SPARSE, PATH_DENSE_LARGE_K = 0, 1, 2, 3
NARROW, WIDE, WIDE_L, MULTI_PASS = 0, 1, 2, 3
E_UNSUPPORTED = -4

M = 1_000_000
WAVE = 66 * 256  # 16 896
ENGINE = {"sm_count": 132, "d": 128, "tc_dtype": FP16}


@pytest.fixture(scope="module")
def driver():
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    env = dict(os.environ)
    # the image exports CC/CXX pointing at a gcc without a usable spec set (as in rectools_b200/build.py)
    env.pop("CC", None)
    env.pop("CXX", None)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "plan_driver")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "plan_driver.cpp")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(cases):
            lines = [" ".join(f"{k}={v}" for k, v in {**ENGINE, **c}.items()) for c in cases]
            out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
            plans = []
            for ln in out.splitlines():
                head, message = ln.split(" message=")
                plan = {k: float(v) if k == "T" else int(v) for k, v in (w.split("=") for w in head.split())}
                plan["message"] = message
                plans.append(plan)
            assert len(plans) == len(cases)
            return plans

        yield run


def plan(driver, **case):
    return driver([case])[0]


def test_narrow_k_cand_ladder(driver):
    # K' = min(32, k + surplus), surplus max(2, k/4) in fp16 and max(6, k/2) in bf16.  Host inputs of 1M rows: chunks of
    # 8 waves = 135 168 rows (n_rows >= 2 chunks), ceil(1M / 135 168) = 8.
    p = plan(driver, n_rows=M, n_pos=M, k=10)
    assert (p["path"], p["mode"], p["nw"], p["k_cand"], p["chunk"], p["n_chunks"]) == (PATH_TC, NARROW, 8, 12, 8 * WAVE, 8)
    assert plan(driver, n_rows=M, n_pos=M, k=10, tc_dtype=BF16)["k_cand"] == 16  # 10 + max(6, 5)
    assert plan(driver, n_rows=M, n_pos=M, k=24)["k_cand"] == 30  # 24 + max(2, 6)
    assert plan(driver, n_rows=M, n_pos=M, k=24, tc_dtype=BF16)["k_cand"] == 32  # min(32, 24 + 12)
    # the config-5 shape (d = 256)
    assert plan(driver, n_rows=M, n_pos=M, k=20, d=256, tc_dtype=BF16)["k_cand"] == 30  # 20 + max(6, 10)
    assert plan(driver, n_rows=M, n_pos=M, k=20, d=256)["k_cand"] == 25  # 20 + max(2, 5)


def test_wide_mode(driver):
    # k = 100: K' = 24; T = int(1.35 * 100 + 40) = 175, lists of round_up(int(175 / 2 * 1.5 + 32), 8) = 168 slots
    p = plan(driver, n_rows=M, n_pos=M, k=100)
    assert (p["path"], p["mode"], p["nw"], p["k_cand"], p["T"], p["cand_stride"]) == (PATH_TC, WIDE, 8, 24, 175, 168)
    assert (p["chunk"], p["n_chunks"]) == (8 * WAVE, 8)


def test_multi_pass_without_wide_mode(driver):
    # B200_WIDE=0 at k = 100: passes of 20 with K' = 25 (fp16) / 30 (bf16); the route is not chunked
    for tc, kc in ((FP16, 25), (BF16, 30)):
        p = plan(driver, n_rows=M, n_pos=M, k=100, tc_dtype=tc, B200_WIDE=0)
        assert (p["path"], p["mode"], p["nw"], p["k_cand"], p["chunk"], p["n_chunks"]) == (PATH_TC, MULTI_PASS, 8, kc, M, 1)


def test_wide_large_k_chunks(driver):
    # k = 1000: T = int(1.6 * 1000 + 64) = 1664 <= n_pos / 2; lists of round_up(int(1664 / 2 * 1.5 + 32), 8) = 1280 slots.
    # 2 lists x 1280 x 8 B = 20 480 B per row; 2 GiB / 20 480 = 104 857 -> 104 704 (multiple of 256) -> 6 waves = 101 376.
    p = plan(driver, n_rows=M, n_pos=M, k=1000, flags=IN_DEV)
    assert (p["path"], p["mode"], p["nw"], p["k_cand"], p["T"], p["cand_stride"]) == (PATH_TC, WIDE_L, 8, 32, 1664, 1280)
    assert (p["chunk"], p["n_chunks"]) == (6 * WAVE, 10)
    # k = 500: T = 864, 432 * 1.5 + 32 = 680 slots; 10 880 B per row: 197 378 -> 197 376 -> 11 waves = 185 856 rows.
    # Device inputs: ceil(1M / 185 856) = 6 chunks; host inputs keep the smaller copy chunk of 135 168 rows: 8 chunks.
    p = plan(driver, n_rows=M, n_pos=M, k=500, flags=IN_DEV)
    assert (p["mode"], p["cand_stride"], p["chunk"], p["n_chunks"]) == (WIDE_L, 680, 11 * WAVE, 6)
    p = plan(driver, n_rows=M, n_pos=M, k=500)
    assert (p["mode"], p["cand_stride"], p["chunk"], p["n_chunks"]) == (WIDE_L, 680, 8 * WAVE, 8)
    # a lowered budget: 8 MiB / 20 480 B = 409 -> 256 rows (below a wave: not rounded to waves)
    p = plan(driver, n_rows=4096, n_pos=M, k=1000, flags=IN_DEV, B200_WIDE_BUDGET_MB=8)
    assert (p["chunk"], p["n_chunks"]) == (256, 16)


def test_path_3(driver):
    # 3 000 whitelisted objects: T = 1664 > 1500, K' = 0, path 3;  k > 1024 and B200_WIDE=0 likewise
    assert plan(driver, n_rows=M, n_pos=3000, k=1000)["path"] == PATH_DENSE_LARGE_K
    assert plan(driver, n_rows=M, n_pos=M, k=1025)["path"] == PATH_DENSE_LARGE_K
    assert plan(driver, n_rows=M, n_pos=M, k=300, B200_WIDE=0)["path"] == PATH_DENSE_LARGE_K
    # k is clipped to the positions: k = 5000 over 3 000 objects is k = 3000
    p = plan(driver, n_rows=M, n_pos=3000, k=5000)
    assert (p["k_out"], p["path"]) == (3000, PATH_DENSE_LARGE_K)


def test_tiny_problem_and_force_flags(driver):
    # 10 x 1 000 = 1e4 < 4e6: the exhaustive kernel, unless FORCE_TC
    p = plan(driver, n_rows=10, n_pos=1000, k=10)
    assert (p["path"], p["n_chunks"]) == (PATH_EXACT, 1)
    p = plan(driver, n_rows=10, n_pos=1000, k=10, flags=FORCE_TC)
    assert (p["path"], p["mode"], p["k_cand"], p["chunk"], p["n_chunks"]) == (PATH_TC, NARROW, 12, 10, 1)
    assert plan(driver, n_rows=M, n_pos=M, k=10, flags=FORCE_EXACT)["path"] == PATH_EXACT
    # an engine without the tensor-core copy
    assert plan(driver, n_rows=M, n_pos=M, k=10, tc_dtype=3)["path"] == PATH_EXACT
    # n_pos < 4 K': 12 x 4 = 48 objects needed
    assert plan(driver, n_rows=M, n_pos=47, k=10)["path"] == PATH_EXACT


def test_shared_thresholds_k_cand(driver):
    # 7 peers, 2 lists: L = 16, c_L = 1.77, target = 10 + max(12, 6) = 22; 16 K' - 28.32 sqrt(K') >= 22 first at K' = 6
    p = plan(driver, n_rows=M, n_pos=M, k=10, n_peers=7, flags=SHARED)
    assert (p["path"], p["k_cand"], p["peers"]) == (PATH_TC, 6, 1)
    # no peers: the protocol runs, the K' ladder is the plain one
    p = plan(driver, n_rows=M, n_pos=M, k=10, flags=SHARED)
    assert (p["k_cand"], p["peers"]) == (12, 1)


def test_hooks(driver):
    # B200_TC_KCAND below k is taken only where lists may be shorter than k
    assert plan(driver, n_rows=M, n_pos=M, k=10, B200_TC_KCAND=20)["k_cand"] == 20
    assert plan(driver, n_rows=M, n_pos=M, k=10, B200_TC_KCAND=8)["k_cand"] == 12
    assert plan(driver, n_rows=M, n_pos=M, k=100, B200_TC_KCAND=8)["k_cand"] == 8
    # a list holds 32 slots: the largest forced K' is taken whole
    assert plan(driver, n_rows=M, n_pos=M, k=10, B200_TC_KCAND=32)["k_cand"] == 32
    # B200_WIDE_T: T = 61 at k = 100 -> round_up(int(30.5 * 1.5 + 32), 8) = 80 slots; T = 400 -> 332, capped at
    # WIDE_MAX / 2 = 256.  B200_CHUNK_ROWS (at least 256)
    p = plan(driver, n_rows=M, n_pos=M, k=100, B200_WIDE_T=61)
    assert (p["T"], p["cand_stride"]) == (61, 80)
    p = plan(driver, n_rows=M, n_pos=M, k=100, B200_WIDE_T=400)
    assert (p["T"], p["cand_stride"]) == (400, 256)
    p = plan(driver, n_rows=10_000, n_pos=M, k=10, B200_CHUNK_ROWS=2048)
    assert (p["chunk"], p["n_chunks"]) == (2048, 5)
    p = plan(driver, n_rows=10_000, n_pos=M, k=10, B200_CHUNK_ROWS=1)
    assert (p["chunk"], p["n_chunks"]) == (256, 40)
    # hooks last one call: the next case sees none
    assert driver([{"n_rows": M, "n_pos": M, "k": 100, "B200_WIDE": 0}, {"n_rows": M, "n_pos": M, "k": 100}])[1]["mode"] == WIDE


def test_sparse_subjects(driver):
    p = plan(driver, n_rows=M, n_pos=M, k=10, sparse=1)
    assert (p["path"], p["n_chunks"], p["error"]) == (PATH_SPARSE, 1, 0)


def test_refusals(driver):
    p = plan(driver, n_rows=M, n_pos=M, k=1025, flags=FORCE_TC)
    assert p["error"] == E_UNSUPPORTED
    assert p["message"] == "b200_rank_topk: tensor-core path unavailable (tc_dtype=1, k=1025, d_pad=128, n_pos=1000000)"
    p = plan(driver, n_rows=M, n_pos=M, k=10, sparse=1, flags=FORCE_TC)
    assert p["error"] == E_UNSUPPORTED and "tensor-core path unavailable" in p["message"]
    p = plan(driver, n_rows=M, n_pos=M, k=100, flags=SHARED)
    assert (p["error"], p["message"]) == (E_UNSUPPORTED, "b200_rank_topk: B200_Q_SHARED_THRESHOLDS needs k <= 24")
    # 8 re-score warps x d floats must fit 64 KiB (d <= 2048)
    p = plan(driver, n_rows=M, n_pos=M, k=10, d=2056)
    assert (p["error"], p["message"]) == (E_UNSUPPORTED, "b200_rank_topk: d too large for the re-score kernel")
    assert plan(driver, n_rows=M, n_pos=M, k=10, d=2048)["error"] == 0
    # nothing to rank: no refusal
    assert plan(driver, n_rows=0, n_pos=M, k=1025, flags=FORCE_TC)["error"] == 0

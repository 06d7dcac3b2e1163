"""CPU: the large-k selection's decisions and order key, compiled with g++ alone.

tests/large_k_driver.cpp prints, per call, the selection mode of the plan (rectools_b200/csrc/plan.h: PASSES = 0, the
ceil(k/32) streaming passes; RADIX = 1, large_k_select_kernel) and the bytes per row its path-2 / path-3 row chunks budget,
and the order key (rectools_b200/csrc/order_key.h) of fp32 bit patterns.  The engine here is an H100 (132 SMs), d = 128."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

FORCE_EXACT, FORCE_TC = 4, 8
FP16 = 1
PATH_EXACT, PATH_TC, PATH_SPARSE, PATH_DENSE_LARGE_K = 0, 1, 2, 3
WIDE_L = 2
PASSES, RADIX = 0, 1
LK_SMEM_PAIRS = 12288  # rectools_b200/csrc/sizes.h
M = 1_000_000
ENGINE = {"sm_count": 132, "d": 128, "tc_dtype": FP16}


@pytest.fixture(scope="module")
def driver():
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    env = dict(os.environ)
    env.pop("CC", None)  # (as in rectools_b200/build.py: the image's CC/CXX may point at an unusable gcc)
    env.pop("CXX", None)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "large_k_driver")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "large_k_driver.cpp")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(lines):
            out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
            out = out.splitlines()
            assert len(out) == len(lines)
            return out

        yield run


def plans(driver, *cases):
    lines = [" ".join(f"{k}={v}" for k, v in {**ENGINE, **c}.items()) for c in cases]
    return [{k: int(v) for k, v in (w.split("=") for w in ln.split())} for ln in driver(lines)]


def plan(driver, **case):
    return plans(driver, case)[0]


def keys(driver, bits):
    (line,) = driver(["key " + " ".join(f"{int(b):x}" for b in bits)])
    return np.array([int(w, 16) for w in line.split()], np.uint64)


# ------------------------------------------------------------------------------------------------ the plan
def test_radix_from_k_1025_on_paths_2_and_3(driver):
    # dense, 1M objects: k = 1024 is the tensor-core wide mode (its passes untouched), k = 1025 path 3 with the radix select
    p = plan(driver, n_rows=M, n_pos=M, k=1024)
    assert (p["path"], p["mode"], p["select"]) == (PATH_TC, WIDE_L, PASSES)
    p = plan(driver, n_rows=M, n_pos=M, k=1025)
    assert (p["path"], p["select"]) == (PATH_DENSE_LARGE_K, RADIX)
    # FORCE_EXACT keeps path 3 at 129 <= k <= 1024 on the passes, path 0 below
    for k, path, sel in ((100, PATH_EXACT, PASSES), (129, PATH_DENSE_LARGE_K, PASSES), (1024, PATH_DENSE_LARGE_K, PASSES),
                         (1025, PATH_DENSE_LARGE_K, RADIX)):
        p = plan(driver, n_rows=M, n_pos=M, k=k, flags=FORCE_EXACT)
        assert (p["path"], p["select"]) == (path, sel), k
    # sparse subjects (EASE): the same boundary
    for k, sel in ((1, PASSES), (1024, PASSES), (1025, RADIX), (20_000, RADIX)):
        p = plan(driver, n_rows=M, n_pos=20_000, k=k, sparse=1)
        assert (p["path"], p["select"]) == (PATH_SPARSE, sel), k


def test_k_none_and_whitelists_shorter_than_k(driver):
    # k = None is k = n_pos (rank_implicit.py:233-234): the whole catalogue, path 3, radix
    p = plan(driver, n_rows=8192, n_pos=M, k=M)
    assert (p["k_out"], p["path"], p["select"]) == (M, PATH_DENSE_LARGE_K, RADIX)
    # k is clipped to the positions before the decision: 1 000 whitelisted positions at k = 5 000 keep the passes
    p = plan(driver, n_rows=M, n_pos=1_000, k=5_000)
    assert (p["k_out"], p["path"], p["select"]) == (1_000, PATH_DENSE_LARGE_K, PASSES)
    p = plan(driver, n_rows=M, n_pos=1_025, k=5_000)
    assert (p["k_out"], p["path"], p["select"]) == (1_025, PATH_DENSE_LARGE_K, RADIX)
    p = plan(driver, n_rows=M, n_pos=1_024, k=5_000, sparse=1)
    assert (p["k_out"], p["path"], p["select"]) == (1_024, PATH_SPARSE, PASSES)


def test_select_hook(driver):
    # B200_SELECT=0: the passes for every k;  =2: the radix select for every k on paths 2 and 3, nowhere else
    for k in (1025, 4096, M):
        assert plan(driver, n_rows=M, n_pos=M, k=k, B200_SELECT=0)["select"] == PASSES
        assert plan(driver, n_rows=M, n_pos=M, k=k, sparse=1, B200_SELECT=0)["select"] == PASSES
    for k in (1, 33, 129, 1000):
        assert plan(driver, n_rows=M, n_pos=M, k=k, sparse=1, B200_SELECT=2)["select"] == RADIX
    p = plan(driver, n_rows=M, n_pos=M, k=200, flags=FORCE_EXACT, B200_SELECT=2)
    assert (p["path"], p["select"]) == (PATH_DENSE_LARGE_K, RADIX)
    p = plan(driver, n_rows=M, n_pos=M, k=100, flags=FORCE_EXACT, B200_SELECT=2)
    assert (p["path"], p["select"]) == (PATH_EXACT, PASSES)
    # the wide mode (whose rejected rows re-rank on the path-3 kernels with the passes) and the narrow mode stay as they are
    for k in (10, 100, 1000):
        p = plan(driver, n_rows=M, n_pos=M, k=k, B200_SELECT=2)
        assert (p["path"], p["select"]) == (PATH_TC, PASSES), k
    # hooks last one call
    a, b = plans(driver, dict(n_rows=M, n_pos=M, k=2000, B200_SELECT=0), dict(n_rows=M, n_pos=M, k=2000))
    assert (a["select"], b["select"]) == (PASSES, RADIX)


def test_refusals_unchanged(driver):
    assert plan(driver, n_rows=M, n_pos=M, k=1025, flags=FORCE_TC)["error"] == -4
    assert plan(driver, n_rows=0, n_pos=M, k=1025)["select"] == PASSES  # nothing to rank


def test_row_chunk_budget(driver):
    # the passes and the in-shared-memory sort budget the score row only (4 B per position, as before); above
    # LK_SMEM_PAIRS survivors the sort's global scratch adds 16 B per entry
    assert plan(driver, n_rows=M, n_pos=M, k=1000, flags=FORCE_EXACT)["row_bytes"] == 4 * M
    assert plan(driver, n_rows=M, n_pos=M, k=LK_SMEM_PAIRS)["row_bytes"] == 4 * M
    assert plan(driver, n_rows=M, n_pos=M, k=LK_SMEM_PAIRS + 1)["row_bytes"] == 4 * M + 16 * (LK_SMEM_PAIRS + 1)
    assert plan(driver, n_rows=M, n_pos=M, k=LK_SMEM_PAIRS + 1, B200_SELECT=0)["row_bytes"] == 4 * M
    # k = None over 1M objects: 20 MB a row, 53 rows (32 on path 3) in 1 GiB;  an EASE catalogue of 20 000 items: 2 684 rows
    p = plan(driver, n_rows=8192, n_pos=M, k=M)
    assert p["row_bytes"] == 20 * M and (1 << 30) // p["row_bytes"] == 53
    p = plan(driver, n_rows=8192, n_pos=20_000, k=20_000, sparse=1)
    assert p["row_bytes"] == 400_000 and (1 << 30) // p["row_bytes"] == 2_684


# ------------------------------------------------------------------------------------------------ the order key
def _f32_bits(values):
    return np.asarray(values, np.float32).view(np.uint32)


def test_order_key_special_values(driver):
    tiny = np.float32(np.finfo(np.float32).tiny)
    fmax = np.float32(np.finfo(np.float32).max)
    bits = np.r_[_f32_bits([0.0, -0.0, 1e-45, -1e-45, tiny, -tiny, fmax, -fmax, np.inf, -np.inf, 1.0, -1.0]),
                 np.array([0x7FC00000, 0x7F800001, 0x7FFFFFFF, 0xFFC00000, 0xFF800001, 0xFFFFFFFF], np.uint32)]
    k = keys(driver, bits)
    assert k[0] == k[1] == 0x80000000  # +-0 tie
    assert k[2] == 0x80000001 and k[3] == 0x7FFFFFFE  # the smallest subnormals either side of zero
    assert k[3] < k[0] < k[2] < k[4] and k[5] < k[3]
    assert k[6] == 0xFF7FFFFF and k[7] == 0x00800000  # +-FLT_MAX: -FLT_MAX is a real, kept score
    assert k[8] == 0xFF800000  # +inf: the largest key
    assert k[9] == 0  # -inf: never selected
    assert k[10] > k[0] > k[11]
    assert (k[12:] == 0).all()  # NaN of either sign and any payload: never selected


def test_order_key_is_monotone(driver):
    rng = np.random.default_rng(5)
    bits = np.r_[rng.integers(0, 1 << 32, 20_000, dtype=np.uint64).astype(np.uint32),
                 _f32_bits(rng.integers(-3, 4, 2_000)),  # many exact ties
                 _f32_bits(rng.standard_normal(2_000) * 1e-40)]  # subnormals
    k = keys(driver, bits).astype(np.int64)
    f = bits.view(np.float32)
    valid = f > -np.inf  # (False for NaN)
    assert (k[~valid] == 0).all() and (k[valid] >= 0x00800000).all() and (k[valid] <= 0xFF800000).all()
    fv, kv = f[valid].astype(np.float64), k[valid]
    i, j = rng.integers(0, len(fv), (2, 200_000))
    np.testing.assert_array_equal(np.sign(kv[i] - kv[j]), np.sign(fv[i] - fv[j]))

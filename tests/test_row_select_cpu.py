"""CPU: stored rows as score rows (path 4, `b200_rank_query.object_rows`) up to the point where a GPU is needed.

tests/rows_plan_driver.cpp prints the plan (rectools_b200/csrc/plan.h) of a call: path 4 for every k once `object_rows`
is given, its refusals, and its row chunks.  The engine here is an H100 (132 SMs) holding a square EASE-shaped matrix.
The RecTools wiring is checked against the reference package: `install()` rebinds `EASEModel._recommend_i2i` and
`uninstall()` restores it, and weights the engine does not rank (not a C-contiguous fp32 matrix) go to the original."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import stage_reference

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))

INVALID, UNSUPPORTED = -1, -4
FORCE_EXACT, FORCE_TC, SHARED_THRESHOLDS, INPUTS_ON_DEVICE = 4, 8, 16, 1
PATH_SPARSE, PATH_ROWS = 2, 4
PASSES, RADIX = 0, 1
S = 12288  # LK_SMEM_PAIRS, rectools_b200/csrc/sizes.h
N = 20_000
ENGINE = {"sm_count": 132, "d": N, "n_objects": N, "tc_dtype": 1}
WAVES8 = 8 * 66 * 256  # 8 waves of CTA pairs on 132 SMs


@pytest.fixture(scope="module")
def driver():
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    env = dict(os.environ)
    env.pop("CC", None)  # (as in rectools_b200/build.py: the image's CC/CXX may point at an unusable gcc)
    env.pop("CXX", None)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "rows_plan_driver")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "rows_plan_driver.cpp")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(cases):
            lines = [" ".join(f"{k}={v}" for k, v in {**ENGINE, "rows": 1, **c}.items()) for c in cases]
            out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
            plans = []
            for ln in out.splitlines():
                head, _, message = ln.partition(" message=")
                p = {k: int(v) for k, v in (w.split("=") for w in head.split())}
                p["message"] = message
                plans.append(p)
            assert len(plans) == len(cases)
            return plans

        yield run


def plan(driver, **case):
    return driver([case])[0]


# ------------------------------------------------------------------------------------------------ the plan
@pytest.mark.parametrize("k", [1, 10, 1024, 1025, S - 1, S, S + 1, None])
def test_stored_rows_take_path_4_for_every_k(driver, k):
    p = plan(driver, n_rows=N, n_pos=N, k=N if k is None else k)  # k = None is k = n_pos
    assert (p["path"], p["select"], p["error"]) == (PATH_ROWS, RADIX, 0)
    assert p["k_out"] == (N if k is None else k)


def test_whitelists_and_flags_keep_path_4(driver):
    # k is clipped to the whitelisted positions; FORCE_EXACT asks for nothing path 4 does not already do
    p = plan(driver, n_rows=N, n_pos=500, k=1000)
    assert (p["k_out"], p["path"]) == (500, PATH_ROWS)
    assert plan(driver, n_rows=N, n_pos=N, k=10, flags=FORCE_EXACT)["path"] == PATH_ROWS
    assert plan(driver, n_rows=N, n_pos=N, k=10, flags=INPUTS_ON_DEVICE)["path"] == PATH_ROWS
    # the selection hook of paths 2 / 3 does not apply: path 4 has one selection
    assert plan(driver, n_rows=N, n_pos=N, k=10, B200_SELECT=0)["select"] == RADIX
    # without object_rows the same shape is the sparse path as before
    assert plan(driver, n_rows=N, n_pos=N, k=10, rows=0, sparse=1)["path"] == PATH_SPARSE


def test_refusals(driver):
    p = plan(driver, n_rows=10, n_pos=N, k=10, d=64)
    assert p["error"] == INVALID and "d == n_objects" in p["message"]
    assert plan(driver, n_rows=10, n_pos=N, k=10, cosine=1)["error"] == UNSUPPORTED
    assert plan(driver, n_rows=10, n_pos=N, k=10, id_offset=1)["error"] == UNSUPPORTED
    assert plan(driver, n_rows=10, n_pos=N, k=10, flags=SHARED_THRESHOLDS)["error"] == UNSUPPORTED
    p = plan(driver, n_rows=10, n_pos=N, k=10, flags=FORCE_TC)
    assert p["error"] == UNSUPPORTED and "FORCE_TC" in p["message"]
    # nothing to rank: no plan, no refusal (as for every path)
    p = plan(driver, n_rows=0, n_pos=N, k=10, d=64)
    assert (p["error"], p["n_chunks"]) == (0, 0)


def test_row_chunks(driver):
    # no score buffer: up to LK_SMEM_PAIRS the chunk holds nothing per row, above it the sort scratch (16 B per entry)
    assert plan(driver, n_rows=N, n_pos=N, k=S)["row_bytes"] == 0
    assert plan(driver, n_rows=N, n_pos=N, k=S + 1)["row_bytes"] == 16 * (S + 1)
    # one chunk below two times 8 waves of CTA pairs, chunks of 8 waves above
    p = plan(driver, n_rows=2 * WAVES8 - 1, n_pos=N, k=10)
    assert (p["chunk"], p["n_chunks"]) == (2 * WAVES8 - 1, 1)
    p = plan(driver, n_rows=2 * WAVES8, n_pos=N, k=10)
    assert (p["chunk"], p["n_chunks"]) == (WAVES8, 2)
    # sort scratch within 1 GiB: 5 460 rows of k = S + 1 (196 624 B each); k = None over 50 000 items: 1 342 rows
    p = plan(driver, n_rows=N, n_pos=N, k=S + 1)
    assert (p["chunk"], p["n_chunks"]) == ((1 << 30) // (16 * (S + 1)), 4)
    p = plan(driver, n_rows=50_000, n_pos=50_000, k=50_000, d=50_000, n_objects=50_000)
    assert (p["chunk"], p["n_chunks"]) == (1342, 38)
    # B200_CHUNK_ROWS (at least 256) sets the chunk for host and device inputs alike
    for flags in (0, INPUTS_ON_DEVICE):
        p = plan(driver, n_rows=600, n_pos=N, k=10, flags=flags, B200_CHUNK_ROWS=256)
        assert (p["chunk"], p["n_chunks"]) == (256, 3)
    assert plan(driver, n_rows=600, n_pos=N, k=10, B200_CHUNK_ROWS=1)["n_chunks"] == 3


def test_query_layout_keeps_its_size():
    """object_rows takes the first reserved slot: the struct keeps its size, the fields before it their offsets."""
    from rectools_b200 import _lib

    q = _lib.Query
    assert ctypes.sizeof(q) == 160
    assert q.object_rows.offset == 144 and q.reserved.offset == 152
    assert _lib.ABI_VERSION == 6


# ------------------------------------------------------------------------------------------------ RecTools wiring
@pytest.fixture()
def ease():
    if not stage_reference.available():
        pytest.skip("reference package neither staged nor checked out")
    added = stage_reference.add_to_path()
    import rectools.models.ease as ease_mod

    yield ease_mod
    import rectools_b200

    rectools_b200.uninstall()
    stage_reference.remove_from_path(added)


def test_install_rebinds_ease_i2i(ease):
    import rectools_b200
    from rectools_b200.integration import ease_recommend_i2i

    orig = ease.EASEModel._recommend_i2i  # pylint: disable=protected-access
    rectools_b200.install(device=0)
    assert ease.EASEModel._recommend_i2i is ease_recommend_i2i  # pylint: disable=protected-access
    rectools_b200.install(device=0)  # a second install keeps the original to restore
    rectools_b200.uninstall()
    assert ease.EASEModel._recommend_i2i is orig  # pylint: disable=protected-access
    rectools_b200.install(device=0, fast_recommend=False)
    assert ease.EASEModel._recommend_i2i is ease_recommend_i2i  # pylint: disable=protected-access
    rectools_b200.uninstall()
    assert ease.EASEModel._recommend_i2i is orig  # pylint: disable=protected-access


def _weight(n, dtype, seed=0):
    w = np.random.default_rng(seed).standard_normal((n, n)).astype(dtype)
    np.fill_diagonal(w, 0.0)
    return w


@pytest.mark.parametrize("layout", ["float64", "fortran", "strided"])
def test_weights_the_engine_does_not_rank_go_to_the_original(ease, layout):
    import rectools_b200

    w = {"float64": _weight(40, np.float64), "fortran": np.asfortranarray(_weight(40, np.float32)),
         "strided": _weight(80, np.float32)[::2, ::2]}[layout]
    model = ease.EASEModel()
    model.weight = w
    targets = np.array([3, 0, 39, 3])
    wl = np.arange(0, 40, 3)
    orig = ease.EASEModel._recommend_i2i  # pylint: disable=protected-access
    expected = [orig(model, targets, None, 5, None), orig(model, targets, None, 5, wl)]
    rectools_b200.install(device=0)
    got = [model._recommend_i2i(targets, None, 5, None), model._recommend_i2i(targets, None, 5, wl)]  # pylint: disable=protected-access
    for e, g in zip(expected, got):
        for a, b in zip(e, g):
            np.testing.assert_array_equal(a, b)
        assert g[2].dtype == w.dtype  # ranked in the weight's own precision


def test_fp32_weights_go_to_the_engine(ease, monkeypatch):
    """A C-contiguous fp32 weight is ranked by the engine that `_recommend_u2i` uses: the one cached for that matrix."""
    import rectools_b200
    from rectools_b200 import integration

    class Asked(Exception):
        pass

    def fake_cached_engine(objects, cosine, device, tc_mode):
        raise Asked(objects, cosine, device, tc_mode)

    monkeypatch.setattr(integration, "cached_engine", fake_cached_engine)
    model = ease.EASEModel()
    model.weight = _weight(40, np.float32)
    rectools_b200.install(device=0, tc_mode="auto")
    with pytest.raises(Asked) as info:
        model._recommend_i2i(np.array([1, 2]), None, 5, None)  # pylint: disable=protected-access
    objects, cosine, device, tc_mode = info.value.args
    assert objects is model.weight and (cosine, device, tc_mode) == (False, 0, "auto")

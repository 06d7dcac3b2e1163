"""CPU: engine groups (b200_rank_group_*) without a GPU -- the row split of rectools_b200/csrc/group_plan.h compiled with
g++, the exported and declared symbols, the `device` argument of `B200Ranker` / `install()` / `make_similarity_module()`,
the engine cache keys, and the refusal to create a group without a device."""
import ctypes as C
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


@pytest.fixture(scope="module")
def driver():
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    env = dict(os.environ)
    env.pop("CC", None)  # (as in rectools_b200/build.py)
    env.pop("CXX", None)
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "group_plan_driver")
        res = subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "group_plan_driver.cpp")],
                             env=env, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr

        def run(lines, extra_env=None):
            e = dict(os.environ)
            e.pop("B200_GROUP_SLICE_ROWS", None)
            e.update(extra_env or {})
            out = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True, env=e).stdout
            return [list(map(int, ln.split())) for ln in out.splitlines()]

        yield run


def split(driver, n_rows, members, forced=0):
    rows, n_slices, *edges = driver([f"split {n_rows} {members} {forced}"])[0]
    return rows, [(edges[2 * i], edges[2 * i + 1]) for i in range(n_slices)]


@pytest.mark.parametrize("members", [1, 2, 3, 8])
@pytest.mark.parametrize("n_rows", [0, 1, 2, 37, 1_000_000])
@pytest.mark.parametrize("forced", [0, 1, 5, 1000])
def test_every_row_in_exactly_one_slice(driver, n_rows, members, forced):
    if forced and n_rows // max(forced, 1) > 100_000:
        pytest.skip("too many slices to print")
    rows, slices = split(driver, n_rows, members, forced)
    if n_rows == 0:
        assert slices == []
        return
    assert slices[0][0] == 0 and slices[-1][1] == n_rows
    for (a0, a1), (b0, _) in zip(slices, slices[1:]):
        assert a1 == b0  # contiguous and ordered
    assert all(r1 - r0 == rows for r0, r1 in slices[:-1]) and 0 < slices[-1][1] - slices[-1][0] <= rows
    if forced:
        assert rows == forced


def test_default_slice_size(driver):
    # one member: the whole batch in one call
    assert split(driver, 1_000_000, 1)[0] == 1_000_000
    # several: 4 slices per member, at least 32 768 rows (or the whole batch)
    assert split(driver, 1_000_000, 2)[0] == 125_000
    assert split(driver, 1_000_000, 8)[0] == 32_768  # ceil(1M / 32) = 31 250 < 32 768
    assert split(driver, 10_000_000, 8)[0] == 312_500
    assert split(driver, 37, 3) == (37, [(0, 37)])  # fewer rows than one slice: one member ranks them
    assert split(driver, 2, 3) == (2, [(0, 2)])


def test_forced_slice_hook(driver):
    assert driver(["hook"]) == [[0]]
    assert driver(["hook"], {"B200_GROUP_SLICE_ROWS": "7"}) == [[7]]
    assert driver(["hook"], {"B200_GROUP_SLICE_ROWS": "-3"}) == [[0]]
    # a group of one member takes forced slices too
    assert split(driver, 37, 1, 5)[1] == [(i, min(i + 5, 37)) for i in range(0, 37, 5)]


def test_csr_slice_rebasing(driver):
    rng = np.random.default_rng(5)
    lens = rng.integers(0, 6, 37)
    lens[3:7] = 0  # empty rows
    for base in (0, 11):  # an indptr that does not start at 0
        indptr = np.r_[0, np.cumsum(lens)] + base
        for forced in (1, 5, 1000):
            _, slices = split(driver, 37, 3, forced)
            for r0, r1 in slices:
                line = f"rebase {r0} {r1} " + " ".join(map(str, indptr))
                got_base, *got = driver([line])[0]
                assert got_base == indptr[r0]
                np.testing.assert_array_equal(got, indptr[r0 : r1 + 1] - indptr[r0])
                assert got[0] == 0 and got[-1] == lens[r0:r1].sum()


def test_group_symbols_declared_and_exported():
    from rectools_b200 import _lib, build

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    group = {n for n in re.findall(r"\b(b200_rank_group_[a-z_]+)\s*\(", header)}
    assert group == {"b200_rank_group_create", "b200_rank_group_create_ex", "b200_rank_group_destroy", "b200_rank_group_get_info",
                     "b200_rank_group_set_subjects", "b200_rank_group_topk"}
    assert group <= set(_lib.EXPORTS)
    build.build()
    lib = _lib.load()
    for name in group:
        assert getattr(lib, name) is not None
    assert "#define B200_RANK_ABI_VERSION 6" in header


def test_group_create_without_gpu_fails_like_engine_create():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from rectools_b200 import B200Ranker, EngineGroup, _lib, build

    build.build()
    lib = _lib.load()
    objects = np.ones((4, 3), np.float32)
    h = C.c_void_p()
    devs = (C.c_int32 * 2)(0, 0)
    assert lib.b200_rank_group_create(C.byref(h), objects.ctypes.data, 4, 3, _lib.DIST_DOT, devs, 2, _lib.TC_AUTO, 0) == _lib.E_CUDA
    assert b"no CUDA device" in lib.b200_rank_last_error()
    assert not h.value
    assert lib.b200_rank_group_create(C.byref(h), objects.ctypes.data, 4, 3, _lib.DIST_DOT, devs, 0, _lib.TC_AUTO, 0) == _lib.E_INVALID
    assert lib.b200_rank_group_topk(None, None, None, None) == _lib.E_INVALID
    with pytest.raises(_lib.B200RankError):
        EngineGroup(objects, cosine=False, devices=[0, 0])
    with pytest.raises(_lib.B200RankError):
        B200Ranker("dot", np.ones((2, 3), np.float32), objects, device=[0, 0])


def test_parse_devices(monkeypatch):
    import torch

    from rectools_b200.ranker import parse_devices

    assert parse_devices(0) == 0 and parse_devices(np.int64(3)) == 3
    assert parse_devices([0]) == (0,) and parse_devices((0, 0, 0)) == (0, 0, 0) and parse_devices(range(2)) == (0, 1)
    assert parse_devices(np.array([1, 0])) == (1, 0)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 4)
    assert parse_devices("all") == (0, 1, 2, 3)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 0)
    from rectools_b200 import _lib

    with pytest.raises(_lib.B200RankError):
        parse_devices("all")
    for bad, exc in (([], ValueError), (-1, ValueError), ([0, -2], ValueError), ("cuda", ValueError), (True, TypeError),
                     ([0, True], TypeError), ([0.0], TypeError), (None, TypeError), (1.5, TypeError)):
        with pytest.raises(exc):
            parse_devices(bad)


class _FakeEngine:
    def __init__(self, device):
        self.device = device


def test_cached_engine_keys_on_the_device_tuple(monkeypatch):
    from rectools_b200 import integration

    made = []

    def fake(objects, cosine, device, tc_mode="auto", **kw):
        made.append(device)
        return _FakeEngine(device)

    monkeypatch.setattr(integration, "new_engine", fake)
    monkeypatch.setattr(integration, "_ENGINE_CACHE_MAX", 8)
    integration.clear_engine_cache()
    try:
        w = np.arange(12, dtype=np.float32).reshape(4, 3)
        a = integration.cached_engine(w, False, 0, "auto")
        b = integration.cached_engine(w, False, (0,), "auto")
        c = integration.cached_engine(w, False, (0, 0), "auto")
        assert integration.cached_engine(w, False, 0, "auto") is a
        assert integration.cached_engine(w, False, (0,), "auto") is b
        assert integration.cached_engine(w, False, (0, 0), "auto") is c
        assert len({id(a), id(b), id(c)}) == 3 and made == [0, (0,), (0, 0)]
    finally:
        integration.clear_engine_cache()


def test_b200_ranker_builds_a_group_for_a_device_sequence(monkeypatch):
    from rectools_b200 import ranker

    built = []

    class Fake:
        def __init__(self, objects, cosine, devices, tc_mode="auto", **kw):
            built.append(("group", tuple(devices)))
            self.n_objects, self.d = objects.shape

        def set_subjects(self, subjects, key=None, owner=None):
            pass

    class FakeEngine(Fake):
        def __init__(self, objects, cosine, device, tc_mode="auto", **kw):  # pylint: disable=super-init-not-called
            built.append(("engine", device))

    monkeypatch.setattr(ranker, "EngineGroup", Fake)
    monkeypatch.setattr(ranker, "Engine", FakeEngine)
    u, i = np.ones((2, 3), np.float32), np.ones((4, 3), np.float32)
    ranker.B200Ranker("dot", u, i, device=1)
    ranker.B200Ranker("dot", u, i, device=[0, 1])
    ranker.B200Ranker("dot", u, i, device=(2,))
    assert built == [("engine", 1), ("group", (0, 1)), ("group", (2,))]
    with pytest.raises(ValueError):
        ranker.B200Ranker("dot", u, i, device=[])


def test_install_parses_the_device_and_uninstall_restores(monkeypatch):
    from oracle import stage_reference

    if not stage_reference.available():
        pytest.skip("reference package neither staged nor checked out")
    import torch

    added = stage_reference.add_to_path()
    try:
        import rectools.models.ease as ease
        import rectools.models.vector as vector
        import rectools_b200
        from rectools_b200.integration import B200ImplicitRanker

        before = (vector.ImplicitRanker, ease.ImplicitRanker, ease.EASEModel._recommend_i2i,  # pylint: disable=protected-access
                  vector.VectorModel.__dict__.get("recommend"), vector.VectorModel.__dict__.get("recommend_to_items"))
        monkeypatch.setattr(torch.cuda, "device_count", lambda: 3)
        for device, parsed in ((0, 0), (2, 2), ([0, 1], (0, 1)), ((0, 0, 0), (0, 0, 0)), ("all", (0, 1, 2))):
            rectools_b200.install(device=device)
            try:
                assert B200ImplicitRanker.default_device == parsed
                assert vector.ImplicitRanker is B200ImplicitRanker and ease.ImplicitRanker is B200ImplicitRanker
            finally:
                rectools_b200.uninstall()
            after = (vector.ImplicitRanker, ease.ImplicitRanker, ease.EASEModel._recommend_i2i,  # pylint: disable=protected-access
                     vector.VectorModel.__dict__.get("recommend"), vector.VectorModel.__dict__.get("recommend_to_items"))
            assert after == before
        for bad in ([], "gpu", -1):
            with pytest.raises((ValueError, TypeError)):
                rectools_b200.install(device=bad)
            rectools_b200.uninstall()
    finally:
        stage_reference.remove_from_path(added)
    B200ImplicitRanker.default_device = 0


def test_similarity_module_passes_devices_to_the_factory():
    from oracle import stage_reference

    if not stage_reference.available():
        pytest.skip("reference package neither staged nor checked out")
    added = stage_reference.add_to_path()
    try:
        from rectools_b200.integration import make_similarity_module

        seen = []

        def factory(**kw):
            seen.append(kw.get("devices", "absent"))
            raise StopIteration

        for devices, exp in ((None, "absent"), ([0, 0], (0, 0))):
            module = make_similarity_module(factory, devices=devices)
            inst = module.__new__(module)
            inst.distance = "dot"
            import torch

            with pytest.raises(StopIteration):
                inst._recommend_u2i(torch.zeros(2, 3), torch.zeros(4, 3), np.arange(2), 2, None, None)  # pylint: disable=protected-access
        assert seen == ["absent", (0, 0)]
    finally:
        stage_reference.remove_from_path(added)

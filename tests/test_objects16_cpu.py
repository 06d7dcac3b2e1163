"""CPU: 16-bit object factors kept at 16 bits (B200_F_OBJECTS_16BIT).

The header's flag equals `_lib`'s constant and the exports still equal the header; create with the flag accepts a host
fp16 matrix up to the device check (B200_E_CUDA without a GPU) while the same call without it is refused as before; the
storage choice of `object_storage_dtype`; and the engine cache never holding a 16-bit engine."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib, build

    build.build()
    return _lib.load()


def _header():
    return open(os.path.join(ROOT, "include", "b200_rank.h")).read()


def test_flag_matches_header_and_exports_unchanged(lib):
    from rectools_b200 import _lib

    header = _header()
    assert int(re.search(r"#define B200_F_OBJECTS_16BIT (\d+)", header).group(1)) == _lib.F_OBJECTS_16BIT
    assert int(re.search(r"#define B200_F_OBJECTS_ON_DEVICE (\d+)", header).group(1)) == _lib.F_OBJECTS_ON_DEVICE
    assert _lib.F_OBJECTS_16BIT & _lib.F_OBJECTS_ON_DEVICE == 0
    assert int(re.search(r"#define B200_RANK_ABI_VERSION (\d+)", header).group(1)) == _lib.ABI_VERSION == 6
    assert set(re.findall(r"\b(b200_rank_[a-z_]+)\s*\(", header)) == set(_lib.EXPORTS)
    for name in _lib.EXPORTS:
        assert getattr(lib, name) is not None


def _no_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_host_16bit_create(lib, dtype):
    """With the flag a host 16-bit matrix passes the argument checks and fails only for want of a device; without it the
    call is refused as a contract violation, as it always was.  The same holds for engine groups."""
    _no_gpu()
    from rectools_b200 import _lib

    dt = _lib.DT_F16 if dtype == "f16" else _lib.DT_BF16
    objects = np.ones((5, 3), np.float16)  # (bf16: the bytes are never read without a device)
    h = C.c_void_p()
    rc = lib.b200_rank_create_ex(C.byref(h), objects.ctypes.data, dt, 5, 3, _lib.DIST_DOT, 0, _lib.TC_AUTO, _lib.F_OBJECTS_16BIT)
    assert rc == _lib.E_CUDA, lib.b200_rank_last_error()
    assert b"no CUDA device" in lib.b200_rank_last_error()
    assert not h.value
    rc = lib.b200_rank_create_ex(C.byref(h), objects.ctypes.data, dt, 5, 3, _lib.DIST_DOT, 0, _lib.TC_AUTO, 0)
    assert rc == _lib.E_INVALID
    assert b"device pointers" in lib.b200_rank_last_error()
    devs = (C.c_int32 * 2)(0, 0)
    g = C.c_void_p()
    rc = lib.b200_rank_group_create_ex(C.byref(g), objects.ctypes.data, dt, 5, 3, _lib.DIST_DOT, devs, 2, _lib.TC_AUTO,
                                       _lib.F_OBJECTS_16BIT)
    assert rc == _lib.E_CUDA


def test_flag_with_fp32_objects_changes_nothing(lib):
    """fp32 objects: the flag is accepted and the call fails exactly where it fails without it (no device)."""
    _no_gpu()
    from rectools_b200 import _lib

    objects = np.ones((5, 3), np.float32)
    h = C.c_void_p()
    for flags in (0, _lib.F_OBJECTS_16BIT):
        rc = lib.b200_rank_create_ex(C.byref(h), objects.ctypes.data, _lib.DT_F32, 5, 3, _lib.DIST_COSINE, 0, _lib.TC_AUTO, flags)
        assert rc == _lib.E_CUDA


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
@pytest.mark.parametrize("distance", ["dot", "cosine", "euclidean"])
@pytest.mark.parametrize("keep", [True, False])
def test_storage_choice(dtype, distance, keep):
    """16-bit objects stay 16-bit with keep_16bit, except for EUCLIDEAN (the augmentation column is no 16-bit value)."""
    import torch

    from rectools_b200 import _lib
    from rectools_b200.ranker import Distance, object_storage_dtype

    want = {"float16": _lib.DT_F16, "bfloat16": _lib.DT_BF16}[dtype] if keep and distance != "euclidean" else _lib.DT_F32
    tdt = getattr(torch, dtype)
    assert object_storage_dtype(distance, tdt, keep) == want
    assert object_storage_dtype(Distance(distance), dtype, keep) == want
    if dtype == "float16":
        assert object_storage_dtype(distance, np.float16, keep) == want
        assert object_storage_dtype(distance, np.zeros(1, np.float16).dtype, keep) == want


@pytest.mark.parametrize("distance", ["dot", "cosine", "euclidean"])
def test_storage_choice_wider_types_are_fp32(distance):
    import torch

    from rectools_b200 import _lib
    from rectools_b200.ranker import object_storage_dtype

    for dt in (np.float32, np.float64, np.int32, torch.float32, torch.float64, "float32"):
        for keep in (True, False):
            assert object_storage_dtype(distance, dt, keep) == _lib.DT_F32


def test_cached_engines_are_fp32(monkeypatch):
    """`B200ImplicitRanker` hands `cached_engine` the fp32 matrix, so numpy fp16 objects and their fp32 copy share one
    widened engine, and no 16-bit engine is ever created through the cache."""
    from rectools_b200 import integration

    made = []

    def fake_new_engine(objects, cosine, device, tc_mode="auto", keep_16bit=False, **kw):
        made.append((objects.dtype, keep_16bit, kw))
        return object()

    monkeypatch.setattr(integration, "new_engine", fake_new_engine)
    integration.clear_engine_cache()
    rng = np.random.default_rng(0)
    objects16 = rng.standard_normal((50, 8)).astype(np.float16)
    subjects = rng.standard_normal((4, 8)).astype(np.float32)
    try:
        with pytest.raises(AttributeError):  # (the stand-in engine cannot hold subjects: only the cache path matters)
            integration.B200ImplicitRanker("dot", subjects, objects16)
        e1 = integration.cached_engine(objects16.astype(np.float32), False, 0, "auto")
        assert len(made) == 1 and made[0] == (np.float32, False, {})
        assert e1 is integration.cached_engine(integration._dense_f32(objects16), False, 0, "auto")  # pylint: disable=protected-access
        assert integration.content_hash(objects16) != integration.content_hash(objects16.astype(np.float32))
    finally:
        integration.clear_engine_cache()

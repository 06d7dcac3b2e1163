"""CPU: without a CUDA device, the engine-less entry points get past their argument checks and fail at their first CUDA
call; each reports B200_E_CUDA with its own name and the line of the failed call."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def lib():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from rectools_b200 import _lib, build

    build.build()
    return _lib.load()


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data


def _check_cuda_failure(lib, rc: int, name: str) -> None:
    from rectools_b200 import _lib

    msg = lib.b200_rank_last_error().decode()
    assert rc == _lib.E_CUDA, (rc, msg)
    assert msg.startswith(name + ": "), msg
    assert "failed at line" in msg, msg


def test_list_reports_cuda_failure(lib):
    from rectools_b200 import _lib

    ids = np.arange(5, dtype=np.int32)
    indptr = np.array([0, 1, 1], dtype=np.int64)
    indices = np.array([2], dtype=np.int32)
    pos = np.full((2, 3), -7, dtype=np.int32)
    counts = np.full(2, -7, dtype=np.int32)
    st = _lib.Stats()
    rc = lib.b200_rank_topk_list(0, 5, _ptr(ids), 2, _ptr(indptr), _ptr(indices), 3, _ptr(pos), _ptr(counts), C.byref(st))
    _check_cuda_failure(lib, rc, "b200_rank_topk_list")
    assert (pos == -7).all() and (counts == -7).all()


def test_list_mix_reports_cuda_failure(lib):
    from rectools_b200 import _lib

    offsets = np.array([0, 3, 5], dtype=np.int64)
    ids = np.array([4, 1, 0, 2, 3], dtype=np.int32)
    quota = np.array([2, 1], dtype=np.int32)
    indptr = np.array([0, 1, 1], dtype=np.int64)
    indices = np.array([1], dtype=np.int32)
    pos = np.full((2, 3), -7, dtype=np.int32)
    counts = np.full(2, -7, dtype=np.int32)
    st = _lib.Stats()
    rc = lib.b200_rank_topk_list_mix(0, 2, _ptr(offsets), _ptr(ids), _ptr(quota), _lib.MIX_ROTATE, 2, _ptr(indptr), _ptr(indices), 3,
                                     _ptr(pos), _ptr(counts), C.byref(st))
    _check_cuda_failure(lib, rc, "b200_rank_topk_list_mix")
    assert (pos == -7).all() and (counts == -7).all()


def test_pairs_reports_cuda_failure(lib):
    from rectools_b200 import _lib

    codes = np.array([0, 1, 0, 1], dtype=np.int64)
    scores = np.array([0.5, 0.25, 1.0, 2.0], dtype=np.float32)
    out_pos = np.full(4, -7, dtype=np.int64)
    out_off = np.full(3, -7, dtype=np.int64)
    st = _lib.Stats()
    rc = lib.b200_rank_topk_pairs(0, None, 4, _ptr(codes), _ptr(scores), _lib.PAIRS_F32, 2, 2, 0, _ptr(out_pos), _ptr(out_off),
                                  C.byref(st))
    _check_cuda_failure(lib, rc, "b200_rank_topk_pairs")


def test_merge_reports_cuda_failure(lib):
    n_lists, n_rows, k = 2, 3, 4
    ids = np.zeros((n_lists, n_rows, k), dtype=np.int32)
    scores = np.zeros((n_lists, n_rows, k), dtype=np.float32)
    counts = np.zeros((n_lists, n_rows), dtype=np.int32)
    out_ids = np.zeros((n_rows, k), dtype=np.int32)
    out_scores = np.zeros((n_rows, k), dtype=np.float32)
    out_counts = np.zeros(n_rows, dtype=np.int32)
    rc = lib.b200_rank_merge(0, None, n_lists, n_rows, k, _ptr(ids), _ptr(scores), _ptr(counts), _ptr(out_ids), _ptr(out_scores),
                             _ptr(out_counts))
    _check_cuda_failure(lib, rc, "b200_rank_merge")

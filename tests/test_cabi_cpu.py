"""CPU: the C-ABI library builds/loads, exports every symbol include/b200_rank.h declares, and fails loudly (no CPU
fallback) when there is no CUDA device.  Host-side logic that needs no GPU is covered here too."""
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


def test_exports_match_header(lib):
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    declared = set(re.findall(r"\b(b200_rank_[a-z_]+)\s*\(", header))
    assert declared == set(_lib.EXPORTS)
    for name in declared:
        assert getattr(lib, name) is not None
    assert lib.b200_rank_abi_version() == _lib.ABI_VERSION


def test_struct_layouts_match_header():
    """ctypes mirrors must list exactly the header's fields, in order."""
    from rectools_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200_rank.h")).read()
    for cname, struct in (
        ("b200_rank_query", _lib.Query),
        ("b200_rank_stats", _lib.Stats),
        ("b200_rank_info", _lib.Info),
        ("b200_rank_snapshot", _lib.Snapshot),
    ):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (cname, cname), header, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = [re.search(r"(\w+)(\[\d+\])?\s*$", stmt.strip()).group(1) for stmt in body.split(";") if stmt.strip()]
        assert names == [f[0] for f in struct._fields_], cname


def test_no_cpu_fallback_without_gpu(lib):
    import ctypes as C

    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from rectools_b200 import B200Ranker, _lib

    with pytest.raises(_lib.B200RankError):
        B200Ranker("dot", np.ones((2, 3), np.float32), np.ones((4, 3), np.float32))
    h = C.c_void_p()
    assert lib.b200_rank_create(C.byref(h), None, 0, 0, 0, 0, 0, 0) == _lib.E_INVALID
    assert b"bad object matrix" in lib.b200_rank_last_error()


def test_flatten_padded():
    from rectools_b200 import flatten_padded

    sids = np.array([5, 2, 9])
    ids = np.array([[1, 2, -1], [3, -1, -1], [4, 5, 6]], dtype=np.int32)
    sc = np.array([[3, 2, 0], [1, 0, 0], [9, 8, 7]], dtype=np.float32)
    s, i, c = flatten_padded(sids, ids, sc, np.array([2, 1, 3], dtype=np.int32))
    np.testing.assert_array_equal(s, [5, 5, 2, 9, 9, 9])
    np.testing.assert_array_equal(i, [1, 2, 3, 4, 5, 6])
    np.testing.assert_array_equal(c, [3, 2, 1, 9, 8, 7])
    s, i, c = flatten_padded(sids, ids, sc, np.array([3, 3, 3], dtype=np.int32))
    assert len(s) == 9


def test_cpu_baseline_matches_oracle():
    """The timed CPU baseline (numpy sgemm + C/OpenMP select) agrees with the numpy restatement."""
    from oracle import cpu_baseline
    from oracle.topk_oracle import calc_norms, implicit_topk
    from tests.helpers import synth_factors, synth_viewed_csr

    u, i = synth_factors(200, 3000, 32, seed=9)
    csr = synth_viewed_csr(200, 3000, 25)
    for norms in (None, calc_norms(i)):
        ids, sc = cpu_baseline.topk_cpu(i, u, 10, norms, csr)
        oid, osc = implicit_topk(i, u, 10, norms, csr)
        np.testing.assert_array_equal(ids, oid)
        np.testing.assert_allclose(sc, osc, rtol=1e-6)

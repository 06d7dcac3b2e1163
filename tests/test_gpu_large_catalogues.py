"""GPU: one engine holding a whole config-4 or config-5 catalogue, against the fp64 oracle.

An engine group replicates the whole catalogue on every member, and the sizes BASELINE.json quotes for configs 4 and 5
are said to fit on one H100.  At config 4 (10M x 128 fp32) the master copy is 5.12 GB, so element offsets pass 2^32 and
the fp16 tensor-core copy (2.56 GB) passes 2^31 bytes; at config 5 (5M x 256 bf16 kept at 16 bits) the borrowed matrix and
the tensor-core copy are 2.56 GB each.  `test_gpu_scale.py` stops at 1M objects.

Results are held to the rounding-interval checker of `tests/score_interval.py` (blocks of objects, so that no fp64 copy
of the catalogue is held): every score one of the fp32 values its fp64 sum can round to, no eligible object left out
ahead of a row's k-th entry, no tolerance and no swapped neighbours, on sampled rows of the largest k of each route.
Every engine kernel sums a pair's terms in index order, so the smaller k of the same catalogue must be bit-identical
prefixes of the checked results, on all rows.

64 sampled rows (spread evenly over the 4096) are checked per route.  Each check scores every object of a row, so one
row is 10M interval checks at config 4 and a 64-row check costs about 90 s of host time; the rows are not special (one
subject generator, the same filter density), and the routes' row-dependent decisions -- fallback, row-list re-rank --
are exercised across all rows by the bit-identical prefix comparisons and, at smaller sizes, by
`tests/test_gpu_score_bits.py` on every row.  256 rows would multiply the file's run time by about four.

Memory: the config-4 engine reports `hbm_bytes` = 8.00 GB after create (master copy, tensor-core copy, norms, staging);
engines are closed between tests.  Path 3 cuts at least 32 rows per chunk whatever N is (`run_dense_large_k`): at
N = 10M that is 1.28 GB of fp32 scores per chunk before any sort scratch, above the 1 GiB budget the chunk rule aims at
(a known gap, not changed here; the k = None call below ranks 8 rows)."""
import time

import numpy as np
import pytest

from tests.helpers import synth_viewed_csr
from tests.score_interval import check_topk
from tests.test_gpu_scale import BLOCK, gen_factors

pytestmark = pytest.mark.gpu

N4, D4 = 10_000_000, 128
N5, D5 = 5_000_000, 256
N_SUBJECTS = 4096


# ------------------------------------------------------------------------------------------------ comparisons
def _same_prefix(got, ref, name):
    """`got` (k columns) is the first k columns of `ref`, bit for bit, counts included."""
    ids, sc, cnt = got
    k = ids.shape[1]
    np.testing.assert_array_equal(cnt, np.minimum(ref[2], k), err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, ref[0][:, :k], err_msg=f"{name}: ids")
    np.testing.assert_array_equal(sc.view(np.int32), ref[1][:, :k].view(np.int32), err_msg=f"{name}: scores")


# ------------------------------------------------------------------------------------------------ config 4
@pytest.fixture(scope="module")
def c4():
    """10M x 128 fp32 objects (bench's generator), 4096 subjects with 100 viewed objects each, 64 sampled rows."""
    t0 = time.time()
    objects = gen_factors(N4, D4, 1)
    subjects = gen_factors(N_SUBJECTS, D4, 0)
    csr = synth_viewed_csr(N_SUBJECTS, N4, 100)
    rows = np.unique(np.linspace(0, N_SUBJECTS - 1, 64).astype(np.int64))
    print(f"config 4: catalogue {time.time() - t0:.1f} s")
    yield objects, subjects, csr, rows


@pytest.fixture
def c4_engine(c4):
    from rectools_b200 import Engine

    eng = Engine(c4[0], cosine=False)
    info = eng.info()
    print(f"config 4 engine: hbm_bytes {info['hbm_bytes'] / 1e9:.2f} GB, tc_dtype {info['tc_dtype']}")
    yield eng
    eng.close()


def test_c4_tensor_core_routes(lib_consts, c4, c4_engine):
    """k = 10 (FORCE_TC), 100 (wide) and 1000 (wide, k > 128) over all 4096 subjects: k = 1000 on the sampled rows against
    the score intervals, k = 10 and 100 its bit-identical prefixes on every row."""
    objects, subjects, csr, rows = c4
    eng = c4_engine
    res = {}
    for k, flags, wide in ((10, lib_consts.Q_FORCE_TC, 0), (100, 0, 1), (1000, 0, 1)):
        t0 = time.time()
        res[k] = eng.topk(k, subjects=subjects, indptr=csr.indptr, indices=csr.indices, flags=flags)
        st = eng.last_stats
        print(f"config 4 k={k}: path {st['path']} wide {st['wide']} n_fallback_rows {st['n_fallback_rows']} "
              f"n_exact_rows {st.get('n_exact_rows')} ({time.time() - t0:.1f} s)")
        assert (st["path"], st["wide"]) == (1, wide), st
        assert st["n_fallback_rows"] <= N_SUBJECTS // 2, st
        assert (res[k][2] == k).all()
    t0 = time.time()
    check_topk(tuple(a[rows] for a in res[1000]), subjects[rows], objects, 1000, filter_csr=csr[rows], name="config 4 k=1000")
    print(f"config 4 check of {len(rows)} rows: {time.time() - t0:.1f} s")
    for k in (10, 100):
        _same_prefix(res[k], res[1000], f"config 4 k={k} against k=1000")


def test_c4_exhaustive_and_radix_routes(lib_consts, c4, c4_engine):
    """The sampled rows on path 3 at k = 1025 against the score intervals, FORCE_EXACT at k = 10 its prefix; 8 rows at
    k = None (10M entries each) against the score intervals."""
    objects, subjects, csr, rows = c4
    eng = c4_engine
    f = csr[rows]
    res = {}
    for k, flags, path in ((10, lib_consts.Q_FORCE_EXACT, 0), (1025, 0, 3)):
        res[k] = eng.topk(k, subjects=subjects[rows], indptr=f.indptr, indices=f.indices, flags=flags)
        assert eng.last_stats["path"] == path, eng.last_stats
    check_topk(res[1025], subjects[rows], objects, 1025, filter_csr=f, name="config 4 path 3 k=1025")
    _same_prefix(res[10], res[1025], "config 4 path 0 k=10 against path 3 k=1025")
    s8 = rows[:8]
    f8 = csr[s8]
    t0 = time.time()
    got = eng.topk(N4, subjects=subjects[s8], indptr=f8.indptr, indices=f8.indices)
    assert eng.last_stats["path"] == 3, eng.last_stats
    print(f"config 4 k=None, 8 rows: {time.time() - t0:.1f} s")
    t0 = time.time()
    check_topk(got, subjects[s8], objects, None, filter_csr=f8, name="config 4 k=None")
    print(f"config 4 k=None check: {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ config 5
@pytest.fixture(scope="module")
def c5(torch):
    """5M x 256 bf16 objects on the device (bench's generator, rounded to bf16), their CPU copy, 4096 bf16-exact fp32
    subjects with 50 viewed objects each.  The catalogue is generated in steps of 1M rows, each of whole 64 K-row seeded
    blocks of `gen_factors`, so that no fp32 copy of all of it is held."""
    dev = torch.device("cuda:0")
    items = torch.empty((N5, D5), dtype=torch.bfloat16, device=dev)
    host = torch.empty((N5, D5), dtype=torch.bfloat16)
    step = 16 * BLOCK
    for r0 in range(0, N5, step):
        r1 = min(r0 + step, N5)
        blk = np.empty((r1 - r0, D5), np.float32)
        for b in range(r0 // BLOCK, (r1 + BLOCK - 1) // BLOCK):
            a0, a1 = b * BLOCK, min((b + 1) * BLOCK, r1)
            g = np.random.default_rng([1, b]).standard_normal((a1 - a0, D5), dtype=np.float32)
            g *= np.float32(1.0 / np.sqrt(D5))
            blk[a0 - r0 : a1 - r0] = g
        host[r0:r1] = torch.from_numpy(blk).to(torch.bfloat16)
    items.copy_(host)
    subjects = torch.from_numpy(gen_factors(N_SUBJECTS, D5, 0)).to(torch.bfloat16).float().numpy()
    csr = synth_viewed_csr(N_SUBJECTS, N5, 50)
    torch.cuda.synchronize()
    yield items, host, subjects, csr
    del items


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def lib_consts():
    from rectools_b200 import _lib

    return _lib


def test_c5_bf16_kept_and_widened(lib_consts, torch, c5):
    """k = 20 over all 4096 rows on the engine that keeps the bf16 matrix at 16 bits (read in place) and on the engine
    that widens it: bit-identical; 64 rows against the score intervals; one call on a 16-bit engine over the matrix at
    element offset 1 (the element-wise re-score at size), bit-identical on those rows."""
    from rectools_b200 import Engine

    items, host, subjects, csr = c5
    kw = dict(objects_device_ptr=items.data_ptr(), shape=(N5, D5), objects_dtype=lib_consts.DT_BF16)
    rows = np.unique(np.linspace(0, N_SUBJECTS - 1, 64).astype(np.int64))
    call = dict(subjects=subjects, indptr=csr.indptr, indices=csr.indices)
    kept = Engine(None, cosine=False, keep_16bit=True, **kw)
    try:
        got = kept.topk(20, **call)
        st = kept.last_stats
        print(f"config 5 kept: hbm_bytes {kept.info()['hbm_bytes'] / 1e9:.2f} GB, path {st['path']} wide {st['wide']} "
              f"n_fallback_rows {st['n_fallback_rows']}")
        assert st["path"] == 1 and st["tc_dtype"] == lib_consts.TC_BF16, st
        assert st["n_fallback_rows"] <= N_SUBJECTS // 2, st
    finally:
        kept.close()
    wide = Engine(None, cosine=False, **kw)
    try:
        ref = wide.topk(20, **call)
        print(f"config 5 widened: n_fallback_rows {wide.last_stats['n_fallback_rows']}")
    finally:
        wide.close()
    for a, b, what in zip(got, ref, ("ids", "scores", "counts")):
        np.testing.assert_array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                      b.view(np.int32) if b.dtype == np.float32 else b, err_msg=f"config 5 kept vs widened: {what}")
    t0 = time.time()
    check_topk(tuple(a[rows] for a in got), subjects[rows], host, 20, filter_csr=csr[rows], name="config 5 k=20")
    print(f"config 5 check of {len(rows)} rows: {time.time() - t0:.1f} s")
    # the same matrix one element into a fresh allocation: rows start 2 bytes past 16-byte boundaries
    flat = items.view(-1)
    moved_buf = torch.empty((flat.numel() + 8,), dtype=torch.bfloat16, device=items.device)
    moved = moved_buf[1 : 1 + flat.numel()].view(N5, D5)
    moved.copy_(items)
    assert moved.data_ptr() % 16 == 2
    torch.cuda.synchronize()
    odd = Engine(None, cosine=False, keep_16bit=True, objects_device_ptr=moved.data_ptr(), shape=(N5, D5),
                 objects_dtype=lib_consts.DT_BF16)
    try:
        f = csr[rows]
        for k, flags in ((20, 0), (20, lib_consts.Q_FORCE_EXACT)):
            o = odd.topk(k, subjects=subjects[rows], indptr=f.indptr, indices=f.indices, flags=flags)
            _same_prefix(o, tuple(a[rows] for a in got), f"config 5 at offset 1 flags={flags}")
    finally:
        odd.close()
        del moved, moved_buf

"""GPU: one engine holding a whole config-4 or config-5 catalogue, against the fp64 oracle.

An engine group replicates the whole catalogue on every member, and the sizes BASELINE.json quotes for configs 4 and 5
are said to fit on one H100.  At config 4 (10M x 128 fp32) the master copy is 5.12 GB, so element offsets pass 2^32 and
the fp16 tensor-core copy (2.56 GB) passes 2^31 bytes; at config 5 (5M x 256 bf16 kept at 16 bits) the borrowed matrix and
the tensor-core copy are 2.56 GB each.  `test_gpu_scale.py` stops at 1M objects.

`rank_oracle` widens the whole catalogue to fp64 at once (10 GB at config 4), so the oracle here scores blocks of 1M
objects and merges a running top-k by (score desc, id asc); `tests/test_large_catalogue_oracle_cpu.py` pins it against
`rank_oracle` on small inputs.  The oracle's fp64 sums come from BLAS, in another order than the engine's, so a score can
round to the neighbouring fp32 value (about one in 10^8): ids are compared exactly on the sampled rows up to k = 1025, and
the k = None rows (10M entries each) allow such one-ulp neighbours to swap.

Memory: the config-4 engine reports `hbm_bytes` = 8.00 GB after create (master copy, tensor-core copy, norms, staging);
engines are closed between tests.  Path 3 cuts at least 32 rows per chunk whatever N is (`run_dense_large_k`): at
N = 10M that is 1.28 GB of fp32 scores per chunk before any sort scratch, above the 1 GiB budget the chunk rule aims at
(a known gap, not changed here; the k = None call below ranks 8 rows)."""
import time

import numpy as np
import pytest

from oracle.topk_oracle import NEG_SENTINEL, calc_norms, neginf_score
from tests.helpers import synth_viewed_csr
from tests.test_gpu_scale import BLOCK, gen_factors

pytestmark = pytest.mark.gpu

BLOCK_OBJECTS = 1 << 20
N4, D4 = 10_000_000, 128
N5, D5 = 5_000_000, 256
N_SUBJECTS = 4096
NEG_MAX = np.float32(-np.finfo(np.float32).max)


# ------------------------------------------------------------------------------------------------ the blocked oracle
def _order_keys(scores: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """uint64 keys whose ascending order is (score desc, id asc): the high word inverts the monotone map of the fp32 bit
    pattern, the low word is the id."""
    u = np.ascontiguousarray(scores, np.float32).view(np.uint32)
    mono = np.where(u >> 31, ~u, u | np.uint32(0x80000000)).astype(np.uint32)  # ascending in the score
    return ((~mono).astype(np.uint64) << np.uint64(32)) | ids.astype(np.uint64)


def _from_keys(keys: np.ndarray) -> tuple:
    ids = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    inv = ~(keys >> np.uint64(32)).astype(np.uint32)
    bits = np.where(inv >> 31, inv & np.uint32(0x7FFFFFFF), ~inv).astype(np.uint32)
    return ids, bits.view(np.float32)


def _rows_f32(objects, sel) -> np.ndarray:
    """Rows `sel` (a slice or ids) of a numpy matrix or a CPU torch tensor (any float type, widened exactly) as fp32."""
    if hasattr(objects, "float"):
        import torch

        return objects[sel if isinstance(sel, slice) else torch.from_numpy(sel)].float().numpy()
    return np.asarray(objects[sel], np.float32)


def blocked_oracle(distance, subjects, objects, k, filter_csr=None, whitelist=None, block=BLOCK_OBJECTS, row_block=64):
    """The engine's answer in padded form (`ec.expected_padded`'s), computed over blocks of `block` positions: fp64 dot
    rounded once to fp32 (COSINE: / the fp32 object norm), filtered pairs at -FLT_MAX, a running top-k per row merged by
    (score desc, id asc), then the trailing sentinel strip as counts (slots beyond: id -1 / score -FLT_MAX).
    `subjects` [n, d] are the batch rows; `filter_csr` [n, >= ids] filters by object id; `whitelist` (sorted) restricts
    the positions.  Returns (ids int32 [n, k_out], scores fp32, counts int32)."""
    subjects = np.asarray(subjects, np.float64)
    n = subjects.shape[0]
    wl = None if whitelist is None else np.asarray(whitelist, np.int64)
    n_pos = objects.shape[0] if wl is None else len(wl)
    k_out = min(n_pos if k is None else int(k), n_pos)
    run = np.empty((n, 0), np.uint64)
    for p0 in range(0, n_pos, block):
        p1 = min(p0 + block, n_pos)
        ids = np.arange(p0, p1, dtype=np.int64) if wl is None else wl[p0:p1]
        blk = _rows_f32(objects, slice(p0, p1) if wl is None else ids)
        blk64 = blk.astype(np.float64)
        norms = calc_norms(blk, "f64").astype(np.float64) if distance == "cosine" else None
        parts = []
        for r0 in range(0, n, row_block):
            r1 = min(r0 + row_block, n)
            s = subjects[r0:r1] @ blk64.T
            if norms is not None:
                s = s / norms[None, :]
            s = s.astype(np.float32) + np.float32(0)  # (-0.0 -> +0.0: the sign of an exact zero is not part of the result)
            if filter_csr is not None:
                for r in range(r0, r1):
                    cols = filter_csr.indices[filter_csr.indptr[r] : filter_csr.indptr[r + 1]]
                    if wl is None:
                        s[r - r0, cols[(cols >= p0) & (cols < p1)] - p0] = NEG_SENTINEL
                    else:
                        s[r - r0, np.isin(ids, cols)] = NEG_SENTINEL
            keys = _order_keys(s, np.broadcast_to(ids, s.shape))
            if k_out < keys.shape[1]:
                keys = np.partition(keys, k_out - 1, axis=1)[:, :k_out]
            parts.append(np.sort(keys, axis=1))
        cand = np.concatenate(parts, axis=0)
        # two sorted runs per row: the stable sort (timsort) merges them
        run = np.sort(np.concatenate([run, cand], axis=1), axis=1, kind="stable")[:, :k_out]
    ids, sc = _from_keys(run)
    valid = sc > np.float32(neginf_score())
    counts = valid.sum(axis=1).astype(np.int32)
    assert (valid == (np.arange(k_out)[None, :] < counts[:, None])).all()
    return np.where(valid, ids, -1).astype(np.int32), np.where(valid, sc, NEG_MAX).astype(np.float32), counts


# ------------------------------------------------------------------------------------------------ comparisons
def _check(got, exp, name, rtol=3e-7):
    """Exact ids and counts, scores within fp32 rounding of the oracle's."""
    ids, sc, cnt = got
    eids, esc, ecnt = exp
    assert ids.shape == eids.shape, f"{name}: shape {ids.shape} vs {eids.shape}"
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, eids, err_msg=f"{name}: ids")
    np.testing.assert_allclose(sc, esc, rtol=rtol, atol=1e-30, err_msg=f"{name}: scores")


def _check_full_rows(got, exp, objects_score, name):
    """k = None rows: counts exact; at every position the two scores agree to one fp32 rounding; where the ids differ,
    the engine's id scores (recomputed) what the oracle has there, so only near-equal neighbours swapped."""
    ids, sc, cnt = got
    eids, esc, ecnt = exp
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_allclose(sc, esc, rtol=3e-7, atol=1e-30, err_msg=f"{name}: scores")
    swapped = 0
    for r in range(ids.shape[0]):
        bad = np.nonzero(ids[r] != eids[r])[0]
        swapped += len(bad)
        if len(bad):
            assert (bad < cnt[r]).all(), f"{name}: row {r} differs in its padding"
            np.testing.assert_allclose(objects_score(r, ids[r, bad]), esc[r, bad], rtol=3e-7, err_msg=f"{name}: row {r} swapped ids")
    total = int(cnt.sum())
    print(f"{name}: {swapped} of {total} positions hold a one-rounding neighbour")
    assert swapped <= max(16, total // 10**6), f"{name}: {swapped} swapped positions"


# ------------------------------------------------------------------------------------------------ config 4
@pytest.fixture(scope="module")
def c4():
    """10M x 128 fp32 objects (bench's generator), 4096 subjects with 100 viewed objects each, 256 sampled rows and
    their oracle at k = 1025 (every smaller k is its prefix)."""
    t0 = time.time()
    objects = gen_factors(N4, D4, 1)
    subjects = gen_factors(N_SUBJECTS, D4, 0)
    csr = synth_viewed_csr(N_SUBJECTS, N4, 100)
    rows = np.unique(np.linspace(0, N_SUBJECTS - 1, 256).astype(np.int64))
    t1 = time.time()
    exp = blocked_oracle("dot", subjects[rows], objects, 1025, csr[rows])
    print(f"config 4: catalogue {t1 - t0:.1f} s, oracle of {len(rows)} rows at k = 1025 {time.time() - t1:.1f} s")
    yield objects, subjects, csr, rows, exp


def _prefix(exp, k, rows=slice(None)):
    ids, sc, cnt = exp
    return ids[rows, :k], sc[rows, :k], np.minimum(cnt[rows], k)


@pytest.fixture
def c4_engine(c4):
    from rectools_b200 import Engine

    eng = Engine(c4[0], cosine=False)
    info = eng.info()
    print(f"config 4 engine: hbm_bytes {info['hbm_bytes'] / 1e9:.2f} GB, tc_dtype {info['tc_dtype']}")
    yield eng
    eng.close()


def test_c4_tensor_core_routes(lib_consts, c4, c4_engine):
    """k = 10 (FORCE_TC), 100 (wide) and 1000 (wide, k > 128) over all 4096 subjects; 256 sampled rows against the
    oracle."""
    objects, subjects, csr, rows, exp = c4
    eng = c4_engine
    for k, flags, wide in ((10, lib_consts.Q_FORCE_TC, 0), (100, 0, 1), (1000, 0, 1)):
        t0 = time.time()
        got = eng.topk(k, subjects=subjects, indptr=csr.indptr, indices=csr.indices, flags=flags)
        st = eng.last_stats
        print(f"config 4 k={k}: path {st['path']} wide {st['wide']} n_fallback_rows {st['n_fallback_rows']} "
              f"n_exact_rows {st.get('n_exact_rows')} ({time.time() - t0:.1f} s)")
        assert (st["path"], st["wide"]) == (1, wide), st
        assert st["n_fallback_rows"] <= N_SUBJECTS // 2, st
        assert (got[2] == k).all()
        _check(tuple(a[rows] for a in got), _prefix(exp, k), f"config 4 k={k}")


def test_c4_exhaustive_and_radix_routes(lib_consts, c4, c4_engine):
    """64 rows with FORCE_EXACT at k = 10, 64 rows on path 3 at k = 1025, 8 rows at k = None."""
    objects, subjects, csr, rows, exp = c4
    eng = c4_engine
    r64 = np.arange(0, len(rows), len(rows) // 64)[:64]
    sids = rows[r64]
    f = csr[sids]
    for k, flags, path in ((10, lib_consts.Q_FORCE_EXACT, 0), (1025, 0, 3)):
        got = eng.topk(k, subjects=subjects[sids], indptr=f.indptr, indices=f.indices, flags=flags)
        assert eng.last_stats["path"] == path, eng.last_stats
        _check(got, _prefix(exp, k, r64), f"config 4 path {path} k={k}")
    s8 = rows[r64[:8]]
    f8 = csr[s8]
    t0 = time.time()
    got = eng.topk(N4, subjects=subjects[s8], indptr=f8.indptr, indices=f8.indices)
    assert eng.last_stats["path"] == 3, eng.last_stats
    print(f"config 4 k=None, 8 rows: {time.time() - t0:.1f} s")
    t0 = time.time()
    full = blocked_oracle("dot", subjects[s8], objects, None, f8)
    print(f"config 4 k=None oracle: {time.time() - t0:.1f} s")
    sub64 = subjects[s8].astype(np.float64)
    _check_full_rows(got, full, lambda r, ids: (objects[ids].astype(np.float64) @ sub64[r]).astype(np.float32), "config 4 k=None")


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
    that widens it: bit-identical; 256 rows against the oracle; one call on a 16-bit engine over the matrix at element
    offset 1 (the element-wise re-score at size)."""
    from rectools_b200 import Engine

    items, host, subjects, csr = c5
    kw = dict(objects_device_ptr=items.data_ptr(), shape=(N5, D5), objects_dtype=lib_consts.DT_BF16)
    rows = np.unique(np.linspace(0, N_SUBJECTS - 1, 256).astype(np.int64))
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
    exp = blocked_oracle("dot", subjects[rows], host, 20, csr[rows])
    print(f"config 5 oracle of {len(rows)} rows: {time.time() - t0:.1f} s")
    _check(tuple(a[rows] for a in got), exp, "config 5 k=20")
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
        sub = rows[:64]
        f = csr[sub]
        for k, flags in ((20, 0), (20, lib_consts.Q_FORCE_EXACT)):
            o = odd.topk(k, subjects=subjects[sub], indptr=f.indptr, indices=f.indices, flags=flags)
            _check(o, _prefix(exp, k, slice(0, 64)), f"config 5 at offset 1 flags={flags}")
    finally:
        odd.close()
        del moved, moved_buf

"""GPU: every ranking route held to the rounding-interval oracle of `tests/score_interval.py`, on continuous factors, with
no tolerance.

Each case ranks and runs the strict checker on ALL rows: every returned score must be one of the fp32 values an fp64 sum
of its pair can round to (almost always exactly one), ids unique and eligible, rows in (score desc, id asc) order, and
no eligible object left out that ranks before a row's k-th entry.  Where two routes rank the same call, their padded
results must also be bit-identical.  Each case prints its checked-entry count, its ambiguous count and its fallback
counts."""
import numpy as np
import pytest
from scipy import sparse

from tests.helpers import synth_factors, synth_viewed_csr
from tests.score_interval import check_topk, norm_interval, widen64

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


def _stats(st):
    return (f"path {st['path']} wide {st['wide']} launches {st['n_tc_launches']} fallback {st['n_fallback_rows']} "
            f"exact {st.get('n_exact_rows')}")


def _same(a, b, name):
    for x, y, what in zip(a, b, ("ids", "scores", "counts")):
        np.testing.assert_array_equal(np.asarray(x).view(np.int32), np.asarray(y).view(np.int32), err_msg=f"{name}: {what}")


def _near_ties(n_rows=1200, n_obj=24_000, d=64, seed=9):
    """Every row scores 300 planted objects highest, within ~1e-6 relative of each other: far below the 16-bit operand
    resolution, so the candidate pass cannot order them and rows go to the 32-slot pass and the exhaustive kernel."""
    rng = np.random.default_rng(seed)
    u = (rng.standard_normal((n_rows, d)) / np.sqrt(d)).astype(np.float32)
    i = (0.2 * rng.standard_normal((n_obj, d)) / np.sqrt(d)).astype(np.float32)
    base = u.mean(axis=0) + 0.5 * rng.standard_normal(d).astype(np.float32) / np.sqrt(d)
    hot = rng.choice(n_obj, 300, replace=False)
    i[hot] = (3.0 * base[None, :] * (1.0 + 1e-6 * rng.standard_normal((300, 1)))).astype(np.float32)
    u = (u * 0.05 + base[None, :]).astype(np.float32)
    # the other half of the rows: plain random subjects
    u[n_rows // 2 :] = (rng.standard_normal((n_rows - n_rows // 2, d)) / np.sqrt(d)).astype(np.float32)
    return u, i


@pytest.fixture(scope="module")
def data():
    u, i = synth_factors(1024, 40_000, 64, seed=77)
    csr = synth_viewed_csr(1024, 40_000, 60, seed=78)
    return u, i, csr


# ------------------------------------------------------------------------------------------------ path 1, narrow
@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("tc_mode", ["fp16", "bf16"])
def test_path1_narrow_near_ties(lib, distance, tc_mode):
    """k = 1, 10, 24 with a filter, a whitelist and an id offset (the engine holds objects [3000, 27000) of a larger
    catalogue); the same call on the exhaustive kernel must be bit-identical."""
    from rectools_b200 import Engine

    u, i = _near_ties()
    id_off = 3_000
    rng = np.random.default_rng(5)
    wl = np.sort(rng.choice(len(i), len(i) * 3 // 4, replace=False)).astype(np.int32)
    csr = synth_viewed_csr(len(u), len(i) + 2 * id_off, 40, seed=6)
    eng = Engine(i, cosine=distance == "cosine", tc_mode=tc_mode, id_offset=id_off)
    try:
        fb = 0
        for k in (1, 10, 24):
            got = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, whitelist=wl, flags=lib.Q_FORCE_TC)
            st = dict(eng.last_stats)
            name = f"narrow {distance}/{tc_mode} k={k} [{_stats(st)}]"
            assert st["path"] == 1, name
            fb += st["n_fallback_rows"]
            check_topk(got, u, i, k, cosine=distance == "cosine", filter_csr=csr, whitelist=wl, id_offset=id_off, name=name)
            ref = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, whitelist=wl, flags=lib.Q_FORCE_EXACT)
            assert eng.last_stats["path"] == 0
            _same(got, ref, name)
        assert fb > 0
    finally:
        eng.close()


def _tied_copies(n_rows=1024, n_obj=40_000, d=64, n_copies=600, seed=13):
    """Exact fp32 ties across the cut: `n_copies` identical objects at ids spread over the whole catalogue (every tile
    split and list of the candidate pass) score highest for the first half of the rows, so each of those rows' top k is
    the k SMALLEST ids of the copies, all tied with the k-th entry; a pass that keeps a larger id drops a tied object at
    a smaller one.  Above them sit 5 strictly better objects for DOT (the cut falls at k - 5 copies); for COSINE they
    point the same way, so all 605 objects tie."""
    rng = np.random.default_rng(seed)
    u, i = synth_factors(n_rows, n_obj, d, seed=seed)
    ids = rng.choice(n_obj, n_copies + 5, replace=False)
    copies, best = ids[:n_copies], ids[n_copies:]
    v = u[: n_rows // 2].mean(axis=0) + 0.3 * rng.standard_normal(d).astype(np.float32) / np.sqrt(d)
    i[copies] = (3.0 * v).astype(np.float32)
    i[best] = (3.3 * v).astype(np.float32)
    u[: n_rows // 2] = (u[: n_rows // 2] * 0.05 + v[None, :]).astype(np.float32)
    return u, i, np.sort(copies), np.sort(best)


@pytest.mark.parametrize("k, flags", [(10, "tc"), (24, "tc"), (100, None), (500, None)])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_path1_exact_ties_across_the_cut(lib, k, flags, distance):
    """The narrow (k <= 24) and wide routes on planted exact fp32 ties across the cut: the tied copies must come back in
    ascending id order and be the smallest ids, bit-identical to the exhaustive kernels."""
    from rectools_b200 import Engine

    u, i, copies, best = _tied_copies()
    csr = synth_viewed_csr(len(u), len(i), 20, seed=14)
    eng = Engine(i, cosine=distance == "cosine")
    try:
        got = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, flags=lib.Q_FORCE_TC if flags else 0)
        st = dict(eng.last_stats)
        name = f"exact ties {distance} k={k} [{_stats(st)}]"
        assert st["path"] == 1, name
        check_topk(got, u, i, k, cosine=distance == "cosine", filter_csr=csr, name=name)
        half = len(u) // 2
        # the cut falls inside the tied group: its smallest ids (DOT: after the 5 better objects, unless viewed)
        tied = copies if distance == "dot" else np.union1d(copies, best)
        assert np.isin(got[0][:half], np.union1d(copies, best)).all() and np.isin(got[0][:half, 5:], tied).all(), name
        ref = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, flags=lib.Q_FORCE_EXACT)
        assert eng.last_stats["path"] == (0 if k <= 128 else 3)
        _same(got, ref, name)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ path 1, wide, k > 128
@pytest.mark.parametrize("k, env", [(25, {}), (100, {}), (128, {}), (60, {"B200_WIDE": "0"}), (129, {}), (500, {}),
                                    (1000, {}), (200, {"B200_WIDE_T": "201"})])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_path1_wide_and_multipass(lib, monkeypatch, data, k, env, distance):
    from rectools_b200 import Engine

    for key, v in env.items():
        monkeypatch.setenv(key, v)
    u, i, csr = data
    eng = Engine(i, cosine=distance == "cosine")
    try:
        got = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices)
        st = dict(eng.last_stats)
        name = f"{distance} k={k} {env} [{_stats(st)}]"
        assert st["path"] == 1 and st["wide"] == (0 if env.get("B200_WIDE") == "0" else 1), name
        if "B200_WIDE_T" in env:
            assert st["n_fallback_rows"] > 0 and st["n_exact_rows"] == st["n_fallback_rows"], name
        check_topk(got, u, i, k, cosine=distance == "cosine", filter_csr=csr, name=name)
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ path 0
@pytest.mark.parametrize("k", [31, 32, 33, 65])
def test_path0_exhaustive(lib, data, k):
    from rectools_b200 import Engine

    u, i, csr = data
    eng = Engine(i, cosine=k == 33)
    try:
        got = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, flags=lib.Q_FORCE_EXACT)
        st = dict(eng.last_stats)
        assert st["path"] == 0, st
        check_topk(got, u, i, k, cosine=k == 33, filter_csr=csr, name=f"path 0 k={k}")
        one = eng.topk(k, subjects=u[7:8], indptr=csr[7].indptr, indices=csr[7].indices, flags=lib.Q_FORCE_EXACT)
        check_topk(one, u[7:8], i, k, cosine=k == 33, filter_csr=csr[7], name=f"path 0 k={k}, one row")
        _same(one, tuple(a[7:8] for a in got), f"path 0 k={k}: one row against the batch")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ path 3
def test_path3_passes_and_radix(lib, monkeypatch, data):
    from rectools_b200 import Engine

    u, i, csr = data
    rows = np.arange(0, len(u), 8)
    sub, f = u[rows], csr[rows]
    eng = Engine(i, cosine=True)
    try:
        for k, flags in ((129, lib.Q_FORCE_EXACT), (1024, lib.Q_FORCE_EXACT), (1025, 0), (None, 0)):
            kk = len(i) if k is None else k
            got = eng.topk(kk, subjects=sub if k else sub[:8], indptr=f.indptr if k else f[:8].indptr,
                           indices=f.indices if k else f[:8].indices, flags=flags)
            st = dict(eng.last_stats)
            assert st["path"] == 3, st
            check_topk(got, sub if k else sub[:8], i, kk, cosine=True, filter_csr=f if k else f[:8], name=f"path 3 k={k}")
        res = {}
        for sel in ("0", "2"):
            monkeypatch.setenv("B200_SELECT", sel)
            res[sel] = eng.topk(1025, subjects=sub, indptr=f.indptr, indices=f.indices)
            assert eng.last_stats["path"] == 3
        _same(res["0"], res["2"], "path 3 k=1025: the passes against the radix selection")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ path 2
@pytest.mark.parametrize("k", [10, 200, 1025])
def test_path2_sparse_subjects_with_duplicate_columns(lib, k):
    """CSR subject rows whose columns repeat (kept as separate terms), DOT."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(k)
    n_rows, n_obj, d = 512, 30_000, 96
    i = (rng.standard_normal((n_obj, d)) / np.sqrt(d)).astype(np.float32)
    nnz = rng.integers(1, 60, n_rows)
    cols = [rng.integers(0, d, m) for m in nnz]  # duplicates likely
    indptr = np.concatenate([[0], np.cumsum(nnz)]).astype(np.int64)
    sp = sparse.csr_matrix((rng.standard_normal(int(nnz.sum())).astype(np.float32), np.concatenate(cols), indptr),
                           shape=(n_rows, d))
    assert not sp.has_canonical_format
    csr = synth_viewed_csr(n_rows, n_obj, 30, seed=k + 1)
    eng = Engine(i, cosine=False)
    try:
        got = eng.topk(k, sparse_subjects=sp, indptr=csr.indptr, indices=csr.indices)
        assert eng.last_stats["path"] == 2, eng.last_stats
        check_topk(got, sp, i, k, filter_csr=csr, name=f"path 2 k={k}")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ 16-bit
def test_16bit_objects_and_subjects(lib, torch, data):
    """fp16 host objects and bf16 device objects kept at 16 bits; fp16 and bf16 subject device buffers (C ABI)."""
    from rectools_b200 import Engine

    u, i, csr = data
    dev = torch.device("cuda:0")
    i16 = i.astype(np.float16)
    eng = Engine(i16, cosine=True, objects_dtype=lib.DT_F16, keep_16bit=True)
    try:
        for k, flags in ((10, lib.Q_FORCE_TC), (100, 0), (10, lib.Q_FORCE_EXACT)):
            got = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, flags=flags)
            check_topk(got, u, i16, k, cosine=True, filter_csr=csr, name=f"fp16 host objects k={k} [{_stats(eng.last_stats)}]")
    finally:
        eng.close()
    tb = torch.from_numpy(i).to(dev).to(torch.bfloat16).contiguous()
    hb = tb.cpu()
    torch.cuda.synchronize()
    eng = Engine(None, cosine=False, keep_16bit=True, objects_device_ptr=tb.data_ptr(), shape=tuple(tb.shape), objects_dtype=lib.DT_BF16)
    try:
        d_ptr = torch.from_numpy(csr.indptr.astype(np.int64)).to(dev)
        d_idx = torch.from_numpy(csr.indices.astype(np.int32)).to(dev)
        for kind, tdt, dt in (("f16", torch.float16, lib.DT_F16), ("bf16", torch.bfloat16, lib.DT_BF16)):
            rows = torch.from_numpy(u).to(tdt)
            d_rows = rows.to(dev).contiguous()
            for k, fl in ((10, lib.Q_FORCE_TC), (300, 0), (32, lib.Q_FORCE_EXACT)):
                n = len(u)
                out = (torch.empty((n, k), dtype=torch.int32, device=dev), torch.empty((n, k), dtype=torch.float32, device=dev),
                       torch.empty((n,), dtype=torch.int32, device=dev))
                st = eng.topk_ptrs(n, k, *(o.data_ptr() for o in out), lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE | fl,
                                   subjects=d_rows.data_ptr(), indptr=d_ptr.data_ptr(), indices=d_idx.data_ptr(), subject_dtype=dt)
                torch.cuda.synchronize()
                got = tuple(o.cpu().numpy() for o in out)
                check_topk(got, rows, hb, k, filter_csr=csr, name=f"bf16 device objects, {kind} device subjects k={k} [{_stats(st)}]")
    finally:
        eng.close()
        del tb


# ------------------------------------------------------------------------------------------------ the pipeline
def test_host_chunks_patch_and_device_inputs(lib, torch, monkeypatch):
    """Host inputs in row chunks of 256: rows re-ranked by the fallback come back in the patch copy; the same call with
    device inputs and outputs is bit-identical."""
    from rectools_b200 import Engine

    u, i = _near_ties(n_rows=1500, seed=11)
    csr = synth_viewed_csr(len(u), len(i), 20, seed=12)
    eng = Engine(i, cosine=False)
    try:
        monkeypatch.setenv("B200_CHUNK_ROWS", "256")
        got = eng.topk(10, subjects=u, indptr=csr.indptr, indices=csr.indices, flags=lib.Q_FORCE_TC)
        st = dict(eng.last_stats)
        monkeypatch.delenv("B200_CHUNK_ROWS")
        assert st["path"] == 1 and st["n_fallback_rows"] > 0, st
        check_topk(got, u, i, 10, filter_csr=csr, name=f"host chunks of 256 [{_stats(st)}]")
        dev = torch.device("cuda:0")
        d_u = torch.from_numpy(u).to(dev)
        d_ptr = torch.from_numpy(csr.indptr.astype(np.int64)).to(dev)
        d_idx = torch.from_numpy(csr.indices.astype(np.int32)).to(dev)
        n = len(u)
        out = (torch.empty((n, 10), dtype=torch.int32, device=dev), torch.empty((n, 10), dtype=torch.float32, device=dev),
               torch.empty((n,), dtype=torch.int32, device=dev))
        eng.topk_ptrs(n, 10, *(o.data_ptr() for o in out), lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE | lib.Q_FORCE_TC,
                      subjects=d_u.data_ptr(), indptr=d_ptr.data_ptr(), indices=d_idx.data_ptr())
        torch.cuda.synchronize()
        _same(tuple(o.cpu().numpy() for o in out), got, "device inputs against host chunks")
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ above the engine
def test_engine_group_and_sharded_merge(lib, torch, rb):
    """A [0, 0] engine group behind `B200Ranker` (bit-identical to one engine), and the item-sharded exchange on one GPU:
    three shard engines, their packed lists merged without and with the global certificate (shared thresholds); the
    rows the certificate rejects are re-ranked without sharing and merged again, as `ShardedB200Ranker` does."""
    from rectools_b200.sharded import EngineShard, Packed, shard_bounds

    u, i = _near_ties(n_rows=2000, n_obj=30_000, seed=21)
    csr = synth_viewed_csr(len(u), len(i), 30, seed=22)
    sids = np.arange(len(u))
    one = rb.B200Ranker("cosine", u, i)
    grp = rb.B200Ranker("cosine", u, i, device=[0, 0])
    for k in (10, 100):
        a = one.rank_padded(sids, k, csr)[1:]
        b = grp.rank_padded(sids, k, csr)[1:]
        _same(a, b, f"group k={k}")
        check_topk(b, u, i, k, cosine=True, filter_csr=csr, name=f"[0, 0] group k={k} [{_stats(grp.last_stats)}]")
    del one, grp
    k, shards = 10, 3
    dev = torch.device("cuda:0")
    d_u = torch.from_numpy(u).to(dev)
    d_ptr = torch.from_numpy(csr.indptr.astype(np.int64)).to(dev)
    d_idx = torch.from_numpy(csr.indices.astype(np.int32)).to(dev)
    n = len(u)
    engines = [EngineShard(i[lo:hi], False, lo, 0, "auto") for lo, hi in shard_bounds(len(i), shards)]

    def shard_pass(rows, epoch):
        """Every shard ranks `rows` into its packed list (with shared thresholds: no local verdict); gathered buffers."""
        r = torch.from_numpy(np.ascontiguousarray(rows)).to(dev)
        sub = csr[rows]
        su, sp = d_u[r].contiguous(), torch.from_numpy(sub.indptr.astype(np.int64)).to(dev)
        si = torch.from_numpy(sub.indices.astype(np.int32)).to(dev)
        bufs = []
        for eng in engines:
            pk = Packed(torch, len(rows), k, dev)
            eng.local_topk(len(rows), k, pk, shared_epoch=epoch, subjects=su.data_ptr(), indptr=sp.data_ptr(),
                           indices=si.data_ptr(), flags=lib.Q_INPUTS_ON_DEVICE | lib.Q_FORCE_TC)
            bufs.append(pk.buf)
        return torch.cat(bufs)

    try:
        for certified in (False, True):
            o_ids, o_sc, o_cnt, fail_rows, fail_count = engines[0].merge(shard_pass(np.arange(n), 7 if certified else 0),
                                                                          shards, n, k, certified=certified)
            torch.cuda.synchronize()
            got = [o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy()]
            if certified:
                # the rows the global certificate rejects are re-ranked without sharing and merged again, as
                # `ShardedB200Ranker` does; every row is then checked
                n_fail = int(fail_count.item())
                bad = np.sort(fail_rows[:n_fail].cpu().numpy().astype(np.int64))
                print(f"certified merge: {n_fail} of {n} rows rejected")
                assert 0 < n_fail < n
                ok = np.setdiff1d(np.arange(n), bad)
                check_topk(tuple(a[ok] for a in got), u[ok], i, k, filter_csr=csr[ok], name="sharded merge, certified rows")
                r_ids, r_sc, r_cnt, _, _ = engines[0].merge(shard_pass(bad, 0), shards, n_fail, k, certified=False)
                torch.cuda.synchronize()
                for a, v in zip(got, (r_ids, r_sc, r_cnt)):
                    a[bad] = v.cpu().numpy()
            check_topk(tuple(got), u, i, k, filter_csr=csr, name=f"sharded merge certified={certified}, every row")
    finally:
        for eng in engines:
            eng.engine.close()


# ------------------------------------------------------------------------------------------------ EUCLIDEAN, COSINE post-scaling
@pytest.mark.parametrize("d", [127, 128])
def test_euclidean_on_the_tensor_cores(lib, rb, d):
    """d = 127 is augmented to 128 (d_pad 128), d = 128 to 129 (d_pad 192).  The checker runs on the augmented DOT
    problem; `rank()`'s distances are `sqrt(max(dots - s, 0))` of the engine scores, bit for bit."""
    from rectools_b200.ranker import prepare_factors

    u, i = synth_factors(1024, 30_000, d, seed=d)
    csr = synth_viewed_csr(len(u), len(i), 40, seed=d + 1)
    sids = np.arange(len(u))
    ranker = rb.B200Ranker("euclidean", u, i)
    assert ranker.engine.info()["d_pad"] == (128 if d == 127 else 192)
    su, si, _, dots = prepare_factors(ranker.distance, u, i)
    # the augmentation itself, independently: subjects [-1, 2u] and objects [|i|^2, i], the norm column an fp32 sum of
    # squares (within d fp32 roundings of the fp64 one); augmented dots are then 2 u.i - |i|^2 up to that column's error
    np.testing.assert_array_equal(su, np.hstack([-np.ones((len(u), 1), np.float32), 2 * u]))
    np.testing.assert_array_equal(si[:, 1:], i)
    sq = np.einsum("ij,ij->i", widen64(i), widen64(i))
    assert (np.abs(si[:, 0] - sq) <= 1e-5 * sq).all()
    aug = widen64(su[:64]) @ widen64(si).T
    ref = 2.0 * widen64(u[:64]) @ widen64(i).T - sq[None, :]
    assert (np.abs(aug - ref) <= 1e-5 * sq[None, :] + 1e-12).all()
    for k in (10, 100):
        sid, ids, sc, cnt = ranker.rank_padded(sids, k, csr, flags=lib.Q_FORCE_TC if k <= 24 else 0)
        st = dict(ranker.last_stats)
        assert st["path"] == 1, st
        check_topk((ids, sc, cnt), su, si, k, filter_csr=csr, name=f"euclidean d={d} k={k} [{_stats(st)}]")
        _, fid, fsc = ranker.rank(sids, k, csr)
        valid = np.arange(ids.shape[1])[None, :] < cnt[:, None]
        np.testing.assert_array_equal(fid, ids[valid])
        exp = np.sqrt(np.maximum(dots[np.repeat(sids, cnt)] - sc[valid], 0)).astype(np.float32)
        np.testing.assert_array_equal(fsc.view(np.int32), exp.view(np.int32))


def test_cosine_subject_norms_host_and_device(lib, rb, torch):
    """COSINE `rank()` divides the engine scores by `subjects_norms`: fp32 norms of fp64 sums, inside the norm interval,
    the same from host arrays and from device tensors, and the division bit for bit."""
    u, i = synth_factors(1024, 30_000, 64, seed=31)
    u[5] = 0.0  # a zero subject: norm 1e-10
    csr = synth_viewed_csr(len(u), len(i), 40, seed=32)
    sids = np.arange(len(u))
    host = rb.B200Ranker("cosine", u, i)
    devr = rb.B200Ranker("cosine", torch.from_numpy(u).cuda(), torch.from_numpy(i).cuda())
    n_lo, n_hi = norm_interval(widen64(u))
    for nm in (host.subjects_norms, devr.subjects_norms):
        assert ((nm >= n_lo) & (nm <= n_hi)).all()
    exact = n_lo == n_hi
    np.testing.assert_array_equal(host.subjects_norms[exact].view(np.int32), devr.subjects_norms[exact].view(np.int32))
    for r in (host, devr):
        sid, ids, sc, cnt = r.rank_padded(sids, 20, csr)
        check_topk((ids, sc, cnt), u, i, 20, cosine=True, filter_csr=csr, name=f"cosine {'device' if r is devr else 'host'}")
        _, fid, fsc = r.rank(sids, 20, csr)
        valid = np.arange(ids.shape[1])[None, :] < cnt[:, None]
        np.testing.assert_array_equal(fid, ids[valid])
        exp = (sc[valid] / r.subjects_norms[np.repeat(sids, cnt)]).astype(np.float32)
        np.testing.assert_array_equal(fsc.view(np.int32), exp.view(np.int32))
    del host, devr

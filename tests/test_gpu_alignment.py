"""GPU: every buffer the engine reads in place, at every offset a tensor view can have.

A device matrix handed to `b200_rank_create_ex` is the engine's master copy for its whole life, and the per-call inputs
and outputs of `b200_rank_topk` are read and written where the caller put them.  None of them is promised to start on a
16-byte boundary: `buf[1:1 + n * d].view(n, d)` is a contiguous tensor 4 bytes past an aligned address, and
`.contiguous()` returns it as it is.  Every case below builds the same call twice -- once over fresh (256-byte aligned)
allocations, once over views that start 1, 2, 3 or 4 elements into a larger allocation -- and the two must return the
same full padded arrays (ids, score bits, counts, unfilled slots).  Sampled rows are checked against the fp64 oracle.

Catalogues are integer-valued (tests/exact_cases.py), exact in fp16 and bf16, so no comparison needs a tolerance; every
call asserts the path it took.  d = 64 has rows that start on 16 bytes only when the matrix does; d = 12 keeps the fp32
rows on 16-byte steps (d % 4 = 0) but not the 16-bit ones; d = 65 puts every other row anywhere."""
import numpy as np
import pytest
from scipy import sparse

from tests import exact_cases as ec

pytestmark = pytest.mark.gpu

N_OBJ, N_ROWS = 20_000, 300
GUARD = 8  # cells before and after every output view that must stay untouched


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def dev(torch):
    return torch.device("cuda:0")


def offset_view(torch, values, elem_off, fill=0):
    """A contiguous device tensor equal to `values` (a device tensor) that starts `elem_off` elements past a fresh
    allocation; the cells around it hold `fill`."""
    n = values.numel()
    buf = torch.full((elem_off + n + GUARD,), fill, dtype=values.dtype, device=values.device)
    assert buf.data_ptr() % 256 == 0
    view = buf[elem_off : elem_off + n].view(values.shape)
    view.copy_(values)
    assert view.is_contiguous() and view.data_ptr() == buf.data_ptr() + elem_off * values.element_size()
    assert view.data_ptr() % 16 == (elem_off * values.element_size()) % 16
    return view


def _same(got, exp, name, zero_sign=True):
    """Full padded arrays; scores bit for bit (`zero_sign=False`: zeros of either sign compare equal, as the fp64
    oracle does not define the sign of an exact zero sum)."""
    ids, sc, cnt = (np.asarray(a) for a in got)
    eids, esc, ecnt = (np.asarray(a) for a in exp)
    assert ids.shape == eids.shape, f"{name}: shape {ids.shape} vs {eids.shape}"
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, eids, err_msg=f"{name}: ids")
    bits = (lambda a: a.astype(np.float32).view(np.int32)) if zero_sign else (
        lambda a: np.where(a == 0, np.float32(0), a).astype(np.float32).view(np.int32))
    np.testing.assert_array_equal(bits(sc), bits(esc), err_msg=f"{name}: score bits")


def _sample_oracle(got, distance, subjects, objects, k, filt=None, wl=None, n=6, name=""):
    rows = np.unique(np.linspace(0, len(subjects) - 1, n).astype(int))
    f = None if filt is None else filt[rows]
    exp = ec.expected_padded(distance, subjects[rows], objects, np.arange(len(rows)), k, f, wl)
    _same(tuple(np.asarray(a)[rows] for a in got), exp, f"{name} oracle", zero_sign=False)


def _tdtype(torch, name):
    return {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[name]


def _dt(lib, name):
    return {"f32": lib.DT_F32, "f16": lib.DT_F16, "bf16": lib.DT_BF16}[name]


def _engine(lib, t, cosine, keep_16bit, dtype):
    from rectools_b200 import Engine

    return Engine(None, cosine=cosine, objects_device_ptr=t.data_ptr(), shape=tuple(t.shape), objects_dtype=_dt(lib, dtype),
                  keep_16bit=keep_16bit)


# ================================================================================================ objects read in place
# (name, element type, keep at 16 bits, element offsets)
OBJECTS = [("f32", "f32", False, (1, 2, 3)), ("f16", "f16", True, (1, 2, 4)), ("bf16", "bf16", True, (1, 2, 4)),
           ("f16_widened", "f16", False, (1,)), ("bf16_widened", "bf16", False, (1,))]
OBJ_CASES = [(name, dt, keep, off) for name, dt, keep, offs in OBJECTS for off in offs]

# (name, k, flags, (path, wide)); k = None: every object
ROUTES = [("path0", 10, "exact", (0, 0)), ("narrow", 10, "tc", (1, 0)), ("wide", 100, "tc", (1, 1)), ("wide_l", 200, "tc", (1, 1)),
          ("path3", 1025, "", (3, 0)), ("all", None, "", (3, 0))]


def _flags(lib, kind):
    return {"exact": lib.Q_FORCE_EXACT, "tc": lib.Q_FORCE_TC, "": 0}[kind]


@pytest.fixture(scope="module")
def cats():
    """{d: (objects [N_OBJ, d] in [-100, 100], subjects [N_ROWS, d] in [-3, 3], a filter)}."""
    out = {}
    for d in (12, 64, 65):
        rng = np.random.default_rng(300 + d)
        rows = [rng.integers(0, N_OBJ, rng.integers(0, 300)) for _ in range(N_ROWS)]
        rows[1] = np.arange(N_OBJ)  # everything viewed
        out[d] = ec.int_matrix(rng, N_OBJ, d, -100, 100), ec.int_matrix(rng, N_ROWS, d), ec.csr_from_rows(rows, N_OBJ)
    return out


@pytest.mark.parametrize("d", [12, 64, 65])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("case", OBJ_CASES, ids=[f"{c[0]}@{c[3]}" for c in OBJ_CASES])
def test_objects_at_an_offset(lib, torch, dev, cats, case, distance, d):
    """Paths 0, 1 (narrow, wide, k = 200), 3 (k = 1025 and k = None) and 2 (sparse subjects, DOT) over an object matrix
    that starts `off` elements into its allocation, against the engine over the aligned copy."""
    name, dtype, keep, off = case
    objects, subjects, filt = cats[d]
    cosine = distance == "cosine"
    aligned = torch.from_numpy(objects).to(dev).to(_tdtype(torch, dtype)).contiguous()
    moved = offset_view(torch, aligned, off, fill=float("nan"))
    torch.cuda.synchronize()
    ref, eng = _engine(lib, aligned, cosine, keep, dtype), _engine(lib, moved, cosine, keep, dtype)
    try:
        for route, k, fl, path in ROUTES:
            n = 40 if k is None else N_ROWS
            kk = N_OBJ if k is None else k
            tag = f"{name}@{off} d={d} {distance} {route}"
            kw = dict(subjects=subjects[:n], indptr=filt[:n].indptr, indices=filt[:n].indices, flags=_flags(lib, fl))
            exp = ref.topk(kk, **kw)
            got = eng.topk(kk, **kw)
            st = eng.last_stats
            assert (st["path"], st["wide"]) == path, (tag, st)
            _same(got, exp, tag)
            _sample_oracle(got, distance, subjects[:n], objects, kk, filt[:n], name=tag)
        if not cosine:  # path 2: the transposed fp32 copy is built from the offset matrix
            sub = sparse.random(N_ROWS, d, density=0.3, format="csr", random_state=d, dtype=np.float32)
            sub.data[:] = np.random.default_rng(d).integers(-3, 4, sub.nnz)
            for k in (10, 1025):
                got = eng.topk(k, sparse_subjects=sub, indptr=filt.indptr, indices=filt.indices)
                assert eng.last_stats["path"] == 2, eng.last_stats
                _same(got, ref.topk(k, sparse_subjects=sub, indptr=filt.indptr, indices=filt.indices), f"{name}@{off} sparse k={k}")
                _sample_oracle(got, "dot", sub.toarray(), objects, k, filt, name=f"{name}@{off} sparse")
    finally:
        ref.close()
        eng.close()


@pytest.mark.parametrize("case", [c for c in OBJ_CASES if c[0] in ("f32", "f16", "bf16")],
                         ids=[f"{c[0]}@{c[3]}" for c in OBJ_CASES if c[0] in ("f32", "f16", "bf16")])
def test_object_rows_at_an_offset(lib, torch, dev, case):
    """Path 4: the stored rows of a d = n matrix at an offset are the score rows."""
    name, dtype, keep, off = case
    n = 600
    rng = np.random.default_rng(7)
    w = ec.int_matrix(rng, n, n, -100, 100)
    aligned = torch.from_numpy(w).to(dev).to(_tdtype(torch, dtype)).contiguous()
    moved = offset_view(torch, aligned, off, fill=float("nan"))
    torch.cuda.synchronize()
    ref, eng = _engine(lib, aligned, False, keep, dtype), _engine(lib, moved, False, keep, dtype)
    try:
        rows = np.concatenate([np.arange(10), rng.integers(0, n, 100)]).astype(np.int64)
        for k in (10, 100, n):
            got = eng.topk(k, object_rows=rows)
            assert eng.last_stats["path"] == 4, eng.last_stats
            _same(got, ref.topk(k, object_rows=rows), f"{name}@{off} rows k={k}")
            exp = ec.expected_padded("dot", np.eye(n, dtype=np.float32)[rows[:8]], w.T, np.arange(8), k)
            _same(tuple(a[:8] for a in got), exp, f"{name}@{off} rows k={k} oracle", zero_sign=False)
    finally:
        ref.close()
        eng.close()


# ================================================================================================ per-call device buffers
def _guarded_out(torch, dev, n_rows, k_out, off):
    """Output views (ids, scores, counts) that start `off` elements into buffers full of sentinels, and the buffers."""
    bufs = (torch.full((off + n_rows * k_out + GUARD,), 777, dtype=torch.int32, device=dev),
            torch.full((off + n_rows * k_out + GUARD,), 5.0, dtype=torch.float32, device=dev),
            torch.full((off + n_rows + GUARD,), -3, dtype=torch.int32, device=dev))
    views = (bufs[0][off : off + n_rows * k_out].view(n_rows, k_out), bufs[1][off : off + n_rows * k_out].view(n_rows, k_out),
             bufs[2][off : off + n_rows])
    return views, bufs


def _read_guarded(torch, views, bufs, off, name):
    torch.cuda.synchronize()
    for v, b, sentinel in zip(views, bufs, (777, 5.0, -3)):
        h = b.cpu().numpy()
        assert (h[:off] == sentinel).all() and (h[off + v.numel() :] == sentinel).all(), f"{name}: a guard cell was written"
    return tuple(v.cpu().numpy() for v in views)


@pytest.fixture(scope="module")
def call_case():
    """Objects [N_OBJ, 65], subjects [N_ROWS, 65], a filter with everything-viewed rows, a whitelist."""
    rng = np.random.default_rng(77)
    d = 65
    objects, subjects = ec.int_matrix(rng, N_OBJ, d, -100, 100), ec.int_matrix(rng, N_ROWS, d)
    rows = [rng.integers(0, N_OBJ + 50, rng.integers(0, 300)) for _ in range(N_ROWS)]
    rows[0], rows[1] = np.empty(0, np.int64), np.arange(N_OBJ)
    wl = np.sort(rng.choice(N_OBJ, N_OBJ // 2, replace=False)).astype(np.int32)
    return objects, subjects, ec.csr_from_rows(rows, N_OBJ), wl


CALL_ROUTES = [("path0", 32, "exact", (0, 0)), ("narrow", 10, "tc", (1, 0)), ("wide", 100, "tc", (1, 1)),
               ("wide_l", 200, "tc", (1, 1)), ("path3", 1025, "", (3, 0))]


@pytest.mark.parametrize("sub_kind,off", [("f32", 1), ("f32", 3), ("f16", 1), ("f16", 3), ("bf16", 1), ("bf16", 3)])
def test_call_inputs_and_outputs_at_offsets(lib, torch, dev, call_case, sub_kind, off):
    """Subjects (fp32 / fp16 / bf16), filter indptr (int64, offset 1), indices (int32, offset `off`), whitelist (offset
    `off`) and the three outputs (offsets 1, 2, 3) all at odd element offsets, with and without the filter and whitelist,
    on paths 0, 1 and 3; against the same call over fresh buffers.  The guard cells around the outputs stay untouched."""
    from rectools_b200 import Engine

    objects, subjects, filt, wl = call_case
    eng = Engine(objects, cosine=False)
    try:
        tdt = _tdtype(torch, sub_kind)
        s_al = torch.from_numpy(subjects).to(dev).to(tdt).contiguous()
        ip_al = torch.from_numpy(filt.indptr.astype(np.int64)).to(dev)
        ix_al = torch.from_numpy(filt.indices.astype(np.int32)).to(dev)
        wl_al = torch.from_numpy(wl).to(dev)
        s_mv, ip_mv, ix_mv, wl_mv = (offset_view(torch, s_al, off, fill=float("nan")), offset_view(torch, ip_al, 1),
                                     offset_view(torch, ix_al, off), offset_view(torch, wl_al, off))
        torch.cuda.synchronize()
        IN_OUT = lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE
        for filtered in (False, True):
            n_pos = len(wl) if filtered else N_OBJ
            for route, k, fl, path in CALL_ROUTES:
                k_out = min(k, n_pos)
                results = []
                for s, ip, ix, w, o_off in ((s_al, ip_al, ix_al, wl_al, 0), (s_mv, ip_mv, ix_mv, wl_mv, None)):
                    extra = dict(indptr=ip.data_ptr(), indices=ix.data_ptr(), whitelist=w.data_ptr(), n_whitelist=len(wl)) if filtered else {}
                    outs = []
                    for o in ((0,) if o_off == 0 else (1, 2, 3)):
                        views, bufs = _guarded_out(torch, dev, N_ROWS, k_out, o)
                        st = eng.topk_ptrs(N_ROWS, k, *(v.data_ptr() for v in views), IN_OUT | _flags(lib, fl), subjects=s.data_ptr(),
                                           subject_dtype=_dt(lib, sub_kind), **extra)
                        tag = f"{sub_kind}@{off} filtered={filtered} {route} out@{o}"
                        assert (st["path"], st["wide"]) == path, (tag, st)
                        outs.append((tag, _read_guarded(torch, views, bufs, o, tag)))
                    results.append(outs)
                (_, exp), = results[0]
                for tag, got in results[1]:
                    _same(got, exp, tag)
                wide = s_al.float().cpu().numpy()
                _sample_oracle(exp, "dot", wide, objects, k, filt if filtered else None, wl if filtered else None,
                               name=f"{sub_kind} filtered={filtered} {route}")
    finally:
        eng.close()


@pytest.mark.parametrize("off", [1, 3])
def test_resident_device_subjects_and_ids_at_offsets(lib, torch, dev, call_case, off):
    """`set_subjects_device` over a matrix `off` elements into its allocation, gathered through device `subject_ids`
    (int64, offset 1), filter and outputs at offsets too; paths 0, 1 and 3 against the aligned engine."""
    from rectools_b200 import Engine

    objects, subjects, filt, _ = call_case
    rng = np.random.default_rng(off)
    sids = rng.integers(0, N_ROWS, 200).astype(np.int64)
    f = filt[sids]
    s_al = torch.from_numpy(subjects).to(dev)
    id_al = torch.from_numpy(sids).to(dev)
    ip_al = torch.from_numpy(f.indptr.astype(np.int64)).to(dev)
    ix_al = torch.from_numpy(f.indices.astype(np.int32)).to(dev)
    s_mv, id_mv, ip_mv, ix_mv = (offset_view(torch, s_al, off, fill=float("nan")), offset_view(torch, id_al, 1),
                                 offset_view(torch, ip_al, 1), offset_view(torch, ix_al, off))
    torch.cuda.synchronize()
    ref, eng = Engine(objects, cosine=False), Engine(objects, cosine=False)
    try:
        ref.set_subjects_device(s_al.data_ptr(), N_ROWS)
        eng.set_subjects_device(s_mv.data_ptr(), N_ROWS)
        for route, k, fl, path in CALL_ROUTES:
            flags = lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE | _flags(lib, fl)
            got = []
            for e, ids, ip, ix, o in ((ref, id_al, ip_al, ix_al, 0), (eng, id_mv, ip_mv, ix_mv, off)):
                views, bufs = _guarded_out(torch, dev, len(sids), k, o)
                st = e.topk_ptrs(len(sids), k, *(v.data_ptr() for v in views), flags, subject_ids=ids.data_ptr(), indptr=ip.data_ptr(),
                                 indices=ix.data_ptr())
                tag = f"resident@{off} {route}"
                assert (st["path"], st["wide"]) == path, (tag, st)
                got.append(_read_guarded(torch, views, bufs, o, tag))
            _same(got[1], got[0], tag)
            _sample_oracle(got[1], "dot", subjects[sids], objects, k, f, name=tag)
    finally:
        ref.close()
        eng.close()


@pytest.mark.parametrize("off", [1, 3])
def test_sparse_subjects_and_object_rows_at_offsets(lib, torch, dev, call_case, off):
    """Path 2 with `sub_indptr` (int64, offset 1), `sub_indices` / `sub_data` (offset `off`); path 4 with `object_rows`
    (int64, offset 1); outputs at offset `off`."""
    from rectools_b200 import Engine

    objects, _, filt, _ = call_case
    d = objects.shape[1]
    n = 120
    a = sparse.random(n, d, density=0.3, format="csr", random_state=off, dtype=np.float32)
    a.data[:] = np.random.default_rng(off).integers(-3, 4, a.nnz)
    w = ec.int_matrix(np.random.default_rng(5), 500, 500, -100, 100)
    rows = np.random.default_rng(6).integers(0, 500, n).astype(np.int64)
    dense, square = Engine(objects, cosine=False), Engine(w, cosine=False)
    try:
        sp_al = [torch.from_numpy(x).to(dev) for x in (a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data)]
        sp_mv = [offset_view(torch, sp_al[0], 1), offset_view(torch, sp_al[1], off), offset_view(torch, sp_al[2], off, fill=float("nan"))]
        r_al = torch.from_numpy(rows).to(dev)
        r_mv = offset_view(torch, r_al, 1)
        torch.cuda.synchronize()
        flags = lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE
        for k in (10, 1025):
            got = []
            for (ip, ix, x), o in ((sp_al, 0), (sp_mv, off)):
                q = lib.Query()
                q.sub_indptr, q.sub_indices, q.sub_data = ip.data_ptr(), ix.data_ptr(), x.data_ptr()
                q.n_rows, q.k, q.flags = n, k, flags
                views, bufs = _guarded_out(torch, dev, n, k, o)
                q.out_ids, q.out_scores, q.out_counts = (v.data_ptr() for v in views)
                assert dense.topk_raw(q)["path"] == 2, dense.last_stats
                got.append(_read_guarded(torch, views, bufs, o, f"sparse@{off} k={k}"))
            _same(got[1], got[0], f"sparse@{off} k={k}")
            _sample_oracle(got[1], "dot", a.toarray(), objects, k, name=f"sparse@{off} k={k}")
        for k in (10, 500):
            got = []
            for r, o in ((r_al, 0), (r_mv, off)):
                views, bufs = _guarded_out(torch, dev, n, k, o)
                st = square.topk_ptrs(n, k, *(v.data_ptr() for v in views), flags, object_rows=r.data_ptr())
                assert st["path"] == 4, st
                got.append(_read_guarded(torch, views, bufs, o, f"rows@{off} k={k}"))
            _same(got[1], got[0], f"rows@{off} k={k}")
            exp = ec.expected_padded("dot", np.eye(500, dtype=np.float32)[rows], w.T, np.arange(n), k)
            _same(got[1], exp, f"rows@{off} k={k} oracle", zero_sign=False)
    finally:
        dense.close()
        square.close()


# ================================================================================================ public API, groups, merges
@pytest.fixture(scope="module")
def api_case():
    rng = np.random.default_rng(404)
    n, d = 30_000, 64
    return ec.int_matrix(rng, n, d, -100, 100), ec.int_matrix(rng, 500, d)


def _rank_equal(a, b, name):
    for x, y in zip(a, b):
        np.testing.assert_array_equal(np.asarray(x), np.asarray(y), err_msg=name)


@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_rankers_over_offset_tensors(torch, dev, api_case, distance):
    """`B200Ranker` over an fp32 CUDA tensor 1 element into its allocation and `B200TorchRanker` over a bf16 one: each
    ranks what the same class ranks over `.clone()` of the tensor (an aligned copy)."""
    from rectools_b200 import B200Ranker, B200TorchRanker

    objects, users = api_case
    sids = np.arange(len(users))
    csr = ec.csr_from_rows([np.arange(r % 50) for r in range(len(users))], len(objects))
    for cls, dtype in ((B200Ranker, torch.float32), (B200TorchRanker, torch.bfloat16)):
        moved = offset_view(torch, torch.from_numpy(objects).to(dev).to(dtype), 1, fill=float("nan"))
        args = (distance, "cuda:0") if cls is B200TorchRanker else (distance,)
        r_mv = cls(*args, users, moved)
        r_al = cls(*args, users, moved.clone())
        assert r_mv.engine.info()["hbm_bytes"] == r_al.engine.info()["hbm_bytes"]  # both read in place
        for k in (10, 100, 1025):
            _rank_equal(r_mv.rank(sids, k, csr), r_al.rank(sids, k, csr), f"{cls.__name__} {distance} k={k}")
        a = r_mv.rank_padded(sids, 10, csr)
        exp = ec.expected_padded(distance, users, objects, np.arange(8), 10, csr[:8])
        if distance == "dot":
            _same(tuple(x[:8] for x in a[1:]), exp, f"{cls.__name__} oracle", zero_sign=False)
        else:  # COSINE ranker scores are divided by the subject norm as well: compare the ids
            np.testing.assert_array_equal(a[1][:8], exp[0], err_msg=f"{cls.__name__} cosine oracle ids")
        r_mv.engine.close()
        r_al.engine.close()


def test_engine_group_over_an_offset_matrix(lib, torch, dev, api_case, monkeypatch):
    """A group [0, 0] over an fp32 matrix at offset 1 and a bf16 matrix kept at 16 bits at offset 1: bit for bit one
    engine over the aligned copy."""
    from rectools_b200 import EngineGroup

    monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "100")
    objects, users = api_case
    rows = [np.arange(r % 40) for r in range(len(users))]
    filt = ec.csr_from_rows(rows, len(objects))
    for dtype, keep in (("f32", False), ("bf16", True)):
        aligned = torch.from_numpy(objects).to(dev).to(_tdtype(torch, dtype))
        moved = offset_view(torch, aligned, 1, fill=float("nan"))
        torch.cuda.synchronize()
        one = _engine(lib, aligned, False, keep, dtype)
        grp = EngineGroup(None, cosine=False, devices=(0, 0), objects_device_ptr=moved.data_ptr(), shape=tuple(moved.shape),
                          objects_dtype=_dt(lib, dtype), keep_16bit=keep)
        try:
            for k, flags in ((10, 0), (100, 0), (10, lib.Q_FORCE_EXACT), (1025, 0)):  # (groups refuse FORCE_TC)
                kw = dict(subjects=users, indptr=filt.indptr, indices=filt.indices, flags=flags)
                _same(grp.topk(k, **kw), one.topk(k, **kw), f"group {dtype}@1 k={k}")
        finally:
            grp.close()
            one.close()


@pytest.mark.parametrize("certified", [False, True])
def test_merges_read_lists_at_offsets(lib, torch, dev, certified):
    """`b200_rank_merge` / `_merge_certified` over lists, bounds and outputs that start 1 and 3 elements into their
    allocations, against the numpy merge."""
    rng = np.random.default_rng(61 + certified)
    n_lists, n_rows, k = 4, 37, 24
    ids, sc, cnt = ec.merge_case(rng, n_lists, n_rows, k)
    bounds = np.where(rng.random((n_lists, n_rows)) < 0.3, -np.inf, rng.integers(-3, 4, (n_lists, n_rows))).astype(np.float32)
    exp = ec.expected_merge(ids, sc, cnt, k, bounds if certified else None)
    h = lib.load()
    for off in (1, 3):
        ins = [offset_view(torch, torch.from_numpy(np.ascontiguousarray(x)).to(dev), off) for x in (ids, sc, cnt, bounds)]
        views, bufs = _guarded_out(torch, dev, n_rows, k, off)
        fail_rows = offset_view(torch, torch.full((n_rows,), -1, dtype=torch.int32, device=dev), off)
        fail_count = offset_view(torch, torch.zeros((1,), dtype=torch.int32, device=dev), off)
        torch.cuda.synchronize()
        out = [v.data_ptr() for v in views]
        p = [x.data_ptr() for x in ins]
        if certified:
            lib.check(h.b200_rank_merge_certified(0, None, n_lists, n_rows, k, *p, 0, *out, fail_rows.data_ptr(), fail_count.data_ptr()))
        else:
            lib.check(h.b200_rank_merge(0, None, n_lists, n_rows, k, *p[:3], *out))
        got = _read_guarded(torch, views, bufs, off, f"merge@{off}")
        _same(got, exp[:3], f"merge certified={certified} @{off}", zero_sign=False)
        if certified:
            np.testing.assert_array_equal(np.sort(fail_rows.cpu().numpy()[: int(fail_count.item())]), exp[3])


@pytest.fixture(scope="module")
def ref():
    from oracle import stage_reference

    if not stage_reference.available():
        pytest.skip("reference package not staged (oracle/_ref)")
    added = stage_reference.add_to_path()
    import rectools  # noqa: F401

    yield
    stage_reference.remove_from_path(added)


@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_similarity_module_over_offset_item_embs(ref, torch, dev, distance):
    """`make_similarity_module()` with bf16 `item_embs` 1 element into their allocation returns the frame of the same
    module over `.clone()`."""
    from scipy import sparse as sp

    from rectools_b200.integration import make_similarity_module

    n_users, n_tokens, d, k = 1000, 20_001, 64, 10
    g = torch.Generator().manual_seed(19)
    user_embs = torch.randn((n_users, d), generator=g) / d**0.5
    moved = offset_view(torch, (torch.randn((n_tokens, d), generator=g) / d**0.5).to(torch.bfloat16).to(dev), 1, fill=float("nan"))
    user_ids = np.random.default_rng(0).permutation(n_users)[:700]
    rng = np.random.default_rng(1)
    cols = rng.integers(1, n_tokens, size=(len(user_ids), 30))
    ui = sp.csr_matrix((np.ones(cols.size, np.float32), (np.repeat(np.arange(len(user_ids)), 30), cols.reshape(-1))),
                       shape=(len(user_ids), n_tokens))
    ui.sum_duplicates()
    ui.data[:] = 1.0
    whitelist = np.arange(1, n_tokens)
    a = make_similarity_module()(distance=distance)._recommend_u2i(  # pylint: disable=protected-access
        user_embs, moved, user_ids, k, whitelist, ui)
    b = make_similarity_module()(distance=distance)._recommend_u2i(  # pylint: disable=protected-access
        user_embs, moved.clone(), user_ids, k, whitelist, ui)
    _rank_equal(a, b, f"similarity module {distance}")
    assert len(a[1]) == len(user_ids) * k

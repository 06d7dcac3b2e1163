"""GPU: candidate sets from device memory (engine path 5, `b200_rank_topk_candidates_device`,
`B200Ranker.rank_candidates_device`).

Raw lists -- ids in any order, repeats, -1 holes, ids >= n_objects -- go to the device route; the same lists normalised
in numpy (valid, sorted, unique) go to the host route, `Engine.topk_candidates`.  Every comparison is of the full padded
arrays, bit for bit.  A representative subset is also checked row by row against the rounding-interval oracle
(`tests/score_interval.check_topk`) with C_r as a complement filter.  Covered: DOT / COSINE; fp32, fp16 and bf16 objects
(16-bit kept at 16 bits); d = 1, 65, 128, 256; raw rows of 0, 1, k-1, k, S-1, S, S+1 and 50 000 entries; unsorted,
descending, all-repeat, all -1 and all >= n_objects rows; k = 1, 10, 1024, 1025 and k above m; filters overlapping the
lists and fully filtered rows; three and more chunks; a non-zero cand_indptr base; subjects in batch order (fp32 / fp16 /
bf16), fp32 with subject_ids, resident subjects set from the host and from the device; device and host outputs; every
refusal with every output untouched; stream ordering against decoys; element-offset views; the ranker API."""
import ctypes as C

import numpy as np
import pytest
from scipy import sparse

from tests.score_interval import check_topk
from tests.test_gpu_candidate_sets import _complement_filter, _engine

pytestmark = pytest.mark.gpu

S = 12288  # LK_SMEM_PAIRS
SLEEP_CYCLES = 300_000_000


@pytest.fixture(scope="module")
def torch():
    import torch as t

    return t


def _raw_rows(rng, n_obj, lens, kinds=None):
    """One raw list per row: `lens[r]` entries of kind kinds[r] -- "mix" (valid ids with repeats, -1 and >= n_obj
    entries, shuffled), "desc", "repeat", "neg", "high"."""
    rows = []
    for r, n in enumerate(lens):
        kind = kinds[r] if kinds is not None else "mix"
        if kind == "mix":
            x = rng.integers(0, n_obj, n)
            x[rng.random(n) < 0.1] = -1
            x[rng.random(n) < 0.05] = n_obj + rng.integers(0, 1000)
            if n > 4:
                x[: n // 4] = x[n // 4 : 2 * (n // 4)]  # repeats
            rng.shuffle(x)
        elif kind == "desc":
            x = np.sort(rng.choice(n_obj, min(n, n_obj), replace=False))[::-1]
        elif kind == "repeat":
            x = np.full(n, rng.integers(0, n_obj))
        elif kind == "neg":
            x = -rng.integers(1, 1 << 31, n)
        else:
            x = n_obj + rng.integers(0, 1 << 20, n)
        rows.append(np.asarray(x, np.int64).astype(np.int32))
    return rows


def _normalised(rows, n_obj):
    clean = [np.unique(r[(r >= 0) & (r < n_obj)]).astype(np.int32) for r in rows]
    indptr = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(c) for c in clean], out=indptr[1:])
    return indptr, (np.concatenate(clean) if clean else np.empty(0)).astype(np.int32)


def _raw(rows, base=0):
    """(indptr with cand_indptr[0] = base, indices with `base` leading junk entries)"""
    indptr = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(r) for r in rows], out=indptr[1:])
    junk = np.full(base, 7, np.int32)
    return indptr + base, np.concatenate([junk] + list(rows)).astype(np.int32)


def _filter(rng, norm, n_obj, full_rows=()):
    indptr, indices = norm
    rows = []
    for r in range(len(indptr) - 1):
        c = indices[indptr[r] : indptr[r + 1]]
        take = c if r in full_rows else c[rng.random(len(c)) < 0.5]
        rows.append(np.unique(np.concatenate([take, rng.choice(n_obj, 5)])).astype(np.int32))
    f = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(x) for x in rows], out=f[1:])
    return f, np.concatenate(rows).astype(np.int32)


def _cuda(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(torch, out):
    return tuple(t.cpu().numpy() if hasattr(t, "cpu") else t for t in out)


def _same(a, b, what):
    ids_a, sc_a, cnt_a = a
    ids_b, sc_b, cnt_b = b
    np.testing.assert_array_equal(cnt_a, cnt_b, err_msg=f"{what}: counts")
    np.testing.assert_array_equal(ids_a, ids_b, err_msg=f"{what}: ids")
    np.testing.assert_array_equal(np.asarray(sc_a, np.float32).view(np.int32), np.asarray(sc_b, np.float32).view(np.int32),
                                  err_msg=f"{what}: score bits")


def _both(torch, eng, k, rows, n_obj, subjects=None, subject_ids=None, filt=None, base=0, host_subjects=None, host_out=False,
          host_subject_ids=None):
    """(device route, host route on the normalised lists), as numpy."""
    norm = _normalised(rows, n_obj)
    f_ind, f_idx = filt if filt is not None else (None, None)
    hs = host_subjects if host_subjects is not None else (subjects.float().cpu().numpy() if subjects is not None else None)
    hid = host_subject_ids if host_subject_ids is not None else (subject_ids.cpu().numpy() if subject_ids is not None else None)
    exp = eng.topk_candidates(k, *norm, subjects=hs, subject_ids=hid, indptr=f_ind, indices=f_idx)
    raw_ptr, raw_idx = _raw(rows, base)
    k_out = min(k, n_obj)
    out = None
    if host_out:
        n = len(rows)
        out = (np.full((n, k_out), 5, np.int32), np.full((n, k_out), 3.0, np.float32), np.full(n, 9, np.int32))
    got = eng.topk_candidates_device(
        k, _cuda(torch, raw_ptr), _cuda(torch, raw_idx), subjects=subjects, subject_ids=subject_ids,
        indptr=None if f_ind is None else _cuda(torch, f_ind), indices=None if f_idx is None else _cuda(torch, f_idx), out=out,
    )
    assert eng.last_stats["path"] == 5, eng.last_stats
    return _np(torch, got), exp, norm


LENS = [0, 1, 9, 10, 1023, 1024, 1025, S - 1, S, S + 1, 50_000]


@pytest.mark.parametrize("k", [1, 10, 1024, 1025, 60_000])
@pytest.mark.parametrize("cosine", [False, True])
def test_row_lengths_and_k(torch, k, cosine):
    rng = np.random.default_rng(k + cosine)
    n_obj, d = 60_000, 24
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng, _ = _engine(objects, cosine)
    lens = LENS + [50, 50, 50, 50, 50]
    kinds = ["mix"] * len(LENS) + ["desc", "repeat", "neg", "high", "mix"]
    rows = _raw_rows(rng, n_obj, lens, kinds)
    subjects = _cuda(torch, rng.standard_normal((len(rows), d)).astype(np.float32))
    got, exp, norm = _both(torch, eng, k, rows, n_obj, subjects=subjects)
    _same(got, exp, f"k={k}")
    assert got[2][len(LENS) + 1] == min(1, k) and got[2][len(LENS) + 2] == 0 and got[2][len(LENS) + 3] == 0
    filt = _filter(rng, norm, n_obj, full_rows=(3, 8))
    got, exp, _ = _both(torch, eng, k, rows, n_obj, subjects=subjects, filt=filt, base=5)
    _same(got, exp, f"k={k} filter base=5")
    assert got[2][3] == 0 and got[2][8] == 0
    if k in (10, 1025):
        comp = _complement_filter(n_obj, *norm, *filt)
        check_topk(got, subjects.cpu().numpy(), objects, k, cosine=cosine, filter_csr=comp, name=f"k={k}", max_ambiguous=1e-3)


@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("d", [1, 65, 128, 256])
@pytest.mark.parametrize("cosine", [False, True])
def test_object_types_and_widths(torch, dtype, d, cosine):
    rng = np.random.default_rng(d)
    n_obj = 20_000
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng, obj_seen = _engine(objects, cosine, dtype)
    rows = _raw_rows(rng, n_obj, rng.integers(0, 3000, 40))
    subjects = _cuda(torch, rng.standard_normal((40, d)).astype(np.float32))
    norm = _normalised(rows, n_obj)
    filt = _filter(rng, norm, n_obj, full_rows=(5,))
    for k in (10, 1025):
        got, exp, _ = _both(torch, eng, k, rows, n_obj, subjects=subjects, filt=filt)
        _same(got, exp, f"{dtype} d={d} k={k}")
        if d in (1, 128):
            comp = _complement_filter(n_obj, *norm, *filt)
            check_topk(got, subjects.cpu().numpy(), obj_seen, k, cosine=cosine, filter_csr=comp, name=f"{dtype} d={d} k={k}",
                       max_ambiguous=1e-3)


@pytest.mark.parametrize("host_out", [False, True])
def test_subject_sources_and_outputs(torch, host_out):
    rng = np.random.default_rng(11 + host_out)
    n_obj, d, n_sub = 30_000, 64, 500
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng, _ = _engine(objects, False)
    rows = _raw_rows(rng, n_obj, rng.integers(0, 2000, 64))
    norm = _normalised(rows, n_obj)
    filt = _filter(rng, norm, n_obj, full_rows=(2,))
    k = 100
    batch = rng.standard_normal((64, d)).astype(np.float32)
    exp = eng.topk_candidates(k, *norm, subjects=batch, indptr=filt[0], indices=filt[1])
    for tdt in (torch.float32, torch.float16, torch.bfloat16):  # batch order, 16-bit widened on the device
        sub = _cuda(torch, batch).to(tdt)
        got, ref, _ = _both(torch, eng, k, rows, n_obj, subjects=sub, filt=filt, host_out=host_out)
        _same(got, ref, f"batch {tdt}")
        if tdt == torch.float32:
            _same(got, exp, "batch fp32")
    table = rng.standard_normal((n_sub, d)).astype(np.float32)
    sids = rng.integers(0, n_sub, 64).astype(np.int64)
    got, ref, _ = _both(torch, eng, k, rows, n_obj, subjects=_cuda(torch, table), subject_ids=_cuda(torch, sids), filt=filt,
                        host_out=host_out, host_subjects=table)
    _same(got, ref, "explicit matrix + subject_ids")
    eng.set_subjects(table)  # resident, from the host
    got, ref, _ = _both(torch, eng, k, rows, n_obj, subject_ids=_cuda(torch, sids), filt=filt, host_out=host_out)
    _same(got, ref, "resident (host)")
    dev_table = _cuda(torch, table)
    eng.set_subjects_device(dev_table.data_ptr(), n_sub)  # resident, from the device: the host route refuses it
    raw_ptr, raw_idx = _raw(rows)
    got = eng.topk_candidates_device(k, _cuda(torch, raw_ptr), _cuda(torch, raw_idx), subject_ids=_cuda(torch, sids),
                                     indptr=_cuda(torch, filt[0]), indices=_cuda(torch, filt[1]))
    _same(_np(torch, got), ref, "resident (device)")


def test_three_and_more_chunks(torch, monkeypatch):
    rng = np.random.default_rng(3)
    n_obj, d = 40_000, 32
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng, _ = _engine(objects, True)
    lens = rng.integers(0, 600, 1000)
    lens[700] = 20_000  # a row that sorts in global scratch, in a later chunk
    rows = _raw_rows(rng, n_obj, lens)
    subjects = _cuda(torch, rng.standard_normal((1000, d)).astype(np.float32))
    norm = _normalised(rows, n_obj)
    filt = _filter(rng, norm, n_obj)
    whole, _, _ = _both(torch, eng, 50, rows, n_obj, subjects=subjects, filt=filt, base=3)
    assert eng.last_stats["n_chunks"] == 1
    monkeypatch.setenv("B200_CHUNK_ROWS", "256")
    for k in (50, 20_000):
        got, exp, _ = _both(torch, eng, k, rows, n_obj, subjects=subjects, filt=filt, base=3)
        assert eng.last_stats["n_chunks"] == 4, eng.last_stats
        _same(got, exp, f"chunks k={k}")
        if k == 50:
            _same(got, whole, "chunked = whole")
    for host_out in (False, True):
        got, exp, _ = _both(torch, eng, 50, rows, n_obj, subjects=subjects, filt=filt, host_out=host_out)
        _same(got, exp, f"chunks host_out={host_out}")


# --------------------------------------------------------------------------------------------------------------- refusals
def _guards(torch, n, k):
    return (torch.full((n, k), 777, dtype=torch.int32, device="cuda"), torch.full((n, k), 5.0, device="cuda"),
            torch.full((n,), -3, dtype=torch.int32, device="cuda"))


def _untouched(torch, out):
    torch.cuda.synchronize()
    assert bool((out[0] == 777).all()) and bool((out[1] == 5.0).all()) and bool((out[2] == -3).all())


def test_refusals_leave_outputs_untouched(torch):
    from rectools_b200 import _lib
    from rectools_b200.ranker import Engine

    rng = np.random.default_rng(4)
    n_obj, d, n = 1000, 16, 8
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng = Engine(objects, cosine=False)
    lib = _lib.load()
    sub = _cuda(torch, rng.standard_normal((n, d)).astype(np.float32))
    ptr = _cuda(torch, np.arange(n + 1, dtype=np.int64) * 3)
    idx = _cuda(torch, rng.integers(0, n_obj, 3 * n).astype(np.int32))
    wl = _cuda(torch, np.arange(10, dtype=np.int32))

    def call(code, words, flags=_lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE, cand_ptr=None, engine=eng, k=10, **fields):
        out = _guards(torch, n, min(k, engine.n_objects))
        q = _lib.Query()
        q.subjects, q.n_rows, q.k, q.flags = sub.data_ptr(), n, k, flags
        q.out_ids, q.out_scores, q.out_counts = (t.data_ptr() for t in out)
        for name, v in fields.items():
            setattr(q, name, v)
        rc = lib.b200_rank_topk_candidates_device(engine._h, C.byref(q), ptr.data_ptr() if cand_ptr is None else cand_ptr,  # pylint: disable=protected-access
                                                  idx.data_ptr(), None)
        msg = lib.b200_rank_last_error().decode()
        assert rc == code and words in msg, (rc, msg)
        _untouched(torch, out)

    I, U, M = _lib.E_INVALID, _lib.E_UNSUPPORTED, _lib.E_NOMEM
    call(I, "B200_Q_INPUTS_ON_DEVICE", flags=_lib.Q_OUTPUTS_ON_DEVICE)
    call(I, "b200_rank_topk_candidates", flags=_lib.Q_OUTPUTS_ON_DEVICE)
    sp = _cuda(torch, np.zeros(n + 1, np.int64))
    call(U, "sub_", sub_indptr=sp.data_ptr(), subjects=None)
    call(U, "object_rows", object_rows=sp.data_ptr(), subjects=None)
    call(U, "whitelist", whitelist=wl.data_ptr(), n_whitelist=10)
    call(U, "SHARED_THRESHOLDS", flags=_lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE | _lib.Q_SHARED_THRESHOLDS)
    call(U, "FORCE_TC", flags=_lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE | _lib.Q_FORCE_TC)
    call(I, "cand_indptr is NULL", cand_ptr=0)
    bad = _cuda(torch, np.array([-1, 2, 4, 6, 8, 10, 12, 14, 16], np.int64))
    call(I, "cand_indptr[0] < 0", cand_ptr=bad.data_ptr())
    bad = _cuda(torch, np.array([0, 3, 6, 5, 12, 15, 18, 21, 24], np.int64))
    call(I, "not monotone at row 2", cand_ptr=bad.data_ptr())
    huge = _cuda(torch, np.r_[0, np.full(n, 200_000_000)].astype(np.int64))  # refused before a single entry is read
    call(M, "row 0", cand_ptr=huge.data_ptr())
    call(I, "k must be positive", k=0)
    call(I, "16-bit subjects", subject_dtype=_lib.DT_F16, subject_ids=sp.data_ptr(), n_subjects_total=n)
    offset = Engine(objects, cosine=False)
    lib.b200_rank_set_id_offset(offset._h, 5)  # pylint: disable=protected-access
    call(U, "id offset", engine=offset)
    wide = Engine(np.ones((4, 49153), np.float32), cosine=False)
    call(U, "d = 49153", engine=wide, subjects=None, subject_ids=sp.data_ptr())


# --------------------------------------------------------------------------------------------------------------- ordering
def _behind_sleep(torch, stream, writes):
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SLEEP_CYCLES)  # pylint: disable=protected-access
        for dst, src in writes:
            dst.copy_(src)
        ev = torch.cuda.Event()
        ev.record(stream)
    assert not ev.query(), "the sleep is too short to test anything"


@pytest.mark.parametrize("producer", ["side", "legacy"])
def test_inputs_wait_for_the_producer_stream(torch, producer):
    from rectools_b200.ranker import Engine

    rng = np.random.default_rng(21)
    n_obj, d, n, m, k = 5000, 32, 64, 300, 20
    objects = rng.integers(-8, 9, (n_obj, d)).astype(np.float32)
    eng = Engine(objects, cosine=False)
    table = {s: rng.integers(-8, 9, (200, d)).astype(np.float32) for s in ("real", "decoy")}
    sids = {s: rng.integers(0, 200, n).astype(np.int64) for s in ("real", "decoy")}
    cands = {s: rng.integers(-1, n_obj, (n, m)).astype(np.int32) for s in ("real", "decoy")}
    nnz = 2 * n
    filt = {s: (np.arange(n + 1, dtype=np.int64) * 2, np.sort(rng.integers(0, n_obj, (n, 2)), axis=1).reshape(-1).astype(np.int32))
            for s in ("real", "decoy")}
    assert len(filt["real"][1]) == nnz
    indptr = np.arange(n + 1, dtype=np.int64) * m

    def expected(s):
        rows = list(cands[s])
        return eng.topk_candidates(k, *_normalised(rows, n_obj), subjects=table[s], subject_ids=sids[s], indptr=filt[s][0],
                                   indices=filt[s][1])

    exp, exp_decoy = expected("real"), expected("decoy")
    assert not np.array_equal(exp[0], exp_decoy[0])
    names = ("table", "sids", "cands", "f_indices")
    real = dict(zip(names, (table["real"], sids["real"], cands["real"], filt["real"][1])))
    decoy = dict(zip(names, (table["decoy"], sids["decoy"], cands["decoy"], filt["decoy"][1])))
    bufs = {name: (_cuda(torch, decoy[name]), _cuda(torch, real[name])) for name in names}
    stream = torch.cuda.Stream() if producer == "side" else torch.cuda.default_stream()
    out = _guards(torch, n, k)
    _behind_sleep(torch, stream, list(bufs.values()))
    eng.topk_candidates_device(
        k, _cuda(torch, indptr), bufs["cands"][0].reshape(-1), subjects=bufs["table"][0], subject_ids=bufs["sids"][0],
        indptr=_cuda(torch, filt["real"][0]), indices=bufs["f_indices"][0], out=out,
        stream=stream.cuda_stream if producer == "side" else 0,
    )
    torch.cuda.synchronize()
    _same(_np(torch, out), exp, f"producer {producer}")


def test_device_outputs_are_not_overwritten_before_the_caller_read_them(torch):
    from rectools_b200.ranker import Engine

    rng = np.random.default_rng(9)
    n_obj, d, n, m, k = 5000, 32, 64, 200, 20
    objects = rng.integers(-8, 9, (n_obj, d)).astype(np.float32)
    eng = Engine(objects, cosine=False)
    a, b = (_cuda(torch, rng.integers(-8, 9, (n, d)).astype(np.float32)) for _ in range(2))
    cands = _cuda(torch, rng.integers(0, n_obj, (n, m)).astype(np.int32)).reshape(-1)
    indptr = _cuda(torch, np.arange(n + 1, dtype=np.int64) * m)
    s = torch.cuda.Stream()
    x = _guards(torch, n, k)
    eng.topk_candidates_device(k, indptr, cands, subjects=a, out=x, stream=s.cuda_stream)
    exp_a = _np(torch, eng.topk_candidates_device(k, indptr, cands, subjects=a))
    exp_b = _np(torch, eng.topk_candidates_device(k, indptr, cands, subjects=b))
    assert not np.array_equal(exp_a[0], exp_b[0])
    y = tuple(torch.empty_like(t) for t in x)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)  # pylint: disable=protected-access
        for dst, src in zip(y, x):
            dst.copy_(src)
        ev = torch.cuda.Event()
        ev.record(s)
    assert not ev.query(), "the sleep is too short to test anything"
    eng.topk_candidates_device(k, indptr, cands, subjects=b, out=x, stream=s.cuda_stream)
    torch.cuda.synchronize()
    _same(_np(torch, y), exp_a, "Y: call 1")
    _same(_np(torch, x), exp_b, "X: call 2")


# -------------------------------------------------------------------------------------------------------------- alignment
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_offset_views(torch, offset):
    rng = np.random.default_rng(30 + offset)
    n_obj, d, n, k = 20_000, 24, 50, 64
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng, _ = _engine(objects, False)
    rows = _raw_rows(rng, n_obj, rng.integers(0, 1500, n))
    raw_ptr, raw_idx = _raw(rows)
    subjects = _cuda(torch, rng.standard_normal((n, d)).astype(np.float32))
    ref = _np(torch, eng.topk_candidates_device(k, _cuda(torch, raw_ptr), _cuda(torch, raw_idx), subjects=subjects))

    def view(a):
        t = _cuda(torch, a).reshape(-1)
        buf = torch.zeros(len(t) + offset + 1, dtype=t.dtype, device="cuda")
        buf[offset : offset + len(t)] = t
        return buf[offset : offset + len(t)]

    out_bufs = [torch.full((n * k + offset + 2,), 777, dtype=torch.int32, device="cuda"),
                torch.full((n * k + offset + 2,), 5.0, device="cuda"), torch.full((n + offset + 2,), -3, dtype=torch.int32, device="cuda")]
    out = (out_bufs[0][offset : offset + n * k].view(n, k), out_bufs[1][offset : offset + n * k].view(n, k),
           out_bufs[2][offset : offset + n])
    got = eng.topk_candidates_device(k, view(raw_ptr), view(raw_idx), subjects=view(subjects.cpu().numpy()).view(n, d), out=out)
    torch.cuda.synchronize()
    _same(_np(torch, got), ref, f"offset {offset}")
    for buf, guard, size in zip(out_bufs, (777, 5.0, -3), (n * k, n * k, n)):  # nothing written outside the views
        assert bool((buf[:offset] == guard).all()) and bool((buf[offset + size :] == guard).all())


# ----------------------------------------------------------------------------------------------------------------- ranker
def _padded_to_csr(cands, n_obj):
    n, m = cands.shape
    rows = np.repeat(np.arange(n), m)
    flat = cands.reshape(-1)
    keep = flat >= 0
    return sparse.csr_matrix((np.ones(int(keep.sum()), np.float32), (rows[keep], flat[keep])), shape=(n, n_obj))


def _flatten(torch, sids, out):
    from rectools_b200.ranker import flatten_padded

    ids, scores, counts = _np(torch, out)
    return flatten_padded(np.asarray(sids, np.int64), ids, scores, counts)


@pytest.mark.parametrize("distance", ["dot", "cosine", "euclidean"])
def test_ranker_matches_rank_candidates(torch, distance):
    from rectools_b200.ranker import B200Ranker

    rng = np.random.default_rng(40)
    n_obj, n_sub, d, m = 30_000, 300, 32, 400
    users = rng.standard_normal((n_sub, d)).astype(np.float32)
    items = rng.standard_normal((n_obj, d)).astype(np.float32)
    ranker = B200Ranker(distance, users, items)
    sids = rng.integers(0, n_sub, 100)
    cands = rng.integers(0, n_obj, (100, m)).astype(np.int64)
    cands[rng.random(cands.shape) < 0.1] = -1
    cands[:5, 200:] = cands[:5, :200]  # repeats
    csr = _padded_to_csr(cands, n_obj)
    filt = sparse.random(100, n_obj, density=0.002, random_state=1, format="csr")
    whitelist = np.sort(rng.choice(n_obj, n_obj // 2, replace=False))
    for k, f, wl in ((10, None, None), (None, None, None), (50, filt, None), (50, filt, whitelist), (None, filt, whitelist)):
        exp = ranker.rank_candidates(sids, csr, k=k, filter_pairs_csr=f, sorted_object_whitelist=wl)
        got = ranker.rank_candidates_device(sids, _cuda(torch, cands), k=k, filter_pairs_csr=f, sorted_object_whitelist=wl)
        flat = _flatten(torch, sids, got)
        what = f"{distance} k={k} filter={f is not None} whitelist={wl is not None}"
        np.testing.assert_array_equal(flat[0], exp[0], err_msg=what)
        np.testing.assert_array_equal(flat[1], exp[1], err_msg=what)
        assert flat[2].dtype == np.asarray(exp[2]).dtype, what
        np.testing.assert_array_equal(flat[2].view(np.int32), np.asarray(exp[2]).view(np.int32), err_msg=what)
    # CUDA subject ids and a CUDA CSR filter give the same
    f_t = torch.sparse_csr_tensor(torch.from_numpy(filt.indptr.astype(np.int64)), torch.from_numpy(filt.indices.astype(np.int64)),
                                  torch.ones(filt.nnz), size=filt.shape).cuda()
    a = ranker.rank_candidates_device(sids, _cuda(torch, cands), k=50, filter_pairs_csr=filt)
    b = ranker.rank_candidates_device(_cuda(torch, sids.astype(np.int64)), _cuda(torch, cands.astype(np.int32)), k=50, filter_pairs_csr=f_t)
    _same(_np(torch, a), _np(torch, b), "cuda subject ids / filter")
    with pytest.raises(ValueError, match="Candidate object ids"):
        ranker.rank_candidates_device(sids, _cuda(torch, np.full((100, 3), n_obj, np.int64)))


@pytest.mark.parametrize("cosine", [False, True])
def test_torch_ranker_over_bf16_tensors(torch, cosine):
    from rectools_b200.integration import B200TorchRanker

    rng = np.random.default_rng(50 + cosine)
    n_obj, n_sub, d, m, k = 20_000, 200, 64, 500, 30
    users = torch.from_numpy(rng.standard_normal((n_sub, d)).astype(np.float32)).cuda().to(torch.bfloat16)
    items = torch.from_numpy(rng.standard_normal((n_obj, d)).astype(np.float32)).cuda().to(torch.bfloat16)
    ranker = B200TorchRanker("cosine" if cosine else "dot", "cuda:0", users, items)
    sids = rng.integers(0, n_sub, 64)
    cands = torch.from_numpy(rng.integers(-1, n_obj, (64, m)).astype(np.int64)).cuda()
    with pytest.raises(NotImplementedError):  # the host route still refuses resident device subjects
        ranker.rank_candidates(sids, _padded_to_csr(cands.cpu().numpy(), n_obj), k=k)
    ids, scores, counts = (t.cpu().numpy() for t in ranker.rank_candidates_device(sids, cands, k=k))
    # the engine's own scores (before the division by the subject norm) against the oracle
    eng = _np(torch, ranker.engine.topk_candidates_device(
        k, torch.arange(65, dtype=torch.int64, device="cuda") * m, cands.to(torch.int32).reshape(-1),
        subject_ids=torch.from_numpy(sids.astype(np.int64)).cuda()))
    norm = _normalised(list(cands.cpu().numpy().astype(np.int32)), n_obj)
    check_topk(eng, users.float().cpu().numpy()[sids], items.float().cpu().numpy(), k, cosine=cosine,
               filter_csr=_complement_filter(n_obj, *norm), name=f"bf16 torch ranker cosine={cosine}", max_ambiguous=1e-3)
    np.testing.assert_array_equal(ids, eng[0])
    np.testing.assert_array_equal(counts, eng[2])
    kept = np.arange(k)[None, :] < counts[:, None]
    want = eng[1] / ranker.subjects_norms[sids][:, None] if cosine else eng[1]
    np.testing.assert_array_equal(scores[kept].view(np.int32), want[kept].astype(np.float32).view(np.int32))


def test_group_and_sparse_rankers_raise(torch):
    from rectools_b200.ranker import B200Ranker

    rng = np.random.default_rng(60)
    items = rng.standard_normal((500, 8)).astype(np.float32)
    cands = _cuda(torch, rng.integers(0, 500, (4, 10)).astype(np.int32))
    ease = B200Ranker("dot", sparse.random(20, 8, density=0.3, format="csr", random_state=0), items)
    with pytest.raises(NotImplementedError, match="sparse"):
        ease.rank_candidates_device(np.arange(4), cands)
    group = B200Ranker("dot", rng.standard_normal((20, 8)).astype(np.float32), items, device=[0, 0])
    with pytest.raises(NotImplementedError, match="engine group"):
        group.rank_candidates_device(np.arange(4), cands)
    with pytest.raises(NotImplementedError, match="engine group"):
        group.engine.topk_candidates_device(10, None, None)


# ------------------------------------------------------------------------------------------------------- memory bound
def test_long_row_scratch_stays_within_the_plan(torch):
    """A chunk of many short rows and one row above S: only the long row sorts in global scratch, so the engine's device
    memory grows by what the plan charges the chunk (8 B per entry, 16 B more per entry of the long row), not by 16 B per
    entry of the whole chunk."""
    rng = np.random.default_rng(70)
    n_obj, d = 100_000, 16
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng, _ = _engine(objects, False)
    lens = [500] * 20_000 + [S + 700]
    rows = _raw_rows(rng, n_obj, lens)
    subjects = _cuda(torch, rng.standard_normal((len(rows), d)).astype(np.float32))
    got, exp, _ = _both(torch, eng, 10, rows, n_obj, subjects=subjects)
    _same(got, exp, "short rows + one long row")
    # (the host route above staged its own buffers: measure the device call alone on a fresh engine)
    eng2, _ = _engine(objects, False)
    before = eng2.info()["hbm_bytes"]
    raw_ptr, raw_idx = _raw(rows)
    again = eng2.topk_candidates_device(10, _cuda(torch, raw_ptr), _cuda(torch, raw_idx), subjects=subjects)
    _same(_np(torch, again), exp, "fresh engine")
    grown = eng2.info()["hbm_bytes"] - before
    total = sum(lens)
    planned = 8 * total + 16 * (S + 700)  # device outputs: no staging
    per_row = 8 * 2 * (len(lens) + 1)  # row pointers and the long rows' scratch offsets
    assert eng2.last_stats["n_chunks"] == 1
    assert grown <= 1.125 * (planned + per_row) + (4 << 20), (grown, planned)
    assert grown < 16 * total  # what sizing the scratch by the whole chunk would take alone


# ---------------------------------------------------------------------------------------------- python argument checks
def test_wrapper_refuses_what_the_engine_takes_on_trust(torch):
    from rectools_b200.ranker import Engine

    rng = np.random.default_rng(80)
    n_obj, d, n, m, k = 2000, 8, 16, 50, 10
    objects = rng.standard_normal((n_obj, d)).astype(np.float32)
    eng = Engine(objects, cosine=False)
    sub = _cuda(torch, rng.standard_normal((n, d)).astype(np.float32))
    ptr = _cuda(torch, np.arange(n + 1, dtype=np.int64) * m)
    idx = _cuda(torch, rng.integers(0, n_obj, n * m).astype(np.int32))
    guards = _guards(torch, n, k)
    for bad in ((guards[0][:, :5],) + guards[1:], (guards[0], guards[1].double(), guards[2]), guards[:2] + (guards[2][:3],)):
        with pytest.raises((TypeError, ValueError), match="`out`"):
            eng.topk_candidates_device(k, ptr, idx, subjects=sub, out=bad)
    _untouched(torch, guards)
    with pytest.raises(ValueError, match="cand_indices"):
        eng.topk_candidates_device(k, ptr, idx[:-1], subjects=sub, out=guards)
    with pytest.raises(IndexError, match="subject id"):
        eng.topk_candidates_device(k, ptr, idx, subjects=sub, subject_ids=_cuda(torch, np.full(n, n, np.int64)), out=guards)
    eng.set_subjects(rng.standard_normal((30, d)).astype(np.float32))
    with pytest.raises(IndexError, match="subject id"):
        eng.topk_candidates_device(k, ptr, idx, subject_ids=_cuda(torch, np.full(n, 30, np.int64)), out=guards)
    f_ptr = _cuda(torch, np.arange(n + 1, dtype=np.int64) * 2)
    with pytest.raises(ValueError, match="filter"):
        eng.topk_candidates_device(k, ptr, idx, subjects=sub, indptr=f_ptr, indices=_cuda(torch, np.zeros(2 * n - 1, np.int32)), out=guards)
    _untouched(torch, guards)
    got = eng.topk_candidates_device(k, ptr, idx, subject_ids=_cuda(torch, np.full(n, 29, np.int64)), indptr=f_ptr,
                                     indices=_cuda(torch, np.zeros(2 * n, np.int32)), out=guards)
    assert got[0] is guards[0] and eng.last_stats["path"] == 5

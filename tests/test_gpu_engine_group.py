"""GPU: engine groups (b200_rank_group_*, `EngineGroup`) against one engine on the same objects.

A group ranks the row slices of a call on its members, each an ordinary engine holding the whole catalogue, so every call
must return the full padded arrays of one engine bit for bit (ids, score bits, counts, unfilled slots) -- whatever path
each slice takes.  Groups [0], [0, 0] and [0, 0, 0] always run; groups over distinct devices need two GPUs.  A sample of
rows is also checked against the fp64 oracle.  Catalogues are integer-valued (tests/exact_cases.py)."""
import threading

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests import exact_cases as ec

pytestmark = pytest.mark.gpu

N_OBJ, D = 20_000, 16
SLEEP_CYCLES = 300_000_000  # as in tests/test_gpu_device_buffers.py


def _n_gpus():
    import torch

    return torch.cuda.device_count()


GROUPS = [
    pytest.param((0,), id="g0"),
    pytest.param((0, 0), id="g00"),
    pytest.param((0, 0, 0), id="g000"),
    pytest.param((0, 1), id="g01", marks=pytest.mark.skipif("_n_gpus() < 2", reason="needs torch.cuda.device_count() >= 2")),
    pytest.param((1, 0, 1), id="g101", marks=pytest.mark.skipif("_n_gpus() < 2", reason="needs torch.cuda.device_count() >= 2")),
]


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


def _same(got, exp, name):
    ids, sc, cnt = got
    eids, esc, ecnt = exp
    assert ids.shape == eids.shape, f"{name}: shape {ids.shape} vs {eids.shape}"
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, eids, err_msg=f"{name}: ids")
    np.testing.assert_array_equal(sc.view(np.int32), esc.view(np.int32), err_msg=f"{name}: score bits")


def _sample_oracle(got, distance, subjects, objects, subject_ids, k, filt=None, wl=None, n=8):
    """The fp64 oracle on a few rows (first, last, and spread between)."""
    rows = np.unique(np.linspace(0, len(subject_ids) - 1, n).astype(int))
    f = filt[rows] if filt is not None else None
    exp = ec.expected_padded(distance, subjects, objects, np.asarray(subject_ids)[rows], k, f, wl)
    ids, sc, cnt = got
    np.testing.assert_array_equal(cnt[rows], exp[2])
    np.testing.assert_array_equal(ids[rows], exp[0])
    np.testing.assert_array_equal(sc[rows], exp[1])


@pytest.fixture(scope="module")
def cat():
    rng = np.random.default_rng(11)
    objects = ec.int_matrix(rng, N_OBJ, D, -100, 100)
    subjects = ec.int_matrix(rng, 4000, D)
    wl = np.sort(rng.choice(N_OBJ, N_OBJ // 2, replace=False)).astype(np.int32)
    return objects, subjects, wl


def _filter(rng, n_rows, n_obj, full_rows=()):
    """Rows of viewed ids with empty rows, ids >= n_obj, duplicates and rows that view everything."""
    rows = [np.sort(rng.integers(0, n_obj + 50, rng.integers(0, 300))) for _ in range(n_rows)]
    rows[0] = np.empty(0, np.int64)
    for r in full_rows:
        if r < n_rows:
            rows[r] = np.arange(n_obj)
    return ec.csr_from_rows(rows, n_obj + 50)


@pytest.fixture(scope="module")
def engines(cat):
    from rectools_b200 import Engine, EngineGroup

    objects, subjects, _ = cat
    made = {}

    def get(devices, cosine):
        key = (devices, cosine)
        if key not in made:
            eng = Engine(objects, cosine=cosine) if devices is None else EngineGroup(objects, cosine=cosine, devices=devices)
            eng.set_subjects(subjects)
            made[key] = eng
        return made[key]

    yield get
    for e in made.values():
        e.close()


# (name, k, flags): paths 0, 1 narrow / wide / k > 128, 3 with the radix selection and k = None
ROUTES = [
    ("path0", 32, "exact"),
    ("narrow", 10, ""),
    ("wide", 100, ""),
    ("wide_l", 500, ""),
    ("radix", 1025, ""),
    ("all", None, ""),
]


@pytest.mark.parametrize("devices", GROUPS)
@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("route", [r[0] for r in ROUTES])
def test_resident_subjects_every_route(lib, cat, engines, monkeypatch, devices, distance, route):
    """Host subject ids into resident host subjects, with a filter (some rows view everything) and a whitelist, in batches
    of 1, fewer rows than members, 37 rows and 3000 rows (600 for k > 1024) cut into five slices with engine chunks of 256."""
    objects, subjects, wl = cat
    _, k, fl = next(r for r in ROUTES if r[0] == route)
    flags = lib.Q_FORCE_EXACT if fl == "exact" else 0
    one, grp = engines(None, distance == "cosine"), engines(devices, distance == "cosine")
    rng = np.random.default_rng(sum(map(ord, route + distance)))
    big = 3000 if k is not None and k <= 500 else 600  # (k = None: 20 000 columns per row)
    for n in (1, len(devices) - 1, 37, big):
        if n == 0:
            continue
        if n == big:
            monkeypatch.setenv("B200_GROUP_SLICE_ROWS", str(big // 4 - 50))
            monkeypatch.setenv("B200_CHUNK_ROWS", "256")
        ids = rng.integers(0, len(subjects), n)
        filt = _filter(rng, n, N_OBJ, full_rows=(1, n - 1))
        for f, w in ((None, None), (filt, None), (filt, wl)):
            n_pos = N_OBJ if w is None else len(w)
            kk = n_pos if k is None else k
            kw = dict(subject_ids=ids, whitelist=w, flags=flags)
            if f is not None:
                kw.update(indptr=f.indptr, indices=f.indices)
            exp = one.topk(kk, **kw)
            got = grp.topk(kk, **kw)
            _same(got, exp, f"{route} n={n} filter={f is not None} wl={w is not None}")
            assert sum(m["k_out"] > 0 for m in grp.last_member_stats) >= 1
            if n == 37 and f is not None:
                _sample_oracle(got, distance, subjects, objects, ids, kk, f, w)
        monkeypatch.delenv("B200_GROUP_SLICE_ROWS", raising=False)
        monkeypatch.delenv("B200_CHUNK_ROWS", raising=False)


@pytest.mark.parametrize("devices", GROUPS)
def test_sparse_subjects_and_filter_with_nonzero_indptr_base(lib, cat, engines, monkeypatch, devices):
    """Path 2 (EASE-shaped CSR subjects, DOT) and a filter whose indptr arrays start at a non-zero offset into their
    indices: the group equals one engine on the zero-based arrays, with slices of 5 rows."""
    objects, subjects, _ = cat
    one, grp = engines(None, False), engines(devices, False)
    rng = np.random.default_rng(3)
    n = 37
    a = sparse.random(n, D, density=0.4, random_state=2, format="csr", dtype=np.float32)
    a.data[:] = rng.integers(-3, 4, a.nnz)
    filt = _filter(rng, n, N_OBJ, full_rows=(5,))
    pad_s, pad_f = 7, 13  # leading entries no row refers to
    s_indptr = a.indptr.astype(np.int64) + pad_s
    s_indices = np.r_[np.zeros(pad_s, np.int32), a.indices.astype(np.int32)]
    s_data = np.r_[np.full(pad_s, 99.0, np.float32), a.data]
    f_indptr = filt.indptr.astype(np.int64) + pad_f
    f_indices = np.r_[np.arange(pad_f, dtype=np.int32), filt.indices.astype(np.int32)]

    def call(eng, base, k, flags, out):
        q = lib.Query()
        if base:
            arrs = (s_indptr, s_indices, s_data, f_indptr, f_indices)
        else:
            arrs = (a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data, filt.indptr.astype(np.int64),
                    filt.indices.astype(np.int32))
        q.sub_indptr, q.sub_indices, q.sub_data, q.csr_indptr, q.csr_indices = [x.ctypes.data for x in arrs]
        q.n_rows, q.k, q.flags = n, k, flags
        q.out_ids, q.out_scores, q.out_counts = [o.ctypes.data for o in out]
        st = eng.topk_raw(q)
        del arrs
        return st

    for k in (10, 1025):
        for slices in ("", "5"):
            if slices:
                monkeypatch.setenv("B200_GROUP_SLICE_ROWS", slices)
            k_out = min(k, N_OBJ)
            outs = [(np.full((n, k_out), 777, np.int32), np.full((n, k_out), 5.0, np.float32), np.full(n, -3, np.int32)) for _ in range(3)]
            assert call(one, False, k, 0, outs[0])["path"] == 2
            call(one, True, k, 0, outs[1])
            st = call(grp, True, k, 0, outs[2])
            assert st["path"] == 2
            _same(outs[1], outs[0], "one engine, indptr base")
            _same(outs[2], outs[0], f"group, indptr base, k={k} slices={slices}")
            exp = ec.expected_padded("dot", a, objects, np.arange(n), k, filt)
            _same(outs[2], exp, "oracle")
            monkeypatch.delenv("B200_GROUP_SLICE_ROWS", raising=False)


@pytest.mark.parametrize("devices", GROUPS)
def test_object_rows_path4(lib, devices, monkeypatch):
    """Path 4 (EASE item-to-item): the stored rows of a d = n_objects group, with a filter and a whitelist, k = 10 and None."""
    from rectools_b200 import Engine, EngineGroup
    from rectools_b200.ranker import rank_object_rows_padded

    rng = np.random.default_rng(4)
    w = ec.int_matrix(rng, 600, 600, -100, 100)
    one, grp = Engine(w, cosine=False), EngineGroup(w, cosine=False, devices=devices)
    try:
        targets = rng.integers(0, 600, 37)
        filt = _filter(rng, 37, 600, full_rows=(2,))
        wl = np.sort(rng.choice(600, 300, replace=False))
        monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "4")
        for k in (10, None):
            for f, wlist in ((None, None), (filt, wl)):
                exp = rank_object_rows_padded(one, targets, k, f, wlist)
                got = rank_object_rows_padded(grp, targets, k, f, wlist)
                assert grp.last_stats["path"] == 4
                for a, b, nm in zip(got[1:], exp[1:], ("ids", "scores", "counts")):
                    np.testing.assert_array_equal(a.view(np.int32) if a.dtype == np.float32 else a,
                                                  b.view(np.int32) if b.dtype == np.float32 else b, err_msg=nm)
    finally:
        one.close()
        grp.close()


def _out(torch, n, k_out, on_device, dev="cuda:0"):
    if on_device:
        return (torch.full((n, k_out), 777, dtype=torch.int32, device=dev), torch.full((n, k_out), 5.0, device=dev),
                torch.full((n,), -3, dtype=torch.int32, device=dev))
    return np.full((n, k_out), 777, np.int32), np.full((n, k_out), 5.0, np.float32), np.full(n, -3, np.int32)


def _ptr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def _host(torch, out):
    torch.cuda.synchronize()
    return tuple(o.cpu().numpy() if hasattr(o, "cpu") else o for o in out)


@pytest.mark.parametrize("devices", GROUPS)
@pytest.mark.parametrize("sub_kind", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("obj_kind", ["f32", "bf16"])
def test_device_inputs_and_outputs(lib, torch, cat, monkeypatch, devices, sub_kind, obj_kind):
    """Device subjects (fp32 / fp16 / bf16, sliced in their own dtype), a device filter with a non-zero indptr base, a
    device whitelist, device and host outputs; fp32 and bf16 device objects (create_ex from the home device)."""
    from rectools_b200 import Engine, EngineGroup

    objects, _, wl = cat
    dev = torch.device(f"cuda:{devices[0]}")
    tdt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
    dt = {"f32": lib.DT_F32, "f16": lib.DT_F16, "bf16": lib.DT_BF16}
    obj_t = torch.from_numpy(objects).to(dev).to(tdt[obj_kind]).contiguous()
    torch.cuda.synchronize()
    kw = dict(objects_device_ptr=obj_t.data_ptr(), shape=objects.shape, objects_dtype=dt[obj_kind])
    with torch.cuda.device(dev):
        one = Engine(None, cosine=False, device=devices[0], **kw)
    grp = EngineGroup(None, cosine=False, devices=devices, **kw)
    try:
        rng = np.random.default_rng(6)
        n = 300
        subs = ec.int_matrix(rng, n, D)
        filt = _filter(rng, n, N_OBJ, full_rows=(3,))
        pad = 9
        sub_t = torch.from_numpy(subs).to(dev).to(tdt[sub_kind]).contiguous()
        ip = torch.from_numpy(filt.indptr.astype(np.int64) + pad).to(dev)
        ix = torch.from_numpy(np.r_[np.zeros(pad, np.int32), filt.indices.astype(np.int32)]).to(dev)
        wl_t = torch.from_numpy(wl).to(dev)
        monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "64")
        for k, use_wl in ((10, False), (100, True), (1025, False)):
            n_pos = len(wl) if use_wl else N_OBJ
            for out_dev in (False, True):
                outs = []
                for eng in (one, grp):
                    out = _out(torch, n, min(k, n_pos), out_dev, dev)
                    flags = lib.Q_INPUTS_ON_DEVICE | (lib.Q_OUTPUTS_ON_DEVICE if out_dev else 0)
                    eng.topk_ptrs(n, k, *map(_ptr, out), flags, subjects=sub_t.data_ptr(), indptr=ip.data_ptr(), indices=ix.data_ptr(),
                                  whitelist=wl_t.data_ptr() if use_wl else 0, n_whitelist=n_pos if use_wl else 0,
                                  subject_dtype=dt[sub_kind])
                    outs.append(_host(torch, out))
                _same(outs[1], outs[0], f"k={k} wl={use_wl} out_dev={out_dev}")
                widened = sub_t.float().cpu().numpy()
                exp = ec.expected_padded("dot", widened, obj_t.float().cpu().numpy(), np.arange(n), k, filt, wl if use_wl else None)
                _same(outs[1], exp, "oracle")
    finally:
        one.close()
        grp.close()


@pytest.mark.parametrize("devices", GROUPS)
def test_resident_device_subjects(lib, torch, cat, monkeypatch, devices):
    from rectools_b200 import Engine, EngineGroup

    objects, subjects, _ = cat
    dev = torch.device(f"cuda:{devices[0]}")
    with torch.cuda.device(dev):
        one = Engine(objects, cosine=True, device=devices[0])
    grp = EngineGroup(objects, cosine=True, devices=devices)
    sub_t = torch.from_numpy(subjects).to(dev)
    torch.cuda.synchronize()
    try:
        one.set_subjects_device(sub_t.data_ptr(), len(subjects))
        grp.set_subjects_device(sub_t.data_ptr(), len(subjects))
        monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "333")
        ids = np.random.default_rng(8).integers(0, len(subjects), 2000)
        for k in (10, 100):
            _same(grp.topk(k, subject_ids=ids), one.topk(k, subject_ids=ids), f"k={k}")
    finally:
        one.close()
        grp.close()


def test_refusals_leave_outputs_untouched(lib, cat, engines):
    objects, subjects, wl = cat
    grp = engines((0, 0), False)
    ids = np.arange(50, dtype=np.int64)
    cases = [
        (dict(flags=lib.Q_FORCE_TC), 10, lib.E_UNSUPPORTED),
        (dict(flags=lib.Q_SHARED_THRESHOLDS), 10, lib.E_UNSUPPORTED),
        (dict(flags=lib.Q_FORCE_TC | lib.Q_FORCE_EXACT), 10, lib.E_UNSUPPORTED),
        (dict(), 0, lib.E_INVALID),
        (dict(subject_dtype=lib.DT_F16), 10, lib.E_INVALID),
    ]
    for kw, k, code in cases:
        out = _out(None, 50, 10, False)
        before = tuple(o.copy() for o in out)
        q = lib.Query()
        q.subject_ids, q.n_rows, q.k, q.flags = ids.ctypes.data, 50, k, kw.get("flags", 0)
        q.subject_dtype = kw.get("subject_dtype", lib.DT_F32)
        q.out_ids, q.out_scores, q.out_counts = [o.ctypes.data for o in out]
        st = (lib.Stats * 2)()
        rc = lib.load().b200_rank_group_topk(grp._h, q, None, st)  # pylint: disable=protected-access
        assert rc == code, (kw, k, rc, lib.load().b200_rank_last_error())
        for a, b in zip(out, before):
            np.testing.assert_array_equal(a, b)
    # host object_rows out of range, on a d = n_objects group
    from rectools_b200 import EngineGroup

    w = np.eye(64, dtype=np.float32)
    g2 = EngineGroup(w, cosine=False, devices=(0, 0))
    try:
        out = _out(None, 3, 5, False)
        before = tuple(o.copy() for o in out)
        with pytest.raises(ValueError, match="object_rows"):
            g2.topk(5, object_rows=np.array([1, 64, 2]), out=out)
        for a, b in zip(out, before):
            np.testing.assert_array_equal(a, b)
        with pytest.raises(NotImplementedError):
            g2.candidate_snapshot()
    finally:
        g2.close()


def test_group_info(cat, engines):
    grp = engines((0, 0), False)
    info = grp.info()
    assert len(info["members"]) == 2 and info["hbm_bytes"] >= sum(m["hbm_bytes"] for m in info["members"])


def _behind_sleep(torch, stream, writes):
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SLEEP_CYCLES)
        for dst, src in writes:
            dst.copy_(src)
        ev = torch.cuda.Event()
        ev.record(stream)
    assert not ev.query(), "the producer finished before the group call: the sleep is too short to test anything"
    return ev


@pytest.mark.parametrize("producer", ["side", "legacy"])
def test_device_inputs_and_outputs_follow_the_caller_stream(lib, torch, cat, engines, monkeypatch, producer):
    """Device inputs written behind a sleep on the caller's stream (a side stream, or the legacy stream with stream = NULL)
    over decoys; device outputs then copied on that stream behind another sleep while a second call overwrites them."""
    objects, _, _ = cat
    grp = engines((0, 0, 0), False)
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(12)
    n, k = 200, 20
    real, decoy = ec.int_matrix(rng, n, D), ec.int_matrix(rng, n, D)
    exp, exp_decoy = (ec.expected_padded("dot", s, objects, np.arange(n), k) for s in (real, decoy))
    assert any(not np.array_equal(a, b) for a, b in zip(exp, exp_decoy))
    buf, src = torch.from_numpy(decoy).to(dev), torch.from_numpy(real).to(dev)
    if producer == "side":
        stream = torch.cuda.Stream()
        q_stream = stream.cuda_stream
    else:
        stream = torch.cuda.current_stream()
        assert stream.cuda_stream == 0
        q_stream = 0
    monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "32")
    x = _out(torch, n, k, True)
    _behind_sleep(torch, stream, [(buf, src)])
    flags = lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE | lib.Q_FORCE_EXACT
    grp.topk_ptrs(n, k, *map(_ptr, x), flags, subjects=buf.data_ptr(), stream=q_stream)
    # the outputs are read behind a sleep on the same stream; the next call must not overwrite them first
    y = tuple(torch.empty_like(t) for t in x)
    second = torch.from_numpy(decoy).to(dev)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SLEEP_CYCLES)
        for dst, s in zip(y, x):
            dst.copy_(s)
        ev = torch.cuda.Event()
        ev.record(stream)
    assert not ev.query()
    grp.topk_ptrs(n, k, *map(_ptr, x), flags, subjects=second.data_ptr(), stream=q_stream)
    _same(_host(torch, y), exp, f"{producer}: first call")
    _same(_host(torch, x), exp_decoy, f"{producer}: second call")


@pytest.mark.parametrize("shared", [True, False], ids=["one_group", "two_groups"])
def test_python_threads(lib, cat, engines, monkeypatch, shared):
    objects, subjects, _ = cat
    one = engines(None, False)
    groups = [engines((0, 0), False)] * 2 if shared else [engines((0, 0), False), engines((0, 0, 0), False)]
    monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "128")
    rng = np.random.default_rng(13)
    batches = [rng.integers(0, len(subjects), 1000) for _ in range(6)]
    expected = [one.topk(10, subject_ids=b) for b in batches]
    results = [None] * len(batches)
    errors = []

    def work(t):
        try:
            for i in range(t, len(batches), 2):
                results[i] = groups[t].topk(10, subject_ids=batches[i])
        except Exception as e:  # pylint: disable=broad-except
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for i, (got, exp) in enumerate(zip(results, expected)):
        _same(got, exp, f"batch {i}")


# ------------------------------------------------------------------------------------------- through install()
@pytest.fixture(scope="module")
def ref():
    if not stage_reference.available():
        pytest.skip("reference package not staged (oracle/_ref)")
    added = stage_reference.add_to_path()
    import rectools  # noqa: F401

    yield
    import rectools_b200

    rectools_b200.uninstall()
    stage_reference.remove_from_path(added)


def _frames_equal(a, b):
    assert list(a.columns) == list(b.columns)
    for c in a.columns:
        np.testing.assert_array_equal(a[c].to_numpy(), b[c].to_numpy(), err_msg=c)


def _factors(n, d, seed):
    return (np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32) / np.sqrt(d)).astype(np.float32)


def test_models_through_install_group_equal_install_int(ref, monkeypatch):
    """`install(device=[0, 0])` against `install(device=0)`: PureSVD and injected ALS `recommend` / `recommend_to_items`,
    EASE `recommend` / `recommend_to_items` (u2i through the sparse scorer, i2i through the stored rows) -- equal frames."""
    from rectools.models import EASEModel, PureSVDModel

    import rectools_b200
    from rectools_b200 import integration
    from tests.ref_models import injected_als, synthetic_dataset

    monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "500")
    dataset = synthetic_dataset(6000, 3000, 30, seed=1)
    models = {
        "puresvd": PureSVDModel(factors=32, random_state=0).fit(dataset),
        "als": injected_als(_factors(6000, 64, 1), _factors(3000, 64, 2)),
        "ease": EASEModel(regularization=200.0).fit(synthetic_dataset(5000, 1200, 25, seed=4)),
    }
    ease_ds = synthetic_dataset(5000, 1200, 25, seed=4)
    users = np.random.default_rng(3).permutation(dataset.user_id_map.external_ids)[:5000]
    wl = dataset.item_id_map.external_ids[::7]
    calls = {
        "u2i": lambda m, ds, us: m.recommend(us, ds, k=10, filter_viewed=True),
        "u2i_whitelist": lambda m, ds, us: m.recommend(us, ds, k=10, filter_viewed=True, items_to_recommend=ds.item_id_map.external_ids[::7]),
        "i2i": lambda m, ds, us: m.recommend_to_items(ds.item_id_map.external_ids[:400], ds, k=6),
    }
    del wl
    results = {}
    for device in (0, [0, 0]):
        rectools_b200.install(device=device)
        try:
            for name, model in models.items():
                ds = ease_ds if name == "ease" else dataset
                us = ease_ds.user_id_map.external_ids[::2] if name == "ease" else users
                for call, fn in calls.items():
                    results[(str(device), name, call)] = fn(model, ds, us)
            if device != 0:
                assert all(isinstance(e, rectools_b200.EngineGroup) for e in integration._ENGINE_CACHE.values())  # pylint: disable=protected-access
        finally:
            rectools_b200.uninstall()
    for (device, name, call), got in results.items():
        if device != "0":
            _frames_equal(got, results[("0", name, call)])


def test_transformer_seam_with_devices(ref, monkeypatch):
    import torch
    from scipy import sparse as sp

    from rectools_b200.integration import make_similarity_module

    monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "300")
    n_users, n_tokens, d, k = 3000, 20_001, 64, 10
    g = torch.Generator().manual_seed(7)
    user_embs = torch.randn((n_users, d), generator=g) / d**0.5
    item_embs = torch.randn((n_tokens, d), generator=g) / d**0.5
    user_ids = np.random.default_rng(0).permutation(n_users)[:2000]
    rng = np.random.default_rng(1)
    cols = rng.integers(1, n_tokens, size=(len(user_ids), 30))
    rows = np.repeat(np.arange(len(user_ids)), 30)
    ui = sp.csr_matrix((np.ones(cols.size, np.float32), (rows, cols.reshape(-1))), shape=(len(user_ids), n_tokens))
    ui.sum_duplicates()
    ui.data[:] = 1.0
    whitelist = np.arange(1, n_tokens)
    dev = torch.device("cuda:0")
    for emb in (item_embs, item_embs.to(torch.bfloat16)):
        for distance in ("dot", "cosine"):
            a = make_similarity_module()(distance=distance)._recommend_u2i(  # pylint: disable=protected-access
                user_embs, emb.to(dev), user_ids, k, whitelist, ui)
            b = make_similarity_module(devices=[0, 0])(distance=distance)._recommend_u2i(  # pylint: disable=protected-access
                user_embs, emb.to(dev), user_ids, k, whitelist, ui)
            for x, y in zip(a, b):
                np.testing.assert_array_equal(np.asarray(x), np.asarray(y))

"""GPU: memory the engine does not own -- 16-bit device subjects and factors, and device buffers on the caller's streams.

A. 16-bit subjects (`query.subject_dtype`, widened on the device) and fp16 / bf16 object factors (`b200_rank_create_ex`)
   against the fp64 oracle of the exactly widened values, on every route that takes dense subjects, with and without a
   device whitelist and filter, into device and host outputs; special values; the reuse of the engine's widened buffer
   across calls of different sizes; the refusals.
B. Ordering.  Every device buffer starts out holding a decoy -- a valid input of the same shape whose answer differs --
   and the real input is written over it on the caller's stream behind a `torch.cuda._sleep`, still pending when the
   engine is called.  A call that does not wait for the caller's stream ranks the decoy.  Decoy index arrays hold
   in-range values only, so a missing wait gives a wrong answer, never an out-of-bounds read.

Catalogues are integer-valued (tests/exact_cases.py), exact in fp16 and bf16; every comparison is of the full padded arrays
(ids, scores, counts, unfilled slots) with no tie tolerance, and every call asserts the path it took."""
import threading

import numpy as np
import pytest
from scipy import sparse

from tests import exact_cases as ec
from tests.tc_reference import Catalogue, check_snapshot

pytestmark = pytest.mark.gpu

N_OBJ, D, N_ROWS = 20_000, 16, 300
# ~150 ms at the H100's boost clock (longer at lower clocks); the tests assert that the producer is still pending
SLEEP_CYCLES = 300_000_000


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


def _same(got, exp, name):
    """Full padded arrays; scores bit for bit (zeros of either sign compare equal: the sign of an exact zero sum is not
    part of the result definition)."""
    ids, sc, cnt = got
    eids, esc, ecnt = exp
    assert ids.shape == eids.shape, f"{name}: shape {ids.shape} vs {eids.shape}"
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, eids, err_msg=f"{name}: ids")
    bits = lambda a: np.where(a == 0, np.float32(0), a).astype(np.float32).view(np.int32)  # noqa: E731
    np.testing.assert_array_equal(bits(sc), bits(esc), err_msg=f"{name}: scores")


def _prefix(exp, k):
    ids, sc, cnt = exp
    return ids[:, :k], sc[:, :k], np.minimum(cnt, k)


def _differs(a, b):
    return any(x.shape != y.shape or not np.array_equal(x, y) for x, y in zip(a, b))


def _tdtype(torch, name):
    return {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[name]


def _dt(lib, name):
    return {"f32": lib.DT_F32, "f16": lib.DT_F16, "bf16": lib.DT_BF16}[name]


def _out(torch, dev, n_rows, k_out, on_device):
    """Output buffers full of garbage (device tensors or numpy arrays)."""
    if on_device:
        return (torch.full((n_rows, k_out), 777, dtype=torch.int32, device=dev), torch.full((n_rows, k_out), 5.0, device=dev),
                torch.full((n_rows,), -3, dtype=torch.int32, device=dev))
    return np.full((n_rows, k_out), 777, np.int32), np.full((n_rows, k_out), 5.0, np.float32), np.full(n_rows, -3, np.int32)


def _ptr(a):
    return a.data_ptr() if hasattr(a, "data_ptr") else a.ctypes.data


def _host(torch, out):
    torch.cuda.synchronize()
    return tuple(o.cpu().numpy() if hasattr(o, "cpu") else o for o in out)


def _engine(torch, dev, objects, cosine, obj_kind, tc_mode="auto"):
    """An engine over `objects` (integer-valued fp32) handed over as fp32 host, fp32 device, fp16 or bf16 device.
    Returns (engine, device tensor to keep alive or None)."""
    from rectools_b200 import Engine, _lib

    if obj_kind == "f32host":
        return Engine(objects, cosine=cosine, tc_mode=tc_mode), None
    kind = {"f32dev": "f32", "f16": "f16", "bf16": "bf16"}[obj_kind]
    t = torch.from_numpy(objects).to(dev).to(_tdtype(torch, kind)).contiguous()
    torch.cuda.synchronize()
    eng = Engine(None, cosine=cosine, tc_mode=tc_mode, objects_device_ptr=t.data_ptr(), shape=objects.shape,
                 objects_dtype=_dt(_lib, kind))
    return eng, t


def _filter(rng, n_rows, n_obj):
    """A filter CSR with empty rows, ids >= n_obj and duplicate entries."""
    rows = [rng.integers(0, n_obj + 100, rng.integers(0, 400)) for _ in range(n_rows)]
    rows[0] = np.empty(0, np.int64)
    rows[1] = np.r_[rows[1], rows[1][:3]]
    return ec.csr_from_rows(rows, n_obj)


# ================================================================================================ A. 16-bit inputs
@pytest.fixture(scope="module")
def cat_a():
    """Objects [N_OBJ, D] in [-100, 100] (few enough ties that the certificate passes rows; exact in fp16 and bf16),
    subjects [N_ROWS, D] in [-3, 3], a whitelist holding the last object, a filter."""
    rng = np.random.default_rng(101)
    objects = ec.int_matrix(rng, N_OBJ, D, -100, 100)
    subjects = ec.int_matrix(rng, N_ROWS, D)
    wl = np.union1d(np.sort(rng.choice(N_OBJ - 1, N_OBJ // 2, replace=False)), [N_OBJ - 1]).astype(np.int32)
    filt = _filter(rng, N_ROWS, N_OBJ)
    return objects, subjects, wl, filt


@pytest.fixture(scope="module")
def oracle_a(cat_a):
    """{(distance, filtered): the oracle at k = n_pos}, computed once per module."""
    objects, subjects, wl, filt = cat_a
    cache = {}

    def get(distance, filtered):
        key = (distance, filtered)
        if key not in cache:
            f, w = (filt, wl) if filtered else (None, None)
            cache[key] = ec.expected_padded(distance, subjects, objects, np.arange(N_ROWS), len(objects) if w is None else len(w), f, w)
        return cache[key]

    return get


# (name, ks, flags, env, path, wide); None = k = n_pos
ROUTES = [
    ("path0", (1, 32, 33, 128), "exact", {}, 0, 0),
    ("narrow", (10,), "tc", {}, 1, 0),
    ("wide", (100,), "tc", {}, 1, 1),
    ("wide_l", (500,), "tc", {}, 1, 1),
    ("path3", (129,), "", {"B200_WIDE": "0"}, 3, 0),
    ("radix", (2000, None), "", {}, 3, 0),
]


def _flags(lib, kind):
    return {"exact": lib.Q_FORCE_EXACT, "tc": lib.Q_FORCE_TC, "": 0}[kind]


@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("sub_kind", ["f16", "bf16"])
@pytest.mark.parametrize("obj_kind", ["f32host", "f32dev", "f16", "bf16"])
def test_16bit_subjects_and_factors_on_every_route(lib, torch, dev, monkeypatch, cat_a, oracle_a, obj_kind, sub_kind, distance):
    objects, subjects, wl, filt = cat_a
    cosine = distance == "cosine"
    eng, keep = _engine(torch, dev, objects, cosine, obj_kind)
    tc = lib.TC_BF16 if obj_kind == "bf16" else lib.TC_FP16  # AUTO: bf16 for bf16 factors, else fp16
    assert eng.info()["tc_dtype"] == tc
    sub16 = torch.from_numpy(subjects).to(dev).to(_tdtype(torch, sub_kind)).contiguous()
    d_wl = torch.from_numpy(wl).to(dev)
    d_ip = torch.from_numpy(filt.indptr.astype(np.int64)).to(dev)
    d_ix = torch.from_numpy(filt.indices.astype(np.int32)).to(dev)
    torch.cuda.synchronize()
    stream = torch.cuda.current_stream().cuda_stream
    for filtered in (False, True):
        exp_all = oracle_a(distance, filtered)
        n_pos = len(wl) if filtered else N_OBJ
        extra = dict(whitelist=d_wl.data_ptr(), n_whitelist=len(wl), indptr=d_ip.data_ptr(), indices=d_ix.data_ptr()) if filtered else {}
        for name, ks, fl, env, path, wide in ROUTES:
            with monkeypatch.context() as m:
                for k_, v_ in env.items():
                    m.setenv(k_, v_)
                for k in ks:
                    k = n_pos if k is None else k
                    for out_dev in (False, True):
                        out = _out(torch, dev, N_ROWS, min(k, n_pos), out_dev)
                        flags = lib.Q_INPUTS_ON_DEVICE | _flags(lib, fl) | (lib.Q_OUTPUTS_ON_DEVICE if out_dev else 0)
                        st = eng.topk_ptrs(N_ROWS, k, *map(_ptr, out), flags, subjects=sub16.data_ptr(), stream=stream,
                                           subject_dtype=_dt(lib, sub_kind), **extra)
                        tag = f"{obj_kind}/{sub_kind}/{distance} filtered={filtered} {name} k={k} out_dev={out_dev}"
                        assert (st["path"], st["wide"]) == (path, wide), (tag, st)
                        assert st["tc_dtype"] == (tc if path == 1 else 0), (tag, st)
                        _same(_host(torch, out), _prefix(exp_all, k), tag)
    eng.close()
    del keep


def _special_rows(torch, kind):
    """16-bit subject rows at the edges of the type, as a torch tensor of that type [n, D]."""
    rng = np.random.default_rng(5)
    rows = np.zeros((8, D), np.float64)
    if kind == "f16":
        rows[0] = rng.integers(-1023, 1024, D) * 2.0**-24  # subnormals (the smallest is 2^-24)
        rows[1] = rng.choice([-65504.0, 65504.0, 0.0, 2.0**-24], D)  # the largest finite values
        rows[2] = rng.integers(-3, 4, D) * 2.0**-14  # around the smallest normal
    else:
        rows[0] = rng.integers(-3, 4, D) * 1e30
        rows[1] = rng.integers(-3, 4, D) * 1e-30
        rows[2] = rng.choice([1e30, -1e-30, 3.0, 0.0], D)
    rows[3] = -0.0  # negative zeros only
    # rows[4]: all zero
    rows[5, 7] = 3.0 if kind == "f16" else 3e30  # a single non-zero element
    rows[6] = -0.0
    rows[6, 0] = -2.0**-24 if kind == "f16" else -1e-30  # the smallest magnitude, among negative zeros
    rows[7] = rng.integers(-3, 4, D)
    return torch.from_numpy(rows.astype(np.float32)).to(_tdtype(torch, kind))


@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("sub_kind", ["f16", "bf16"])
def test_16bit_subjects_special_values(lib, torch, dev, cat_a, sub_kind, distance):
    """Subnormals, the largest finite values, 1e+-30, -0.0, an all-zero row and a single non-zero element, against the
    oracle over the exactly widened values, on the exhaustive kernel and the tensor-core path."""
    objects = cat_a[0]
    eng, _ = _engine(torch, dev, objects, distance == "cosine", "f32host")
    rows = _special_rows(torch, sub_kind)
    wide = rows.to(torch.float32).numpy()  # widening is exact
    assert np.isfinite(wide).all()
    n = len(wide)
    d_rows = rows.to(dev).contiguous()
    torch.cuda.synchronize()
    exp = ec.expected_padded(distance, wide, objects, np.arange(n), 100)
    for k, fl, path in ((32, lib.Q_FORCE_EXACT, 0), (10, lib.Q_FORCE_TC, 1), (100, lib.Q_FORCE_TC, 1)):
        for out_dev in (False, True):
            out = _out(torch, dev, n, k, out_dev)
            flags = lib.Q_INPUTS_ON_DEVICE | fl | (lib.Q_OUTPUTS_ON_DEVICE if out_dev else 0)
            st = eng.topk_ptrs(n, k, *map(_ptr, out), flags, subjects=d_rows.data_ptr(), subject_dtype=_dt(lib, sub_kind))
            tag = f"{sub_kind}/{distance} k={k} out_dev={out_dev}"
            assert st["path"] == path, (tag, st)
            _same(_host(torch, out), _prefix(exp, k), tag)
    eng.close()


@pytest.mark.parametrize("sub_kind", ["f16", "bf16"])
def test_widened_buffer_reuse_across_calls(lib, torch, dev, cat_a, sub_kind):
    """One engine: host subjects (600 rows), 16-bit (200 rows: the buffer holds the last call's rows beyond them),
    16-bit (900 rows: the buffer grows), host again; each on the exhaustive kernel and the tensor-core path."""
    objects = cat_a[0]
    eng, _ = _engine(torch, dev, objects, False, "f32host")
    rng = np.random.default_rng(17)
    for step, (n, kind) in enumerate(((600, "host"), (200, sub_kind), (900, sub_kind), (600, "host"))):
        subjects = ec.int_matrix(rng, n, D)
        exp = ec.expected_padded("dot", subjects, objects, np.arange(n), 32)
        for k, fl, path in ((32, lib.Q_FORCE_EXACT, 0), (10, lib.Q_FORCE_TC, 1)):
            tag = f"step {step} ({kind}, {n} rows) k={k}"
            if kind == "host":
                got = eng.topk(k, subjects=subjects, flags=fl)
                st = eng.last_stats
            else:
                d_sub = torch.from_numpy(subjects).to(dev).to(_tdtype(torch, kind))
                torch.cuda.synchronize()
                out = _out(torch, dev, n, k, False)
                st = eng.topk_ptrs(n, k, *map(_ptr, out), lib.Q_INPUTS_ON_DEVICE | fl, subjects=d_sub.data_ptr(),
                                   subject_dtype=_dt(lib, kind))
                got = out
            assert st["path"] == path, (tag, st)
            _same(got, _prefix(exp, k), tag)
    eng.close()


@pytest.fixture(scope="module")
def tie_case():
    """A tie catalogue (planted blocks across ranks / split edges, exact ties everywhere), 800 rows, and its oracle at k = 500."""
    from rectools_b200 import Engine

    probe = Engine(np.ones((64, 4), np.float32), cosine=False)
    sm = int(probe.info()["sm_count"])
    probe.close()
    cat = ec.tie_catalogue(sm, n_obj=100_000, n_subjects=800)
    assert np.abs(cat.objects).max() <= 256 and np.abs(cat.subjects).max() <= 256  # exact in bf16 and fp16
    return cat, ec.expected_padded("dot", cat.subjects, cat.objects, np.arange(len(cat.subjects)), 500)


@pytest.mark.parametrize("kind", ["f16", "bf16"])
def test_tie_catalogue_in_16_bits_takes_the_fallback(lib, torch, dev, monkeypatch, tie_case, kind):
    """The tie catalogue as 16-bit objects and subjects: planted ties make the certificate fail, so rows are re-ranked from
    the widened copies; three or more row chunks on the tensor-core routes (the wide mode's list budget for 16-bit device
    subjects, B200_CHUNK_ROWS for host subjects)."""
    cat, exp = tie_case
    n = len(cat.subjects)
    eng, keep = _engine(torch, dev, cat.objects, False, kind)
    tc = lib.TC_BF16 if kind == "bf16" else lib.TC_FP16
    d_sub = torch.from_numpy(cat.subjects).to(dev).to(_tdtype(torch, kind)).contiguous()
    torch.cuda.synchronize()
    for k, env, min_chunks in ((10, {}, 1), (100, {}, 1), (500, {"B200_WIDE_BUDGET_MB": "1"}, 3)):
        with monkeypatch.context() as m:
            for k_, v_ in env.items():
                m.setenv(k_, v_)
            out = _out(torch, dev, n, k, True)
            st = eng.topk_ptrs(n, k, *map(_ptr, out), lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE | lib.Q_FORCE_TC,
                               subjects=d_sub.data_ptr(), subject_dtype=_dt(lib, kind))
        tag = f"{kind} 16-bit subjects k={k}"
        assert st["path"] == 1 and st["tc_dtype"] == tc and st["n_chunks"] >= min_chunks, (tag, st)
        assert st["n_fallback_rows"] > 0, (tag, st)
        _same(_host(torch, out), _prefix(exp, k), tag)
    with monkeypatch.context() as m:
        m.setenv("B200_CHUNK_ROWS", "256")
        for k in (10, 100):
            got = eng.topk(k, subjects=cat.subjects, flags=lib.Q_FORCE_TC)
            st = eng.last_stats
            tag = f"{kind} objects, host subjects k={k}"
            assert st["path"] == 1 and st["tc_dtype"] == tc and st["n_chunks"] >= 3 and st["n_fallback_rows"] > 0, (tag, st)
            _same(got, _prefix(exp, k), tag)
    eng.close()
    del keep


def test_16bit_refusals_leave_outputs_untouched(lib, torch, dev, cat_a):
    from rectools_b200 import Engine

    objects, subjects, _, _ = cat_a
    eng = Engine(objects, cosine=False)
    eng.set_subjects(subjects)
    d16 = torch.from_numpy(subjects).to(dev).half()
    h16 = subjects.astype(np.float16)
    d_ids = torch.arange(10, dtype=torch.int64, device=dev)
    d_rows = torch.arange(10, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    IN = lib.Q_INPUTS_ON_DEVICE
    cases = {
        "host 16-bit subjects": dict(flags=0, subjects=h16.ctypes.data, subject_dtype=lib.DT_F16),
        "16-bit subjects + subject_ids": dict(flags=IN, subjects=d16.data_ptr(), subject_ids=d_ids.data_ptr(),
                                              n_subjects_total=len(subjects), subject_dtype=lib.DT_F16),
        "16-bit resident subjects": dict(flags=IN, subject_ids=d_ids.data_ptr(), subject_dtype=lib.DT_BF16),
        "subject_dtype + object_rows": dict(flags=IN, object_rows=d_rows.data_ptr(), subject_dtype=lib.DT_F16),
        "subject_dtype 3": dict(flags=IN, subjects=d16.data_ptr(), subject_dtype=3),
    }
    for name, kw in cases.items():
        out = _out(torch, dev, 10, 10, False)
        flags = kw.pop("flags")
        with pytest.raises(ValueError):
            eng.topk_ptrs(10, 10, *map(_ptr, out), flags, **kw)
        assert (out[0] == 777).all() and (out[1] == 5.0).all() and (out[2] == -3).all(), name
    eng.close()
    with pytest.raises(ValueError, match="16-bit object factors must be device pointers"):
        Engine(objects.astype(np.float16), cosine=False, objects_dtype=lib.DT_F16)


# ================================================================================================ B. stream ordering
def _behind_sleep(torch, stream, writes):
    """Synchronise (the buffers hold their decoys), then on `stream`: sleep, copy each real input over its buffer.
    Asserts that the copies are still pending on return."""
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        torch.cuda._sleep(SLEEP_CYCLES)
        for dst, src in writes:
            dst.copy_(src)
        ev = torch.cuda.Event()
        ev.record(stream)
    assert not ev.query(), "the producer finished before the engine call: the sleep is too short to test anything"
    return ev


def _decoyed(torch, dev, real, decoy):
    """(buffer holding the decoy, device copy of the real input) of one input array."""
    assert real.shape == decoy.shape and real.dtype == decoy.dtype
    return torch.from_numpy(np.ascontiguousarray(decoy)).to(dev), torch.from_numpy(np.ascontiguousarray(real)).to(dev)


def _same_nnz_indptr(rng, indptr):
    """Another row split of the same entries: a decoy indptr with the same indptr[n]."""
    nnz, n = int(indptr[-1]), len(indptr) - 1
    return np.r_[0, np.sort(rng.integers(0, nnz + 1, n - 1)), nnz].astype(np.int64)


@pytest.fixture(scope="module")
def cat_b():
    rng = np.random.default_rng(202)
    return ec.int_matrix(rng, N_OBJ, D, -100, 100), rng


@pytest.fixture(scope="module")
def engines_b(cat_b):
    from rectools_b200 import Engine

    objects, _ = cat_b
    dot, cos = Engine(objects, cosine=False), Engine(objects, cosine=True)
    yield dot, cos
    dot.close()
    cos.close()


def _route_case(lib, route, cat_b, engines_b):
    """(engine, real inputs {name: array}, decoy inputs, call(ptrs) -> kwargs for topk_ptrs / a Query, n_rows, k, flags,
    expected path, oracle(inputs) -> padded expectation)."""
    from rectools_b200 import Engine

    objects, _ = cat_b
    rng = np.random.default_rng(sum(map(ord, route)))
    n, m = 64, 400
    if route == "rows":  # path 4: the stored rows of a d = n_objects engine are the score rows
        w = ec.int_matrix(rng, 600, 600, -100, 100)
        real = {"object_rows": rng.choice(600, n, replace=False).astype(np.int64)}
        decoy = {"object_rows": rng.choice(600, n, replace=False).astype(np.int64)}
        eng = Engine(w, cosine=False)
        oracle = lambda x: ec.expected_padded("dot", np.eye(600, dtype=np.float32)[x["object_rows"]], w.T, np.arange(n), 50)  # noqa: E731
        return eng, real, decoy, n, 50, 0, 4, oracle
    if route == "sparse":  # path 2
        a = sparse.random(n, D, density=0.5, random_state=1, format="csr", dtype=np.float32)
        real = {"sub_indptr": a.indptr.astype(np.int64), "sub_indices": a.indices.astype(np.int32),
                "sub_data": rng.integers(-3, 4, a.nnz).astype(np.float32)}
        decoy = {"sub_indptr": _same_nnz_indptr(rng, real["sub_indptr"]), "sub_indices": rng.integers(0, D, a.nnz).astype(np.int32),
                 "sub_data": rng.integers(-3, 4, a.nnz).astype(np.float32)}
        oracle = lambda x: ec.expected_padded(  # noqa: E731
            "dot", sparse.csr_matrix((x["sub_data"], x["sub_indices"], x["sub_indptr"]), shape=(n, D)), objects, np.arange(n), 20)
        return engines_b[0], real, decoy, n, 20, 0, 2, oracle
    real = {"subjects": ec.int_matrix(rng, m, D)}
    decoy = {"subjects": ec.int_matrix(rng, m, D)}
    if route in ("path0", "path1"):  # subjects through subject_ids, a filter
        real["subject_ids"] = rng.integers(0, m, n).astype(np.int64)
        decoy["subject_ids"] = rng.integers(0, m, n).astype(np.int64)
        f_real, f_decoy = _filter(rng, n, N_OBJ), _filter(rng, n, N_OBJ)
        nnz = min(f_real.nnz, f_decoy.nnz)  # the same nnz: cut both to the shorter
        real["indptr"] = np.minimum(f_real.indptr, nnz).astype(np.int64)
        real["indices"] = f_real.indices[:nnz].astype(np.int32)
        decoy["indptr"] = np.minimum(f_decoy.indptr, nnz).astype(np.int64)
        decoy["indices"] = f_decoy.indices[:nnz].astype(np.int32)
        k, flags, path = (32, lib.Q_FORCE_EXACT, 0) if route == "path0" else (10, lib.Q_FORCE_TC, 1)

        def oracle(x):
            f = sparse.csr_matrix((np.ones(len(x["indices"]), np.float32), x["indices"], x["indptr"]), shape=(n, N_OBJ + 100))
            return ec.expected_padded("dot", x["subjects"], objects, x["subject_ids"], k, f)

        return engines_b[0], real, decoy, n, k, flags, path, oracle
    real["subjects"], decoy["subjects"] = real["subjects"][:n], decoy["subjects"][:n]
    if route == "wide":  # a whitelist
        real["whitelist"] = np.sort(rng.choice(N_OBJ, N_OBJ // 2, replace=False)).astype(np.int32)
        decoy["whitelist"] = np.sort(rng.choice(N_OBJ, N_OBJ // 2, replace=False)).astype(np.int32)
        oracle = lambda x: ec.expected_padded("cosine", x["subjects"], objects, np.arange(n), 100, None, x["whitelist"])  # noqa: E731
        return engines_b[1], real, decoy, n, 100, lib.Q_FORCE_TC, 1, oracle
    if route == "radix":  # path 3, k > 1024
        oracle = lambda x: ec.expected_padded("dot", x["subjects"], objects, np.arange(n), 2000)  # noqa: E731
        return engines_b[0], real, decoy, n, 2000, 0, 3, oracle
    assert route == "f16"  # 16-bit subjects: the widening runs after the wait
    real["subjects"], decoy["subjects"] = real["subjects"].astype(np.float16), decoy["subjects"].astype(np.float16)
    oracle = lambda x: ec.expected_padded("dot", x["subjects"].astype(np.float32), objects, np.arange(n), 10)  # noqa: E731
    return engines_b[0], real, decoy, n, 10, lib.Q_FORCE_TC, 1, oracle


def _query(lib, n, k, flags, stream, ptrs, out, n_pos):
    q = lib.Query()
    q.subjects, q.subject_ids = ptrs.get("subjects"), ptrs.get("subject_ids")
    q.n_rows, q.n_subjects_total = n, (400 if "subject_ids" in ptrs else 0)
    q.csr_indptr, q.csr_indices = ptrs.get("indptr"), ptrs.get("indices")
    q.whitelist, q.n_whitelist = ptrs.get("whitelist"), (n_pos if "whitelist" in ptrs else 0)
    q.sub_indptr, q.sub_indices, q.sub_data = ptrs.get("sub_indptr"), ptrs.get("sub_indices"), ptrs.get("sub_data")
    q.object_rows = ptrs.get("object_rows")
    q.subject_dtype = lib.DT_F16 if "subjects" in ptrs and ptrs.get("_f16") else lib.DT_F32
    q.k, q.flags = k, flags
    q.out_ids, q.out_scores, q.out_counts = map(_ptr, out)
    q.stream = stream or None
    return q


@pytest.mark.parametrize("producer", ["side", "legacy"])
@pytest.mark.parametrize("route", ["path0", "path1", "wide", "sparse", "radix", "rows", "f16"])
def test_device_inputs_wait_for_the_producer_stream(lib, torch, dev, cat_b, engines_b, route, producer):
    """Every device input is written behind a sleep on the caller's stream: a side stream passed as query.stream, or the
    legacy default stream with query.stream = NULL."""
    eng, real, decoy, n, k, flags, path, oracle = _route_case(lib, route, cat_b, engines_b)
    exp, exp_decoy = oracle(real), oracle(decoy)
    assert _differs(exp, exp_decoy), "the decoy must have another answer"
    bufs = {name: _decoyed(torch, dev, real[name], decoy[name]) for name in real}
    if producer == "side":
        stream = torch.cuda.Stream()
        q_stream = stream.cuda_stream
    else:
        stream = torch.cuda.current_stream()
        assert stream == torch.cuda.default_stream() and stream.cuda_stream == 0, "torch's current stream is the legacy stream"
        q_stream = 0
    ptrs = {name: b.data_ptr() for name, (b, _) in bufs.items()}
    if route == "f16":
        ptrs["_f16"] = True
    n_pos = len(real["whitelist"]) if "whitelist" in real else eng.n_objects
    out = _out(torch, dev, n, min(k, n_pos), False)
    _behind_sleep(torch, stream, [(b, r) for b, r in bufs.values()])
    st = eng.topk_raw(_query(lib, n, k, flags | lib.Q_INPUTS_ON_DEVICE, q_stream, ptrs, out, n_pos))
    assert st["path"] == path, st
    _same(out, exp, f"{route} / {producer}")
    if route == "rows":
        eng.close()


def test_device_outputs_are_not_overwritten_before_the_caller_read_them(lib, torch, dev, cat_b, engines_b):
    """Call 1 writes device outputs X on stream S; S then sleeps and copies X to Y; call 2 writes X on S.  Y holds call 1's
    answer, X call 2's."""
    objects, _ = cat_b
    eng = engines_b[0]
    rng = np.random.default_rng(9)
    a, b = ec.int_matrix(rng, 64, D), ec.int_matrix(rng, 64, D)
    exp_a, exp_b = (ec.expected_padded("dot", s, objects, np.arange(64), 20) for s in (a, b))
    assert _differs(exp_a, exp_b)
    s = torch.cuda.Stream()
    x = _out(torch, dev, 64, 20, True)
    flags = lib.Q_OUTPUTS_ON_DEVICE | lib.Q_FORCE_EXACT
    eng.topk_ptrs(64, 20, *map(_ptr, x), flags, subjects=a.ctypes.data, stream=s.cuda_stream)
    y = tuple(torch.empty_like(t) for t in x)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        for dst, src in zip(y, x):
            dst.copy_(src)
        ev = torch.cuda.Event()
        ev.record(s)
    assert not ev.query(), "the sleep is too short to test anything"
    st = eng.topk_ptrs(64, 20, *map(_ptr, x), flags, subjects=b.ctypes.data, stream=s.cuda_stream)
    assert st["path"] == 0, st
    _same(_host(torch, y), exp_a, "Y: call 1")
    _same(_host(torch, x), exp_b, "X: call 2")


@pytest.mark.parametrize("obj_kind", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_create_reads_device_objects_after_the_producer(lib, torch, dev, monkeypatch, cat_b, obj_kind, distance):
    """The object matrix is written behind a sleep on the legacy stream over a decoy with other row norms and another
    absmax; create must derive norms, eps and the tensor-core copy from the real matrix.  DOT: the captured tensor-core
    pass is checked against an fp64 restatement over the real objects (a copy built from the decoy breaks premise P1)."""
    from rectools_b200 import Engine

    objects, _ = cat_b
    cosine = distance == "cosine"
    decoy = (np.roll(objects, 1, axis=0) * 2).astype(np.float32)  # exact in 16 bits too
    tdt = _tdtype(torch, obj_kind)
    buf = torch.from_numpy(decoy).to(dev).to(tdt).contiguous()
    real = torch.from_numpy(objects).to(dev).to(tdt)
    _behind_sleep(torch, torch.cuda.default_stream(), [(buf, real)])
    eng = Engine(None, cosine=cosine, objects_device_ptr=buf.data_ptr(), shape=objects.shape, objects_dtype=_dt(lib, obj_kind))
    bf16 = obj_kind == "bf16"
    assert eng.info()["tc_dtype"] == (lib.TC_BF16 if bf16 else lib.TC_FP16)
    rng = np.random.default_rng(41)
    subjects = ec.int_matrix(rng, 300, D)
    exp = ec.expected_padded(distance, subjects, objects, np.arange(300), 100)
    for k, fl, path in ((10, lib.Q_FORCE_TC, 1), (100, lib.Q_FORCE_TC, 1), (32, lib.Q_FORCE_EXACT, 0)):
        with monkeypatch.context() as m:
            m.setenv("B200_TC_SNAPSHOT", "1")
            got = eng.topk(k, subjects=subjects, flags=fl)
        st = eng.last_stats
        tag = f"{obj_kind}/{distance} k={k}"
        assert st["path"] == path, (tag, st)
        _same(got, _prefix(exp, k), tag)
        if path == 1 and not cosine:
            snap = eng.candidate_snapshot()
            assert snap is not None, tag
            cat = Catalogue(objects, cosine=False, bf16=bf16)
            rows = snap["rows"].astype(np.int64)
            rep = check_snapshot(snap, cat, subjects[rows], sparse.csr_matrix((len(rows), N_OBJ), dtype=np.float32))
            assert rep.ok, f"{tag}: {rep.summary()}"
    eng.close()
    del buf


def test_resident_device_subjects_wait_for_the_legacy_stream(lib, torch, dev, cat_b):
    """set_subjects_device, then the matrix is rewritten in place behind a sleep on the legacy stream; a call with host
    subject_ids, host outputs and stream NULL gathers the rewritten rows."""
    from rectools_b200 import Engine

    objects, _ = cat_b
    rng = np.random.default_rng(13)
    real, decoy = ec.int_matrix(rng, 400, D), ec.int_matrix(rng, 400, D)
    sids = rng.integers(0, 400, 64).astype(np.int64)
    for k, fl, path in ((32, lib.Q_FORCE_EXACT, 0), (10, lib.Q_FORCE_TC, 1)):
        eng = Engine(objects, cosine=False)
        buf, src = _decoyed(torch, dev, real, decoy)
        torch.cuda.synchronize()
        eng.set_subjects_device(buf.data_ptr(), 400)
        exp = ec.expected_padded("dot", real, objects, sids, k)
        assert _differs(exp, ec.expected_padded("dot", decoy, objects, sids, k))
        _behind_sleep(torch, torch.cuda.default_stream(), [(buf, src)])
        got = eng.topk(k, subject_ids=sids, flags=fl)
        assert eng.last_stats["path"] == path, eng.last_stats
        _same(got, exp, f"resident device subjects k={k}")
        eng.close()


@pytest.mark.parametrize("certified", [False, True])
def test_merges_read_lists_behind_the_stream(lib, torch, dev, certified):
    """b200_rank_merge / _certified on stream S, their lists written on S behind a sleep."""
    rng = np.random.default_rng(23 + certified)
    n_lists, n_rows, k = 4, 37, 24
    real, decoy = ec.merge_case(rng, n_lists, n_rows, k), ec.merge_case(rng, n_lists, n_rows, k)
    b_real = np.where(rng.random((n_lists, n_rows)) < 0.3, -np.inf, rng.integers(-3, 4, (n_lists, n_rows))).astype(np.float32)
    b_decoy = np.full((n_lists, n_rows), -np.inf, np.float32)
    exp = ec.expected_merge(*real, k, b_real if certified else None)
    assert _differs(exp[:3], ec.expected_merge(*decoy, k)[:3])
    bufs = [_decoyed(torch, dev, r, d_) for r, d_ in zip(real + (b_real,), decoy + (b_decoy,))]
    o_ids = torch.full((n_rows, k), 777, dtype=torch.int32, device=dev)
    o_sc = torch.full((n_rows, k), 5.0, device=dev)
    o_cnt = torch.full((n_rows,), -3, dtype=torch.int32, device=dev)
    fail_rows = torch.full((n_rows,), -1, dtype=torch.int32, device=dev)
    fail_count = torch.zeros((1,), dtype=torch.int32, device=dev)
    s = torch.cuda.Stream()
    _behind_sleep(torch, s, bufs)
    h = lib.load()
    ptrs = [b.data_ptr() for b, _ in bufs]
    if certified:
        lib.check(h.b200_rank_merge_certified(0, s.cuda_stream, n_lists, n_rows, k, *ptrs, 0, o_ids.data_ptr(), o_sc.data_ptr(),
                                              o_cnt.data_ptr(), fail_rows.data_ptr(), fail_count.data_ptr()))
    else:
        lib.check(h.b200_rank_merge(0, s.cuda_stream, n_lists, n_rows, k, *ptrs[:3], o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr()))
    s.synchronize()
    _same((o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy()), exp[:3], f"merge certified={certified}")
    if certified:
        np.testing.assert_array_equal(np.sort(fail_rows.cpu().numpy()[: int(fail_count.item())]), exp[3])


@pytest.mark.parametrize("shared", [False, True], ids=["two_engines", "one_engine"])
def test_threads_on_their_own_streams(lib, torch, dev, cat_b, engines_b, shared):
    """Two Python threads, each on its own stream with device inputs and outputs, 20 calls each alternating DOT / COSINE
    and k = 10 / 100 (two engines); then both threads on one engine."""
    objects, _ = cat_b
    rng = np.random.default_rng(31)
    subs = [ec.int_matrix(rng, 64, D) for _ in range(2)]
    dists = ["dot"] if shared else ["dot", "cosine"]
    exp = {(t, d_): ec.expected_padded(d_, subs[t], objects, np.arange(64), 100) for t in range(2) for d_ in dists}
    engs = {"dot": engines_b[0], "cosine": engines_b[1]}
    errors = []
    barrier = threading.Barrier(2)

    def work(t):
        try:
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                sub = torch.from_numpy(subs[t]).to(dev)
                barrier.wait()
                for i in range(20):
                    d_ = dists[i % len(dists)]
                    k = (10, 100)[(i // 2) % 2]
                    out = _out(torch, dev, 64, k, True)
                    engs[d_].topk_ptrs(64, k, *map(_ptr, out), lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE | lib.Q_FORCE_TC,
                                       subjects=sub.data_ptr(), stream=s.cuda_stream)
                    s.synchronize()
                    got = tuple(o.cpu().numpy() for o in out)
                    _same(got, _prefix(exp[(t, d_)], k), f"thread {t} call {i} {d_} k={k}")
        except BaseException as e:  # pylint: disable=broad-except
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors[0]

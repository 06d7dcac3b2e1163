"""GPU: 16-bit object factors kept at 16 bits (B200_F_OBJECTS_16BIT) against the widened engine.

Every fp16 / bf16 value is exact in fp32, and every kernel that reads the objects widens each element on load to the type
it computes in, in the same order.  So two engines built from the same 16-bit values -- one widened into an fp32 master
copy (no flag), one that keeps them at 16 bits -- must return the same full padded arrays (ids, score bits, counts,
unfilled slots) on every path: 0 (exhaustive), 1 (tensor-core candidates + fp64 re-score, narrow / wide / k > 128),
2 (sparse subjects), 3 (k > 1024 and k = None) and 4 (stored rows).  The fused kernel reads the tensor-core copy, which
must come out byte-identical: its snapshots are compared too.  Sampled rows are checked against the fp64 oracle."""
import gc

import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests import exact_cases as ec

pytestmark = pytest.mark.gpu

N_MAIN, D_MAIN = 70_000, 200
DTYPES = ["float16", "bfloat16"]


@pytest.fixture(scope="module")
def torch():
    import torch

    return torch


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


def _dt(lib, torch, t):
    return {torch.float16: lib.DT_F16, torch.bfloat16: lib.DT_BF16}[t.dtype]


def _catalogue(torch, rng, n, d, dtype, extreme=False):
    """16-bit objects on the device with special rows: zeros (zero-norm COSINE rows), -0.0, 16-bit subnormals, a
    duplicate; `extreme` adds the largest finite value, +-inf and NaN."""
    tdt = getattr(torch, dtype)
    fi = torch.finfo(tdt)
    x = torch.from_numpy(rng.standard_normal((n, d)).astype(np.float32)).to(tdt)
    specials = [
        lambda r: r.zero_(),
        lambda r: r.fill_(-0.0),
        lambda r: r.fill_(fi.tiny / 4),  # subnormal in the 16-bit type
        lambda r: r.__setitem__(slice(0, 1), -fi.tiny / 8),
    ]
    if extreme:
        specials += [
            lambda r: r.__setitem__(slice(0, 1), fi.max),
            lambda r: r.__setitem__(slice(0, 1), -fi.max),
            lambda r: r.__setitem__(slice(0, 1), float("inf")),
            lambda r: r.__setitem__(slice(0, 1), float("-inf")),
            lambda r: r.__setitem__(slice(0, 1), float("nan")),
        ]
    for i, f in enumerate(specials):
        if 3 * i + 1 < n:
            f(x[3 * i + 1])
    if n > 40:
        x[40] = x[41]  # exact duplicates: ties broken by id
    return x if not torch.cuda.is_available() else x.cuda()


def _pair(lib, torch, t, cosine, tc_mode="auto"):
    """(widened engine, 16-bit engine) over the same device matrix."""
    from rectools_b200 import Engine

    kw = dict(objects_device_ptr=t.data_ptr(), shape=tuple(t.shape), objects_dtype=_dt(lib, torch, t), tc_mode=tc_mode)
    return Engine(None, cosine=cosine, **kw), Engine(None, cosine=cosine, keep_16bit=True, **kw)


def _same(got, exp, name):
    ids, sc, cnt = got
    eids, esc, ecnt = exp
    assert ids.shape == eids.shape, f"{name}: shape {ids.shape} vs {eids.shape}"
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, eids, err_msg=f"{name}: ids")
    np.testing.assert_array_equal(sc.view(np.int32), esc.view(np.int32), err_msg=f"{name}: score bits")


def _filter(rng, n_rows, n_obj, full_rows=()):
    rows = [np.sort(rng.integers(0, n_obj + 20, rng.integers(0, 200))) for _ in range(n_rows)]
    rows[0] = np.empty(0, np.int64)
    for r in full_rows:
        if r < n_rows:
            rows[r] = np.arange(n_obj)  # everything viewed: an empty row
    return ec.csr_from_rows(rows, n_obj + 20)


def _device_call(lib, torch, eng, k, subjects, filt, wl, flags):
    """Device subjects (fp32, fp16 or bf16, batch order), filter, whitelist and outputs."""
    dev = torch.device("cuda", eng.device)
    n = subjects.shape[0]
    n_pos = eng.n_objects if wl is None else len(wl)
    k_out = min(k, n_pos)
    sdt = {torch.float32: lib.DT_F32, torch.float16: lib.DT_F16, torch.bfloat16: lib.DT_BF16}[subjects.dtype]
    keep = [subjects]
    kw = {}
    if filt is not None:
        ip = torch.from_numpy(filt.indptr.astype(np.int64)).to(dev)
        ix = torch.from_numpy(filt.indices.astype(np.int32)).to(dev)
        keep += [ip, ix]
        kw.update(indptr=ip.data_ptr(), indices=ix.data_ptr())
    if wl is not None:
        w = torch.from_numpy(np.asarray(wl, np.int32)).to(dev)
        keep.append(w)
        kw.update(whitelist=w.data_ptr(), n_whitelist=len(wl))
    oi = torch.full((n, k_out), 7, dtype=torch.int32, device=dev)
    os_ = torch.full((n, k_out), 7.0, dtype=torch.float32, device=dev)
    oc = torch.full((n,), 7, dtype=torch.int32, device=dev)
    eng.topk_ptrs(n, k, oi.data_ptr(), os_.data_ptr(), oc.data_ptr(), flags | lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE,
                  subjects=subjects.data_ptr(), stream=torch.cuda.current_stream(dev).cuda_stream, subject_dtype=sdt, **kw)
    torch.cuda.synchronize(dev)
    return oi.cpu().numpy(), os_.cpu().numpy(), oc.cpu().numpy()


def _sample_oracle(got, distance, subjects, objects32, k, filt=None, wl=None, n=6):
    rows = np.unique(np.linspace(0, len(subjects) - 1, n).astype(int))
    f = filt[rows] if filt is not None else None
    exp = ec.expected_padded(distance, subjects, objects32, rows, k, f, wl)
    _same(tuple(a[rows] for a in got), exp, "oracle")


# (name, k, flags): path 0, path 1 narrow / wide / 128 < k <= 1024, path 3 (k > 1024 and k = None: n_pos)
ROUTES = [("path0", 10, "exact"), ("narrow", 10, ""), ("wide", 100, ""), ("wide_l", 200, ""), ("k1024", 1024, ""),
          ("path3", 1025, ""), ("all", None, "")]


@pytest.fixture(scope="module")
def main_cat(torch):
    out = {}
    for dtype in DTYPES:
        rng = np.random.default_rng(5 + len(dtype))
        out[dtype] = _catalogue(torch, rng, N_MAIN, D_MAIN, dtype)
    return out


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("route", [r[0] for r in ROUTES])
def test_routes_bit_identical(lib, torch, main_cat, monkeypatch, dtype, distance, route):
    """Host subjects in row chunks of 256 (four chunks) with a filter that empties some rows and a whitelist; resident
    subjects by id; device fp32 / fp16 / bf16 subjects into device outputs.  Widened and 16-bit engines must agree bit for
    bit, and sampled rows match the fp64 oracle."""
    _, k, fl = next(r for r in ROUTES if r[0] == route)
    flags = lib.Q_FORCE_EXACT if fl == "exact" else 0
    t = main_cat[dtype]
    objects32 = t.float().cpu().numpy()
    wide, kept = _pair(lib, torch, t, distance == "cosine")
    try:
        rng = np.random.default_rng(sum(map(ord, route + distance + dtype)))
        n_rows = 40 if k is None else 800
        subjects = rng.standard_normal((n_rows, D_MAIN)).astype(np.float32)
        subjects[2] = 0.0
        wl = np.sort(rng.choice(N_MAIN, N_MAIN // 2, replace=False)).astype(np.int32)
        filt = _filter(rng, n_rows, N_MAIN, full_rows=(1, n_rows - 1))
        kk = N_MAIN if k is None else k
        monkeypatch.setenv("B200_CHUNK_ROWS", "256")  # (the hook's floor)
        for name, w, f in (("plain", None, None), ("filter+wl", wl, filt)):
            a = wide.topk(kk, subjects=subjects, indptr=None if f is None else f.indptr, indices=None if f is None else f.indices,
                          whitelist=w, flags=flags)
            b = kept.topk(kk, subjects=subjects, indptr=None if f is None else f.indptr, indices=None if f is None else f.indices,
                          whitelist=w, flags=flags)
            _same(b, a, f"{name} host")
            if route in ("narrow", "wide", "wide_l") and fl == "":
                assert kept.last_stats["path"] == 1, kept.last_stats
            if route == "narrow" and w is None:
                assert kept.last_stats["n_chunks"] >= 3, kept.last_stats
            _sample_oracle(b, distance, subjects, objects32, kk, f, w)
        monkeypatch.delenv("B200_CHUNK_ROWS")
        # resident subjects, ids out of order and repeated
        for e in (wide, kept):
            e.set_subjects(subjects)
        sid = rng.integers(0, n_rows, n_rows)
        _same(kept.topk(kk, subject_ids=sid, whitelist=wl, flags=flags), wide.topk(kk, subject_ids=sid, whitelist=wl, flags=flags),
              "resident")
        # device inputs and outputs, subjects in three types
        dev = torch.device("cuda:0")
        for sdt in (torch.float32, torch.float16, torch.bfloat16):
            s = torch.from_numpy(subjects).to(sdt).to(dev).contiguous()
            a = _device_call(lib, torch, wide, kk, s, filt, wl, flags)
            b = _device_call(lib, torch, kept, kk, s, filt, wl, flags)
            _same(b, a, f"device {sdt}")
    finally:
        wide.close()
        kept.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("d", [1, 3, 8, 63, 65, 200, 320])
def test_widths_and_sizes(lib, torch, dtype, d):
    """d across the vector / element-wise re-score loads and the 64-wide steps of the exhaustive kernels, n_obj from 1 up,
    catalogues with +-inf, NaN and the largest finite value: paths 0, 1 (forced, narrow and wide) and 3."""
    for n_obj in (1, 7, 4000):
        for extreme in (False, True):
            rng = np.random.default_rng(d * 1000 + n_obj + extreme)
            t = _catalogue(torch, rng, n_obj, d, dtype, extreme=extreme)
            subjects = rng.standard_normal((70, d)).astype(np.float32)
            filt = _filter(rng, 70, n_obj, full_rows=(3,))
            for distance in ("dot", "cosine"):
                wide, kept = _pair(lib, torch, t, distance == "cosine")
                try:
                    for k, flags in ((5, lib.Q_FORCE_EXACT), (10, lib.Q_FORCE_TC), (100, lib.Q_FORCE_TC), (1025, 0), (10, 0)):
                        if flags == lib.Q_FORCE_TC and n_obj < 4 * 32:
                            continue
                        a = wide.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, flags=flags)
                        b = kept.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, flags=flags)
                        _same(b, a, f"d={d} n={n_obj} extreme={extreme} {distance} k={k} flags={flags}")
                        if flags == lib.Q_FORCE_TC:
                            assert kept.last_stats["path"] == 1
                    if not extreme and n_obj > 1:
                        _sample_oracle(b, distance, subjects, t.float().cpu().numpy(), 10, filt)
                finally:
                    wide.close()
                    kept.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_sparse_subjects(lib, torch, dtype):
    """Path 2: the transposed fp32 copy is built from the 16-bit rows."""
    rng = np.random.default_rng(3)
    n_obj, d = 5000, 65
    t = _catalogue(torch, rng, n_obj, d, dtype, extreme=True)
    wide, kept = _pair(lib, torch, t, False)
    try:
        sub = sparse.random(200, d, density=0.2, format="csr", random_state=4, dtype=np.float32)
        filt = _filter(rng, 200, n_obj, full_rows=(5,))
        wl = np.sort(rng.choice(n_obj, 3000, replace=False)).astype(np.int32)
        for k in (10, 1025, n_obj):
            for w in (None, wl):
                a = wide.topk(k, sparse_subjects=sub, indptr=filt.indptr, indices=filt.indices, whitelist=w)
                b = kept.topk(k, sparse_subjects=sub, indptr=filt.indptr, indices=filt.indices, whitelist=w)
                assert kept.last_stats["path"] == 2
                _same(b, a, f"sparse k={k}")
    finally:
        wide.close()
        kept.close()


@pytest.mark.parametrize("dtype", DTYPES)
def test_object_rows(lib, torch, dtype):
    """Path 4 on a square 16-bit matrix with +-inf, NaN, subnormals: the stored rows are widened before the order key."""
    rng = np.random.default_rng(8)
    n = 3000
    t = _catalogue(torch, rng, n, n, dtype, extreme=True)
    wide, kept = _pair(lib, torch, t, False)
    try:
        rows = np.concatenate([np.arange(20), rng.integers(0, n, 300)]).astype(np.int64)
        filt = _filter(rng, len(rows), n, full_rows=(7,))
        wl = np.sort(rng.choice(n, 2000, replace=False)).astype(np.int32)
        for k in (10, 1025, n):
            for w in (None, wl):
                a = wide.topk(k, object_rows=rows, indptr=filt.indptr, indices=filt.indices, whitelist=w)
                b = kept.topk(k, object_rows=rows, indptr=filt.indptr, indices=filt.indices, whitelist=w)
                assert kept.last_stats["path"] == 4
                _same(b, a, f"rows k={k}")
        # the scores are the stored values themselves
        ids, sc, cnt = kept.topk(10, object_rows=rows[20:])
        m = t.float().cpu().numpy()
        for r in range(5):
            np.testing.assert_array_equal(sc[r, : cnt[r]], m[rows[20 + r], ids[r, : cnt[r]]])
    finally:
        wide.close()
        kept.close()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_snapshots_equal(lib, torch, main_cat, monkeypatch, dtype, distance):
    """The fused pass reads the tensor-core copy, and the approximate score of a (row, object) pair is a function of that
    copy and the row alone: every pair both snapshots hold must carry the same score bits, so the copy built from 16-bit
    rows is the one built from the widened rows on every candidate seen.  The metadata (eps, obj_exp, max_obj_norm, the
    row exponents, the pass's shape) must be equal too.  Which pairs a list keeps depends on the order the tiles arrive in
    (the adaptive thresholds), which varies between runs even on one engine: the widened engine runs twice to bound that
    variation, and the 16-bit engine must share at least as many pairs with it."""
    monkeypatch.setenv("B200_TC_SNAPSHOT", "1")
    t = main_cat[dtype]
    wide, kept = _pair(lib, torch, t, distance == "cosine")

    def pairs(s):
        ids, sc, cnt = s["cand_ids"], s["cand_scores"], s["cand_counts"]
        held = (np.arange(ids.shape[2])[None, None, :] < np.minimum(cnt, ids.shape[2])[:, :, None]) & (ids >= 0) & (ids != 0x7FFFFFFF)
        rows = np.broadcast_to(np.arange(ids.shape[1])[None, :, None], ids.shape)
        key = rows[held].astype(np.int64) * (1 << 31) + ids[held]
        key, first = np.unique(key, return_index=True)
        return key, sc[held].view(np.int32)[first]

    try:
        subjects = np.random.default_rng(1).standard_normal((256, D_MAIN)).astype(np.float32)
        snaps = []
        for e in (wide, wide, kept):
            e.topk(10, subjects=subjects)
            snaps.append(e.candidate_snapshot())
        shared = []
        for a, b in ((snaps[0], snaps[1]), (snaps[0], snaps[2])):
            assert a is not None and b is not None
            assert a.keys() == b.keys()
            for key in a:
                if key in ("row_exp", "rows"):
                    np.testing.assert_array_equal(a[key], b[key], err_msg=key)
                elif not isinstance(a[key], np.ndarray) and key != "n_fb":  # (the verdicts follow the lists)
                    assert a[key] == b[key], key
            ka, sa = pairs(a)
            kb, sb = pairs(b)
            common, ia, ib = np.intersect1d(ka, kb, return_indices=True)
            np.testing.assert_array_equal(sa[ia], sb[ib], err_msg="approximate scores of shared pairs")
            shared.append(len(common) / len(ka))
        print(f"pairs shared with the first widened run: widened {shared[0]:.4f}, 16-bit {shared[1]:.4f}")
        assert shared[0] > 0.9 and shared[1] > 0.9
    finally:
        wide.close()
        kept.close()


def test_hbm_bytes(lib, torch):
    """Borrowed 16-bit device objects hold exactly n*d*4 bytes less than the widened engine; host fp16 objects, uploaded
    into an owned 16-bit buffer, exactly n*d*2 less than the same values uploaded as fp32."""
    from rectools_b200 import B200Ranker, Engine

    rng = np.random.default_rng(2)
    n, d = 12_345, 72
    for dtype in DTYPES:
        t = _catalogue(torch, rng, n, d, dtype)
        for cosine in (False, True):
            wide, kept = _pair(lib, torch, t, cosine)
            try:
                assert wide.info()["hbm_bytes"] - kept.info()["hbm_bytes"] == n * d * 4
            finally:
                wide.close()
                kept.close()
    x16 = rng.standard_normal((n, d)).astype(np.float16)
    for cosine in (False, True):
        e32 = Engine(x16.astype(np.float32), cosine=cosine)
        e16 = Engine(x16, cosine=cosine, objects_dtype=lib.DT_F16, keep_16bit=True)
        try:
            assert e32.info()["hbm_bytes"] - e16.info()["hbm_bytes"] == n * d * 2
            sub = rng.standard_normal((300, d)).astype(np.float32)
            for k in (10, 100, 1025):
                _same(e16.topk(k, subjects=sub), e32.topk(k, subjects=sub), f"host fp16 k={k}")
        finally:
            e32.close()
            e16.close()
    # B200Ranker over numpy fp16 objects: kept by default, widened with keep_16bit=False; same answers
    sub = rng.standard_normal((500, d)).astype(np.float32)
    for distance in ("dot", "cosine", "euclidean"):
        r16 = B200Ranker(distance, sub, x16)
        r32 = B200Ranker(distance, sub, x16, keep_16bit=False)
        diff = r32.engine.info()["hbm_bytes"] - r16.engine.info()["hbm_bytes"]
        assert diff == (0 if distance == "euclidean" else n * d * 2), distance
        for a, b in zip(r16.rank(np.arange(500), k=20), r32.rank(np.arange(500), k=20)):
            np.testing.assert_array_equal(np.asarray(a), np.asarray(b))


def test_group_00_matches_one_engine(lib, torch, main_cat, monkeypatch):
    """A group [0, 0] created with the flag: both members borrow the home matrix; bit for bit one engine's answer."""
    from rectools_b200 import EngineGroup

    monkeypatch.setenv("B200_GROUP_SLICE_ROWS", "100")
    for dtype in DTYPES:
        t = main_cat[dtype]
        for cosine in (False, True):
            wide, kept = _pair(lib, torch, t, cosine)
            grp = EngineGroup(None, cosine=cosine, devices=(0, 0), objects_device_ptr=t.data_ptr(), shape=tuple(t.shape),
                              objects_dtype=_dt(lib, torch, t), keep_16bit=True)
            try:
                info = grp.info()
                assert info["hbm_bytes"] - sum(m["hbm_bytes"] for m in info["members"]) >= 0
                assert all(wide.info()["hbm_bytes"] - m["hbm_bytes"] == N_MAIN * D_MAIN * 4 for m in info["members"])
                rng = np.random.default_rng(4)
                subjects = rng.standard_normal((450, D_MAIN)).astype(np.float32)
                filt = _filter(rng, 450, N_MAIN, full_rows=(2,))
                for k, flags in ((10, 0), (100, 0), (10, lib.Q_FORCE_EXACT), (1025, 0)):
                    g = grp.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, flags=flags)
                    _same(g, kept.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, flags=flags), f"group k={k}")
                    _same(g, wide.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, flags=flags), f"wide k={k}")
            finally:
                grp.close()
                wide.close()
                kept.close()


def test_torch_ranker_keeps_dropped_tensor_alive(torch):
    """`B200TorchRanker` reads a bf16 tensor in place: after the caller drops every reference (and the allocator hands the
    freed blocks of other tensors out again) it still ranks what the widened ranker ranks."""
    from rectools_b200 import B200TorchRanker

    g = torch.Generator().manual_seed(3)
    n, d = 30_000, 64
    users = torch.randn((800, d), generator=g)
    emb = torch.randn((n, d), generator=g).to(torch.bfloat16).cuda()
    ref = B200TorchRanker("dot", "cuda:0", users, emb.clone(), keep_16bit=False)
    ranker = B200TorchRanker("dot", "cuda:0", users, emb)
    assert ref.engine.info()["hbm_bytes"] - ranker.engine.info()["hbm_bytes"] == n * d * 4
    exp = ref.rank(np.arange(800), k=50)
    del emb
    gc.collect()
    junk = [torch.full((n, d), float("nan"), dtype=torch.bfloat16, device="cuda") for _ in range(4)]
    torch.cuda.synchronize()
    got = ranker.rank(np.arange(800), k=50)
    for a, b in zip(got, exp):
        np.testing.assert_array_equal(np.asarray(a), np.asarray(b))
    del junk


@pytest.fixture(scope="module")
def ref():
    if not stage_reference.available():
        pytest.skip("reference package not staged (oracle/_ref)")
    added = stage_reference.add_to_path()
    import rectools  # noqa: F401

    yield
    stage_reference.remove_from_path(added)


@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_similarity_module_bf16(ref, torch, distance):
    """`make_similarity_module()` over bf16 `item_embs`: the default (kept at 16 bits) returns the frame of
    `keep_16bit=False`."""
    from scipy import sparse as sp

    from rectools_b200.integration import make_similarity_module

    n_users, n_tokens, d, k = 2000, 20_001, 64, 10
    g = torch.Generator().manual_seed(9)
    user_embs = torch.randn((n_users, d), generator=g) / d**0.5
    item_embs = (torch.randn((n_tokens, d), generator=g) / d**0.5).to(torch.bfloat16).cuda()
    user_ids = np.random.default_rng(0).permutation(n_users)[:1500]
    rng = np.random.default_rng(1)
    cols = rng.integers(1, n_tokens, size=(len(user_ids), 30))
    rows = np.repeat(np.arange(len(user_ids)), 30)
    ui = sp.csr_matrix((np.ones(cols.size, np.float32), (rows, cols.reshape(-1))), shape=(len(user_ids), n_tokens))
    ui.sum_duplicates()
    ui.data[:] = 1.0
    whitelist = np.arange(1, n_tokens)
    a = make_similarity_module()(distance=distance)._recommend_u2i(  # pylint: disable=protected-access
        user_embs, item_embs, user_ids, k, whitelist, ui)
    b = make_similarity_module(keep_16bit=False)(distance=distance)._recommend_u2i(  # pylint: disable=protected-access
        user_embs, item_embs, user_ids, k, whitelist, ui)
    c = make_similarity_module(keep_16bit=True)(distance=distance)._recommend_u2i(  # pylint: disable=protected-access
        user_embs, item_embs, user_ids, k, whitelist, ui)
    for x, y, z in zip(a, b, c):
        np.testing.assert_array_equal(np.asarray(x), np.asarray(y))
        np.testing.assert_array_equal(np.asarray(x), np.asarray(z))
    assert len(a[1]) == len(user_ids) * k

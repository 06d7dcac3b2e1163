"""GPU: the exhaustive kernels at their edges, against the fp64 oracle in the engine's padded form.

`exact_topk_kernel` + `merge_select_kernel` (path 0), `dense_scores_kernel` + `scores_topk_kernel` (path 3),
`sparse_scores_kernel` (path 2) and `b200_rank_merge` / `b200_rank_merge_certified` are the engine's ground truth: every row
the tensor-core certificate rejects, every tiny call, FORCE_EXACT, k > 128 off the wide mode and every EASE call end here.
The catalogues of tests/exact_cases.py have integer-valued factors, so exact ties sit on every pass boundary, tile, object
split and row chunk, plus planted tie blocks across given ranks and positions.  Every comparison is of the full padded
arrays -- ids, scores, counts and every unfilled slot (-1 / -FLT_MAX) -- in the order (score desc, id asc), with no tie
tolerance, and every call asserts the path it took."""
import numpy as np
import pytest
from scipy import sparse

from oracle.topk_oracle import rank_oracle
from tests import exact_cases as ec

pytestmark = pytest.mark.gpu

K_PATH0 = [1, 31, 32, 33, 63, 64, 65, 100, 128]
K_PATH3 = [129, 159, 160, 161, 1000]


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
    np.testing.assert_array_equal(sc, esc, err_msg=f"{name}: scores")


def _prefix(exp, k, rows=slice(None)):
    """The expectation for a smaller k (and a leading subset of rows): a prefix of the padded rows."""
    ids, sc, cnt = exp
    return ids[rows, :k], sc[rows, :k], np.minimum(cnt[rows], k)


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


# ------------------------------------------------------------------------------------------------ catalogues
@pytest.fixture(scope="module")
def sm_count():
    from rectools_b200 import Engine

    eng = Engine(np.ones((64, 4), np.float32), cosine=False)
    sm = int(eng.info()["sm_count"])
    eng.close()
    return sm


@pytest.fixture(scope="module")
def big(sm_count):
    """{distance: (catalogue, engine with the catalogue's subjects resident, whitelist)} on 300 000 objects."""
    from rectools_b200 import Engine

    out = {}
    for distance in ("dot", "cosine"):
        cat = ec.tie_catalogue(sm_count, cosine=distance == "cosine")
        n = len(cat.objects)
        rng = np.random.default_rng(7)
        wl = np.union1d(np.sort(rng.choice(n - 1, n // 2, replace=False)), [n - 1]).astype(np.int32)
        eng = Engine(cat.objects, cosine=distance == "cosine")
        eng.set_subjects(cat.subjects)
        out[distance] = (cat, eng, wl)
    yield out
    for _, eng, _ in out.values():
        eng.close()


@pytest.fixture(scope="module")
def small():
    """{distance: (objects, subjects)}: 1 100 integer objects (COSINE: pooled rows), 80 subjects, d = 8."""
    rng = np.random.default_rng(11)
    return {
        "dot": (ec.int_matrix(rng, 1_100, 8), ec.int_matrix(rng, 80, 8)),
        "cosine": (ec.pooled_matrix(rng, 1_100, 8, 60), ec.int_matrix(rng, 80, 8)),
    }


# ------------------------------------------------------------------------------------------------ 1. path 0
@pytest.mark.parametrize("with_wl", [False, True])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_path0_pass_and_split_boundaries(lib, big, sm_count, distance, with_wl):
    """FORCE_EXACT over k across the pass boundaries and n_rows across the object-split counts (1 row: the most splits) and
    the 4-rows-per-warp / 32-rows-per-block tails; the planted blocks cross k0 = 32 / 64 / 96 / 128 and split / tile edges."""
    cat, eng, wl = big[distance]
    whitelist = wl if with_wl else None
    n_pos = len(cat.objects) if whitelist is None else len(wl)
    exp = ec.expected_padded(distance, cat.subjects, cat.objects, np.arange(129), 128, None, whitelist)
    zero = exp[0][ec.ZERO_ROW]  # a zero subject: everything ties, the first positions in id order
    np.testing.assert_array_equal(zero, np.arange(128) if whitelist is None else wl[:128])
    for n_rows in (1, 3, 32, 33, 129):
        for k in K_PATH0:
            got = eng.topk(k, subjects=cat.subjects[:n_rows], whitelist=whitelist, flags=lib.Q_FORCE_EXACT)
            st = eng.last_stats
            name = f"{distance} wl={with_wl} rows={n_rows} k={k}"
            assert st["path"] == 0 and st["n_splits"] == ec.exact_splits(n_rows, n_pos, sm_count), (name, st)
            _same(got, _prefix(exp, k, slice(0, n_rows)), name)


# ------------------------------------------------------------------------------------------------ 2. path 3
def _path3_call(big):
    """2 000 rows over 300 000 objects (three 864-row chunks, the last ragged): resident subjects through a permuted row
    map with repeats (the planted and zero rows sit at the chunk edges), a filter in every row, ids >= N included."""
    cat, eng, _ = big["dot"]
    n = len(cat.objects)
    rng = np.random.default_rng(21)
    sids = np.r_[rng.permutation(len(cat.subjects)), rng.integers(0, len(cat.subjects), 500)].astype(np.int64)
    chunk = ec.dense_chunk_rows(n)
    assert chunk == 864
    edges = [0, chunk - 1, chunk, chunk + 1, 2 * chunk - 1, 2 * chunk, 2 * chunk + 1, len(sids) - 1]
    sids[edges] = [5, 4, 2, ec.ZERO_ROW, 1, 3, 6, 5]
    rows = [rng.integers(0, n + 100, rng.integers(0, 300)) for _ in sids]
    for e in edges:  # rows at the chunk edges: part of their planted block (or of the first positions) filtered
        block = next((p["block"] for p in cat.plants if p["row"] == sids[e]), np.arange(200))
        rows[e] = np.r_[rows[e], block[::3], block[:2]]  # (block[:2] twice: duplicate entries)
    return cat, eng, sids, ec.csr_from_rows(rows, n)


@pytest.fixture(scope="module")
def path3_case(big):
    cat, eng, sids, filt = _path3_call(big)
    return cat, eng, sids, filt, ec.expected_padded("dot", cat.subjects, cat.objects, sids, max(K_PATH3), filt)


def test_path3_row_chunks_row_map_and_filter_host_inputs(lib, path3_case):
    cat, eng, sids, filt, exp = path3_case
    for k in K_PATH3:
        got = eng.topk(k, subject_ids=sids, indptr=filt.indptr, indices=filt.indices, flags=lib.Q_FORCE_EXACT)
        assert eng.last_stats["path"] == 3, eng.last_stats
        _same(got, _prefix(exp, k), f"path 3 host k={k}")


def test_path3_row_chunks_row_map_and_filter_device_inputs(lib, path3_case):
    import torch

    cat, eng, sids, filt, exp = path3_case
    dev = torch.device("cuda:0")
    d_sids = torch.from_numpy(sids).to(dev)
    d_ip = torch.from_numpy(filt.indptr.astype(np.int64)).to(dev)
    d_ix = torch.from_numpy(filt.indices.astype(np.int32)).to(dev)
    torch.cuda.synchronize()
    for k in (160, 1000):
        ids = np.full((len(sids), k), 777, np.int32)
        sc = np.full((len(sids), k), 5.0, np.float32)
        cnt = np.full(len(sids), -3, np.int32)
        st = eng.topk_ptrs(len(sids), k, ids.ctypes.data, sc.ctypes.data, cnt.ctypes.data, lib.Q_INPUTS_ON_DEVICE | lib.Q_FORCE_EXACT,
                           subject_ids=d_sids.data_ptr(), indptr=d_ip.data_ptr(), indices=d_ix.data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream)
        assert st["path"] == 3, st
        _same((ids, sc, cnt), _prefix(exp, k), f"path 3 device k={k}")


@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("with_wl", [False, True])
def test_path3_k_up_to_the_catalogue(lib, small, distance, with_wl):
    """k = 1024, 1025 and None (all positions) on a small catalogue, through `B200Ranker.rank_padded`."""
    import rectools_b200 as rb

    objects, subjects = small[distance]
    n = len(objects)
    rng = np.random.default_rng(23)
    wl = np.sort(rng.choice(n, 1_050, replace=False)) if with_wl else None
    filt = ec.csr_from_rows([rng.integers(0, n + 10, rng.integers(0, 40)) for _ in range(70)], n)
    ranker = rb.B200Ranker(distance, subjects, objects)
    sids = np.arange(70)
    for k in (1024, 1025, None):
        _, ids, sc, cnt = ranker.rank_padded(sids, k, filt, wl, flags=lib.Q_FORCE_EXACT)
        assert ranker.last_stats["path"] == 3, ranker.last_stats
        _same((ids, sc, cnt), ec.expected_padded(distance, subjects, objects, sids, k, filt, wl), f"{distance} wl={with_wl} k={k}")


# ------------------------------------------------------------------------------------------------ 3. exhausted rows
def _sparse_rows(rng, n_rows, d, nnz_list=()):
    """CSR subjects: rows with the given nnz first, then random ones; duplicate columns kept, data in halves (-1.5 .. 1.5)."""
    nnz = list(nnz_list) + list(rng.integers(0, 2 * d, n_rows - len(nnz_list)))
    indptr = np.r_[0, np.cumsum(nnz)].astype(np.int64)
    indices = rng.integers(0, d, int(indptr[-1])).astype(np.int32)
    data = (rng.choice([-3, -2, -1, 1, 2, 3], int(indptr[-1])) / 2).astype(np.float32)
    return sparse.csr_matrix((data, indices, indptr), shape=(n_rows, d))


@pytest.mark.parametrize("with_wl", [False, True])
@pytest.mark.parametrize("path", [0, 2, 3])
def test_exhausted_rows_keep_their_padding(lib, path, with_wl):
    """Filters that leave 0, 1, 31, 32, 33, k - 1, k and k + 1 survivors: rows run out before a later pass, and every slot
    past the count is -1 / -FLT_MAX even though the previous call left real results in the engine's output buffers."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(31 + path)
    n, d = 5_000, 64
    objects = ec.int_matrix(rng, n, d)
    wl = np.sort(rng.choice(n, 3_000, replace=False)).astype(np.int32) if with_wl else None
    k = 200 if path == 3 else 100
    survivors = [0, 1, 31, 32, 33, k - 1, k, k + 1, 64, 65, 96]
    n_rows = 40
    filt = ec.filter_keeping(rng, n, survivors + [n] * (n_rows - len(survivors)), candidates=wl)
    eng = Engine(objects, cosine=False)
    if path == 2:
        subjects = _sparse_rows(rng, n_rows, d, [0, 1, 300])
        kw = dict(sparse_subjects=subjects)
    else:
        subjects = ec.int_matrix(rng, n_rows, d)
        kw = dict(subjects=subjects, flags=lib.Q_FORCE_EXACT)
    eng.topk(k, whitelist=wl, **kw)  # fills the output buffers
    got = eng.topk(k, indptr=filt.indptr, indices=filt.indices, whitelist=wl, **kw)
    assert eng.last_stats["path"] == path, eng.last_stats
    exp = ec.expected_padded("dot", subjects, objects, np.arange(n_rows), k, filt, wl)
    assert exp[2][: len(survivors)].tolist() == [min(s, k) for s in survivors]
    _same(got, exp, f"path {path} wl={with_wl}")
    eng.close()


# ------------------------------------------------------------------------------------------------ 4. whitelist / filter edges
@pytest.mark.parametrize("k", [50, 200])
@pytest.mark.parametrize("wl_kind", ["len1", "len31", "len33", "with_last", "none"])
def test_whitelist_and_filter_edges(lib, small, k, wl_kind):
    """Whitelists of 1, 31 and 33 positions (shorter than k) and one holding object N - 1; filter ids >= N, duplicate
    entries, entries outside the whitelist, empty rows and a row that filters every whitelisted object."""
    from rectools_b200 import Engine

    objects, subjects = small["dot"]
    n = len(objects)
    rng = np.random.default_rng(41)
    wl = {
        "len1": np.array([n - 1]), "len31": np.sort(rng.choice(n, 31, replace=False)), "len33": np.sort(rng.choice(n, 33, replace=False)),
        "with_last": np.union1d(rng.choice(n - 1, 400, replace=False), [n - 1]), "none": None,
    }[wl_kind]
    pos = np.arange(n) if wl is None else wl
    rows = [
        np.array([], np.int64),  # empty
        pos,  # every whitelisted object
        np.r_[pos[:5], pos[:5], pos[3:9]],  # duplicates
        np.r_[n, n + 1, n + 1000, pos[-1]],  # ids >= N
        np.setdiff1d(np.arange(0, n, 2), pos)[:300],  # outside the whitelist only
        np.r_[pos[::2], np.arange(n, n + 20)],
    ]
    rows += [rng.integers(0, n + 5, rng.integers(0, 30)) for _ in range(34)]
    filt = ec.csr_from_rows(rows, n)
    eng = Engine(objects, cosine=False)
    wl32 = None if wl is None else wl.astype(np.int32)
    got = eng.topk(k, subjects=subjects[:40], indptr=filt.indptr, indices=filt.indices, whitelist=wl32, flags=lib.Q_FORCE_EXACT)
    k_out = min(k, len(pos))
    assert eng.last_stats["path"] == (3 if k_out > 128 else 0), eng.last_stats
    exp = ec.expected_padded("dot", subjects, objects, np.arange(40), k, filt, wl)
    assert exp[2][1] == 0 and exp[2][0] == k_out
    _same(got, exp, f"wl={wl_kind} k={k}")
    eng.close()


# ------------------------------------------------------------------------------------------------ 5. d edges
@pytest.mark.parametrize("d", [1, 2, 63, 64, 65, 127, 129, 320])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
def test_d_edges_of_the_exhaustive_kernels(lib, distance, d):
    """d across the 64-wide k steps of exact_topk_kernel (EX_DK) and dense_scores_kernel (DS_DK): path 0 and path 3."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(d)
    n = 2_000
    objects = ec.pooled_matrix(rng, n, d, 90) if distance == "cosine" else ec.int_matrix(rng, n, d)
    subjects = ec.int_matrix(rng, 40, d)
    filt = ec.csr_from_rows([rng.integers(0, n, rng.integers(0, 50)) for _ in range(40)], n)
    eng = Engine(objects, cosine=distance == "cosine")
    for k, path in ((70, 0), (150, 3)):
        got = eng.topk(k, subjects=subjects, indptr=filt.indptr, indices=filt.indices, flags=lib.Q_FORCE_EXACT)
        assert eng.last_stats["path"] == path, eng.last_stats
        _same(got, ec.expected_padded(distance, subjects, objects, np.arange(40), k, filt), f"{distance} d={d} k={k}")
    eng.close()


# ------------------------------------------------------------------------------------------------ 6. extreme values
def _rank_vs_oracle(distance, subjects, objects, k, filt=None, name=""):
    import rectools_b200 as rb

    ranker = rb.B200Ranker(distance, subjects, objects)
    sids = np.arange(len(subjects))
    got = ranker.rank(sids, k, filt)
    exp = rank_oracle(distance, subjects, objects, sids, k, filt, accum="f64")
    for g, e, what in zip(got, exp, ("subjects", "ids", "scores")):
        np.testing.assert_array_equal(np.asarray(g), np.asarray(e), err_msg=f"{name}: {what}")
    return ranker


@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("kind", ["overflow", "subnormal"])
def test_extreme_magnitudes(lib, distance, kind):
    """Factors near 1e20, whose dots round to +inf (ties among infinities) or -inf (dropped, as the reference strips them);
    products in the subnormal range, and subnormal factors.  Path 0 (k = 100, four passes) and path 3 (k = 200)."""
    rng = np.random.default_rng(51)
    n, d = 1_500, 8
    objects = ec.int_matrix(rng, n, d)
    subjects = ec.int_matrix(rng, 24, d)
    if kind == "overflow":  # (COSINE scores are at most |u|: huge, finite)
        objects[rng.choice(n, 300, replace=False)] *= np.float32(1e20)
        subjects[:12] *= np.float32(1e20)
    else:
        objects[rng.choice(n, 600, replace=False)] *= np.float32(1e-20)
        objects[rng.choice(n, 100, replace=False)] *= np.float32(1e-39)  # fp32 subnormals
        subjects[:12] *= np.float32(1e-20)
    filt = ec.csr_from_rows([rng.integers(0, n, 20) for _ in range(24)], n)
    sc = ec.engine_scores(subjects, objects, distance == "cosine")
    if distance == "dot" and kind == "overflow":
        assert np.isposinf(sc).sum(axis=1).max() > 40 and np.isneginf(sc).any()
    elif distance == "dot":
        assert ((sc != 0) & (np.abs(sc) < np.finfo(np.float32).tiny)).sum() > 100
    for k, path in ((100, 0), (200, 3)):
        ranker = _rank_vs_oracle(distance, subjects, objects, k, filt, f"{kind} {distance} k={k}")
        assert ranker.last_stats["path"] == path, ranker.last_stats


def test_real_scores_at_the_sentinel(lib):
    """d = 1, real scores of exactly -FLT_MAX and its neighbour: the kernels return them (only -inf is dropped), the
    wrapper strips them from the end of the row as the reference does (rank_implicit.py:107-118)."""
    from rectools_b200 import Engine

    lo = np.float32(ec.neginf_score())
    objects = np.array([[-ec.FLT_MAX], [1.0], [lo], [-1.0], [ec.FLT_MAX], [np.nextafter(lo, np.float32(0))], [0.0]], np.float32)
    subjects = np.array([[1.0], [-1.0], [0.0], [2.0]], np.float32)  # (row 3: 2 * -FLT_MAX = -inf)
    eng = Engine(objects, cosine=False)
    ids, sc, cnt = eng.topk(7, subjects=subjects)
    assert eng.last_stats["path"] == 0
    assert cnt.tolist() == [7, 7, 7, 4]
    assert ids[0].tolist() == [4, 1, 6, 3, 5, 2, 0] and sc[0, -1] == -ec.FLT_MAX and sc[0, -2] == lo
    eng.close()
    ranker = _rank_vs_oracle("dot", subjects, objects, 7, name="sentinel")
    _, ids, sc, cnt = ranker.rank_padded(np.arange(4), 7)
    assert cnt.tolist() == [5, 6, 7, 4]
    assert (ids[0, 5:] == -1).all() and (sc[0, 5:] == -ec.FLT_MAX).all()


# ------------------------------------------------------------------------------------------------ 7. sparse subjects
@pytest.mark.parametrize("with_wl", [False, True])
@pytest.mark.parametrize("n_obj", [4_000, 4_001, 4_002, 4_003])
def test_sparse_subjects(lib, n_obj, with_wl):
    """Rows of 0, 1, 255, 256, 257 and 1 000 non-zeros (duplicate columns left unsummed, weights +-0.5 .. +-1.5), n_obj % 4
    in {0, 1, 2, 3} (the float4 and scalar branches), with and without a whitelist, k across the pass boundaries."""
    import rectools_b200 as rb

    rng = np.random.default_rng(n_obj)
    d = 300
    objects = ec.int_matrix(rng, n_obj, d)
    csr = _sparse_rows(rng, 40, d, [0, 1, 255, 256, 257, 1_000])
    assert not csr.has_canonical_format  # duplicates
    wl = np.sort(rng.choice(n_obj, n_obj // 2 + 3, replace=False)) if with_wl else None
    filt = ec.csr_from_rows([rng.integers(0, n_obj + 9, rng.integers(0, 60)) for _ in range(40)], n_obj)
    ranker = rb.B200Ranker("dot", csr, objects)
    sids = np.arange(40)
    for k in (1, 32, 33, 200, None):
        _, ids, sc, cnt = ranker.rank_padded(sids, k, filt, wl)
        assert ranker.last_stats["path"] == 2, ranker.last_stats
        _same((ids, sc, cnt), ec.expected_padded("dot", csr, objects, sids, k, filt, wl), f"n_obj={n_obj} wl={with_wl} k={k}")


def test_sparse_subjects_row_chunks(lib):
    """n_pos = 270 000, d = 64 != N, 2 500 rows: three 994-row chunks of score rows, the filter offset per chunk."""
    from rectools_b200 import Engine

    rng = np.random.default_rng(61)
    n, d = 270_000, 64
    objects = ec.int_matrix(rng, n, d)
    csr = _sparse_rows(rng, 2_500, d, [0, 300])
    assert ec.sparse_chunk_rows(n) == 994
    filt = ec.csr_from_rows([rng.integers(0, n + 50, rng.integers(0, 100)) for _ in range(2_500)], n)
    eng = Engine(objects, cosine=False)
    for k in (33,):
        got = eng.topk(k, sparse_subjects=csr, indptr=filt.indptr, indices=filt.indices)
        assert eng.last_stats["path"] == 2, eng.last_stats
        _same(got, ec.expected_padded("dot", csr, objects, np.arange(2_500), k, filt), f"sparse chunks k={k}")
    eng.close()


# ------------------------------------------------------------------------------------------------ 8. invariance
@pytest.mark.parametrize("k", [100, 200])
def test_a_rows_result_does_not_depend_on_the_call_shape(lib, big, monkeypatch, k):
    """Bit-identical rows: ranked alone (the most object splits) and inside a batch, under B200_CHUNK_ROWS, with host and
    device inputs, and with subject_ids in either order."""
    import torch

    cat, eng, wl = big["dot"]
    n_rows = 129
    flags = lib.Q_FORCE_EXACT
    path = 0 if k <= 128 else 3
    base = eng.topk(k, subjects=cat.subjects[:n_rows], whitelist=wl, flags=flags)
    assert eng.last_stats["path"] == path
    for r in (0, 5, 6, 8, 9, ec.ZERO_ROW, 77, 128):
        one = eng.topk(k, subjects=cat.subjects[r : r + 1], whitelist=wl, flags=flags)
        for a, b in zip(one, base):
            np.testing.assert_array_equal(_bits(a[0]), _bits(b[r]), err_msg=f"row {r} alone")
    sids = np.arange(n_rows, dtype=np.int64)
    for order in (sids, sids[::-1].copy()):
        got = eng.topk(k, subject_ids=order, whitelist=wl, flags=flags)
        for a, b in zip(got, base):
            np.testing.assert_array_equal(_bits(a), _bits(b[order]), err_msg="subject_ids order")
    monkeypatch.setenv("B200_CHUNK_ROWS", "256")
    got = eng.topk(k, subjects=np.tile(cat.subjects[:n_rows], (5, 1)), whitelist=wl, flags=flags)
    for a, b in zip(got, base):
        np.testing.assert_array_equal(_bits(a), _bits(np.concatenate([b] * 5)), err_msg="B200_CHUNK_ROWS")
    monkeypatch.delenv("B200_CHUNK_ROWS")
    dev = torch.device("cuda:0")
    d_sub = torch.from_numpy(cat.subjects[:n_rows].copy()).to(dev)
    d_wl = torch.from_numpy(wl).to(dev)
    torch.cuda.synchronize()
    k_out = min(k, len(wl))
    ids, sc, cnt = np.empty((n_rows, k_out), np.int32), np.empty((n_rows, k_out), np.float32), np.empty(n_rows, np.int32)
    st = eng.topk_ptrs(n_rows, k, ids.ctypes.data, sc.ctypes.data, cnt.ctypes.data, flags | lib.Q_INPUTS_ON_DEVICE,
                       subjects=d_sub.data_ptr(), whitelist=d_wl.data_ptr(), n_whitelist=len(wl),
                       stream=torch.cuda.current_stream().cuda_stream)
    assert st["path"] == path
    for a, b in zip((ids, sc, cnt), base):
        np.testing.assert_array_equal(_bits(a), _bits(b), err_msg="device inputs")


# ------------------------------------------------------------------------------------------------ 9. the merge
def _merge(lib, ids, sc, cnt, k, bounds=None, packed=False, n_rows=None):
    """b200_rank_merge (bounds None) / b200_rank_merge_certified on device copies of numpy lists [n_lists, n_rows, L]; packed:
    one buffer per list [ids n*k | score bits n*k | counts n | bound bits n] (sharded.Packed).  Outputs start as garbage."""
    import torch

    dev = torch.device("cuda:0")
    n_lists, n, L = ids.shape
    n_rows = n if n_rows is None else n_rows
    o_ids = torch.full((max(n, 1), k), 12345, dtype=torch.int32, device=dev)
    o_sc = torch.full((max(n, 1), k), 3.5, dtype=torch.float32, device=dev)
    o_cnt = torch.full((max(n, 1),), -9, dtype=torch.int32, device=dev)
    fail_rows = torch.full((max(n, 1),), -7, dtype=torch.int32, device=dev)
    fail_count = torch.zeros((1,), dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    if packed:
        buf = np.concatenate([ids.reshape(n_lists, -1), sc.reshape(n_lists, -1).view(np.int32), cnt, bounds.view(np.int32)], axis=1)
        g = torch.from_numpy(np.ascontiguousarray(buf)).to(dev)
        base, stride = g.data_ptr(), buf.shape[1]
        ptrs = (base, base + 4 * n * L, base + 8 * n * L, base + 8 * n * L + 4 * n)
    else:
        keep = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (ids, sc, cnt) + ((bounds,) if bounds is not None else ())]
        ptrs, stride = tuple(t.data_ptr() for t in keep), 0
    torch.cuda.synchronize()
    h = lib.load()
    if bounds is None:
        lib.check(h.b200_rank_merge(0, stream, n_lists, n_rows, k, *ptrs[:3], o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr()))
    else:
        lib.check(h.b200_rank_merge_certified(0, stream, n_lists, n_rows, k, *ptrs, stride, o_ids.data_ptr(), o_sc.data_ptr(),
                                              o_cnt.data_ptr(), fail_rows.data_ptr(), fail_count.data_ptr()))
    torch.cuda.synchronize()
    return o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy(), fail_rows.cpu().numpy()[: int(fail_count.item())]


@pytest.mark.parametrize("k", [1, 10, 31, 32, 33, 100, 1000])
@pytest.mark.parametrize("n_lists", [1, 2, 3, 8, 40])
def test_merge(lib, n_lists, k):
    rng = np.random.default_rng(n_lists * 1000 + k)
    ids, sc, cnt = ec.merge_case(rng, n_lists, 37, k)
    got = _merge(lib, ids, sc, cnt, k)
    _same(got[:3], ec.expected_merge(ids, sc, cnt, k)[:3], f"merge lists={n_lists} k={k}")


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("k", [1, 10, 32])
@pytest.mark.parametrize("n_lists", [3, 40])
def test_merge_certified(lib, n_lists, k, packed):
    """The certificate: a bound equal to the k-th merged score rejects, one ulp below accepts; all bounds -inf accept a
    short row; a finite bound rejects a row with fewer than k entries; more than 32 lists; fail_rows is the expected set."""
    rng = np.random.default_rng(n_lists * 100 + k)
    n_rows = 45
    ids, sc, cnt = ec.merge_case(rng, n_lists, n_rows, k)
    cnt[:, 2:6] = 0
    cnt[0, 2] = cnt[0, 3] = k  # rows 2 and 3: k entries in list 0
    cnt[n_lists - 1, 4] = cnt[n_lists - 1, 5] = max(0, k - 1)  # rows 4 and 5: short
    ids[0, 2:4, :k] = np.arange(k) * 3
    ids[-1, 4:6, :k] = np.arange(k) * 5 + 1
    m_ids, m_sc, m_cnt, _ = ec.expected_merge(ids, sc, cnt, k)
    bounds = np.where(rng.random((n_lists, n_rows)) < 0.5, -np.inf, rng.integers(-4, 4, (n_lists, n_rows))).astype(np.float32)
    bounds[:, 0] = -np.inf  # row 0: no entries, no bound
    bounds[:, 2:6] = -np.inf
    bounds[n_lists // 2, 2] = m_sc[2, k - 1]  # == the k-th score: reject
    bounds[n_lists - 1, 3] = np.nextafter(m_sc[3, k - 1], np.float32(-np.inf))  # one ulp below: accept
    bounds[0, 5] = np.float32(-1e30)  # short row, finite bound: reject (row 4: all -inf, accept)
    exp = ec.expected_merge(ids, sc, cnt, k, bounds)
    assert 2 in exp[3] and 3 not in exp[3] and 4 not in exp[3] and 5 in exp[3] and 0 not in exp[3]
    got = _merge(lib, ids, sc, cnt, k, bounds, packed)
    _same(got[:3], exp[:3], f"certified lists={n_lists} k={k} packed={packed}")
    assert len(np.unique(got[3])) == len(got[3]), "duplicate fail rows"
    np.testing.assert_array_equal(np.sort(got[3]), exp[3])


def test_merge_refusals(lib):
    rng = np.random.default_rng(3)
    ids, sc, cnt = ec.merge_case(rng, 2, 4, 33)
    with pytest.raises(NotImplementedError):
        _merge(lib, ids, sc, cnt, 33, np.full((2, 4), -np.inf, np.float32))
    for bounds in (None, np.full((2, 4), -np.inf, np.float32)):
        o_ids, o_sc, o_cnt, fails = _merge(lib, ids[:, :, :32], np.ascontiguousarray(sc[:, :, :32]), np.minimum(cnt, 32), 32, bounds,
                                           n_rows=0)
        assert (o_ids == 12345).all() and (o_sc == 3.5).all() and (o_cnt == -9).all() and len(fails) == 0  # n_rows = 0: untouched

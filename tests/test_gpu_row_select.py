"""GPU: stored rows as score rows (path 4, `row_select_kernel`, rectools_b200/csrc/row_select.cuh) and EASE item-to-item
through `install()`.

The engine holds a square fp32 matrix W (an EASE weight) and ranks rows of it in place: target t scores object j with
W[t, j].  Every comparison is of the full padded arrays -- ids, score bits, counts and every unfilled slot (-1 / -FLT_MAX):
  * against a numpy restatement: the row's values at the call's positions, filtered objects, -inf and NaN dropped, ordered
    by (score desc, id asc) with -0 == +0;
  * against an independent route of the engine: objects W^T ranked with one-hot sparse subjects e_t (path 2), whose
    fp64-accumulated score fp32(1 * W[t, j]) is W[t, j] -- except that it turns -0 into +0, so score bits are compared
    with -0 read as +0 there.
k runs across the shared-memory capacity S of the survivors' sort up to the whole catalogue."""
import numpy as np
import pytest
from scipy import sparse

from oracle import stage_reference
from tests import exact_cases as ec

pytestmark = pytest.mark.gpu

S = 12288  # LK_SMEM_PAIRS (rectools_b200/csrc/sizes.h)
N = 13_000  # items: n_pos > S + 1 with and without the whitelist
FMAX = np.finfo(np.float32).max
TINY = np.finfo(np.float32).tiny


def _weights(seed=0):
    """EASE-shaped fp32 weights with planted special values and ties across the order key's digits."""
    rng = np.random.default_rng(seed)
    w = (rng.standard_normal((N, N), dtype=np.float32) * 0.01).astype(np.float32)
    np.fill_diagonal(w, 0.0)
    specials = np.array([0.0, -0.0, -np.inf, np.nan, FMAX, -FMAX, TINY / 4, -TINY / 4, TINY, np.inf], np.float32)
    for r in range(0, 40):  # every target row below gets a share of them
        cols = rng.choice(N, 300, replace=False)
        w[r, cols] = rng.choice(specials, 300)
    # rows 5 .. 9: values of consecutive floats around digit boundaries of the order key, hundreds of copies each
    bases = np.array([0x3C23D70A, 0x3C23D700, 0x3C2400FF, 0xBC23D70A, 0x3C000000, 0x00000001], np.uint32)
    vals = np.concatenate([(b + np.arange(-3, 4, dtype=np.int64)).astype(np.uint32) for b in bases]).view(np.float32)
    w[5:10] = rng.choice(vals, (5, N))
    w[10] = -0.0  # one tie over the whole row, of -0
    w[11, ::2] = 0.0
    w[12] = -np.inf  # nothing to rank
    w[13] = np.nan
    return w


@pytest.fixture(scope="module")
def case():
    from rectools_b200 import Engine

    w = _weights()
    eng = Engine(w, cosine=False)
    yield w, eng
    eng.close()


def _filter(rng, n_rows):
    """Filter rows with ids >= N and repeated ids; row 3 filters everything, row 4 all but 300 objects."""
    rows = [np.sort(rng.integers(0, N + 500, rng.integers(0, 2_000))) for _ in range(n_rows)]
    rows[1] = np.sort(np.r_[rows[1], rows[1][:50]])  # repeated ids count once
    rows[3] = np.arange(N)
    rows[4] = np.delete(np.arange(N), rng.choice(N, 300, replace=False))
    return ec.csr_from_rows(rows, N)


def _expected(w, targets, k_out, filt=None, wl=None):
    """numpy restatement of path 4: padded (ids, scores, counts)."""
    pos_ids = np.arange(N) if wl is None else np.asarray(wl, np.int64)
    ids = np.full((len(targets), k_out), -1, np.int32)
    sc = np.full((len(targets), k_out), -FMAX, np.float32)
    cnt = np.zeros(len(targets), np.int32)
    for r, t in enumerate(targets):
        vals = w[t, pos_ids]
        keep = vals > -np.inf  # (False for NaN)
        if filt is not None:
            keep &= ~np.isin(pos_ids, filt.indices[filt.indptr[r]:filt.indptr[r + 1]])
        i, v = pos_ids[keep], vals[keep]
        order = np.lexsort((i, -v.astype(np.float64)))[:k_out]  # (score desc, id asc); -0 == +0 as float comparisons
        c = len(order)
        ids[r, :c], sc[r, :c], cnt[r] = i[order], v[order], c
    return ids, sc, cnt


def _bits_same(got, exp, name, zero_sign=False):
    ids, sc, cnt = got
    eids, esc, ecnt = exp
    assert ids.shape == eids.shape, f"{name}: shape {ids.shape} vs {eids.shape}"
    np.testing.assert_array_equal(cnt, ecnt, err_msg=f"{name}: counts")
    np.testing.assert_array_equal(ids, eids, err_msg=f"{name}: ids")
    if zero_sign:  # path 2 accumulates from +0: -0 comes back as +0
        sc, esc = sc + np.float32(0), esc + np.float32(0)
    np.testing.assert_array_equal(np.ascontiguousarray(sc).view(np.int32), np.ascontiguousarray(esc).view(np.int32),
                                  err_msg=f"{name}: score bits")


def _prefix(exp, k):
    ids, sc, cnt = exp
    return ids[:, :k], sc[:, :k], np.minimum(cnt, k)


KS = [1, 10, 100, 1024, 1025, S - 1, S, S + 1, "n_pos", None]


@pytest.mark.parametrize("with_wl", [False, True])
def test_against_numpy_and_path_2(case, with_wl):
    """k = 1 .. the whole catalogue, with and without a whitelist, filters with out-of-range and repeated ids and an
    everything-filtered row, repeated targets, planted special values and ties."""
    import rectools_b200 as rb
    from rectools_b200 import Engine

    w, eng = case
    rng = np.random.default_rng(7)
    targets = np.r_[np.arange(14), rng.integers(0, N, 18), [5, 5, 0, 13]].astype(np.int64)
    wl = np.sort(rng.choice(N, N - 500, replace=False)) if with_wl else None
    n_pos = N if wl is None else len(wl)
    filt = _filter(rng, len(targets))
    full = _expected(w, targets, n_pos, filt, wl)
    assert full[2][3] == 0 and full[2][12] == 0 and full[2][13] == 0  # everything filtered, all -inf, all NaN
    ranker = rb.B200Ranker("dot", np.zeros((1, N), np.float32), w, engine=eng)
    # the independent route: W^T as objects, one-hot CSR subjects (path 2)
    eng_t = Engine(np.ascontiguousarray(w.T), cosine=False)
    onehot = sparse.csr_matrix((np.ones(len(targets), np.float32), targets, np.arange(len(targets) + 1)), shape=(len(targets), N))
    for k in KS:
        kk = n_pos if k == "n_pos" else k
        k_out = n_pos if kk is None else kk
        _, ids, sc, cnt = ranker.rank_object_rows_padded(targets, kk, filt, wl)
        st = ranker.last_stats
        assert (st["path"], st["k_out"], st["n_launches"], st["n_chunks"]) == (4, k_out, 1, 1), st
        assert st["ms_select"] > 0
        name = f"wl={with_wl} k={k}"
        _bits_same((ids, sc, cnt), _prefix(full, k_out), name)
        got_t = eng_t.topk(k_out, sparse_subjects=onehot, indptr=filt.indptr, indices=filt.indices,
                           whitelist=None if wl is None else wl.astype(np.int32))
        assert eng_t.last_stats["path"] == 2
        _bits_same((ids, sc, cnt), got_t, name + " vs path 2", zero_sign=True)
    eng_t.close()
    # the flat triplet of the reference's i2i (ease.py:183-188)
    t, i, s = ranker.rank_object_rows(targets[:3], 7, None, wl)
    e = _expected(w, targets[:3], 7, None, wl)
    np.testing.assert_array_equal(t, np.repeat(targets[:3], 7))
    np.testing.assert_array_equal(i, e[0].reshape(-1))
    np.testing.assert_array_equal(s, e[1].reshape(-1))


@pytest.mark.parametrize("device_io", [False, True])
def test_three_row_chunks(case, monkeypatch, device_io):
    """600 rows in chunks of 256 (B200_CHUNK_ROWS), host and device inputs / outputs, k inside and above S."""
    import torch

    from rectools_b200 import _lib

    w, eng = case
    rng = np.random.default_rng(11)
    targets = rng.integers(0, N, 600).astype(np.int64)
    wl = np.sort(rng.choice(N, N - 100, replace=False)).astype(np.int32)
    filt = _filter(rng, len(targets))
    monkeypatch.setenv("B200_CHUNK_ROWS", "256")
    for k in (10, S + 1):
        exp = _expected(w, targets, k, filt, wl)
        if not device_io:
            got = eng.topk(k, object_rows=targets, indptr=filt.indptr, indices=filt.indices, whitelist=wl)
        else:
            dev = torch.device("cuda", 0)
            t_rows = torch.from_numpy(targets).to(dev)
            t_ip = torch.from_numpy(filt.indptr.astype(np.int64)).to(dev)
            t_ix = torch.from_numpy(filt.indices.astype(np.int32)).to(dev)
            t_wl = torch.from_numpy(wl).to(dev)
            o_ids = torch.empty((600, k), dtype=torch.int32, device=dev)
            o_sc = torch.empty((600, k), dtype=torch.float32, device=dev)
            o_cnt = torch.empty(600, dtype=torch.int32, device=dev)
            eng.topk_ptrs(600, k, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(),
                          _lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE, object_rows=t_rows.data_ptr(), indptr=t_ip.data_ptr(),
                          indices=t_ix.data_ptr(), whitelist=t_wl.data_ptr(), n_whitelist=len(wl))
            torch.cuda.synchronize()
            got = (o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy())
        st = eng.last_stats
        assert (st["path"], st["n_chunks"], st["n_launches"]) == (4, 3, 3), st
        _bits_same(got, exp, f"device_io={device_io} k={k}")


def test_refusals(case):
    from rectools_b200 import Engine, _lib

    w, eng = case
    rows = np.array([0, 1], np.int64)
    with pytest.raises(ValueError, match="object_rows"):
        eng.topk(5, object_rows=np.array([0, N], np.int64))  # out of range (host input)
    with pytest.raises(ValueError, match="object_rows"):
        eng.topk(5, object_rows=np.array([-1], np.int64))
    with pytest.raises(NotImplementedError):
        eng.topk(5, object_rows=rows, flags=_lib.Q_FORCE_TC)
    q = _lib.Query()  # object_rows together with subject_ids, straight through the C ABI
    ids, sc, cnt = np.empty((2, 5), np.int32), np.empty((2, 5), np.float32), np.empty(2, np.int32)
    q.object_rows, q.subject_ids, q.n_rows, q.k = rows.ctypes.data, rows.ctypes.data, 2, 5
    q.out_ids, q.out_scores, q.out_counts = ids.ctypes.data, sc.ctypes.data, cnt.ctypes.data
    with pytest.raises(ValueError, match="excludes"):
        eng.topk_raw(q)
    small = np.random.default_rng(1).standard_normal((50, 50)).astype(np.float32)
    rect = Engine(small[:, :20], cosine=False)
    with pytest.raises(ValueError, match="d == n_objects"):
        rect.topk(5, object_rows=rows)
    cos = Engine(small, cosine=True)
    with pytest.raises(NotImplementedError, match="COSINE"):
        cos.topk(5, object_rows=rows)
    off = Engine(small, cosine=False, id_offset=100)
    with pytest.raises(NotImplementedError, match="id offset"):
        off.topk(5, object_rows=rows)
    ok = Engine(small, cosine=False)
    # shared thresholds are refused as unsupported even when the call has more rows than the engine shares thresholds for
    import torch

    pub, peer = (torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(2))
    shared = Engine(small, cosine=False)
    shared.peer_attach(pub, [peer])
    with pytest.raises(NotImplementedError, match="SHARED_THRESHOLDS"):
        shared.topk(5, object_rows=rows, flags=_lib.Q_SHARED_THRESHOLDS)
    shared.close()
    ids, sc, cnt = ok.topk(5, object_rows=rows)
    _bits_same((ids, sc, cnt), _small_expected(small, rows, 5), "small")
    for e in (rect, cos, off, ok):
        e.close()


def _small_expected(w, rows, k):
    out_i, out_s = [], []
    for t in rows:
        o = np.lexsort((np.arange(len(w)), -w[t].astype(np.float64)))[:k]
        out_i.append(o)
        out_s.append(w[t, o])
    return np.array(out_i, np.int32), np.array(out_s, np.float32), np.full(len(rows), k, np.int32)


# ------------------------------------------------------------------------------------------------ EASE through install()
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


def _same_i2i(exp_df, got_df, weight_score):
    """Same frame up to the order inside tie groups: target column, scores and ranks equal; ids equal wherever the scores
    differ, every tie group equal as a set -- except a group cut off at the end of a target's list, whose ids need only
    carry that score (the reference takes an arbitrary subset of such a group)."""
    assert list(exp_df.columns) == list(got_df.columns)
    assert [str(t) for t in exp_df.dtypes] == [str(t) for t in got_df.dtypes]
    np.testing.assert_array_equal(exp_df["target_item_id"].to_numpy(), got_df["target_item_id"].to_numpy())
    np.testing.assert_array_equal(exp_df["score"].to_numpy(), got_df["score"].to_numpy())
    if "rank" in exp_df:
        np.testing.assert_array_equal(exp_df["rank"].to_numpy(), got_df["rank"].to_numpy())
    tgt, sc = got_df["target_item_id"].to_numpy(), got_df["score"].to_numpy()
    ei, gi = exp_df["item_id"].to_numpy(), got_df["item_id"].to_numpy()
    bounds = np.flatnonzero((tgt[1:] != tgt[:-1]) | (sc[1:] != sc[:-1])) + 1
    starts, ends = np.r_[0, bounds], np.r_[bounds, len(sc)]
    for a, b in zip(starts, ends):
        if b - a == 1:
            assert ei[a] == gi[a]
        elif b == len(sc) or tgt[b] != tgt[a]:
            assert all(weight_score(tgt[a], i) == sc[a] for i in gi[a:b])
        else:
            assert set(ei[a:b]) == set(gi[a:b])


def test_ease_recommend_to_items_through_install(ref):
    from rectools.models import EASEModel

    import rectools_b200
    from rectools_b200 import integration
    from tests.ref_models import synthetic_dataset

    dataset = synthetic_dataset(4000, 1500, 20, seed=6)
    model = EASEModel(regularization=300.0).fit(dataset)
    assert model.weight.dtype == np.float32 and model.weight.flags.c_contiguous
    items = dataset.item_id_map.external_ids
    targets = np.r_[items[::5], items[:3]]
    wl = items[::4]
    calls = {
        "filter_itself": lambda: model.recommend_to_items(targets, dataset, k=10),
        "keep_itself": lambda: model.recommend_to_items(targets, dataset, k=10, filter_itself=False),
        "whitelist": lambda: model.recommend_to_items(targets, dataset, k=25, items_to_recommend=wl),
        "whitelist_keep": lambda: model.recommend_to_items(targets, dataset, k=25, filter_itself=False, items_to_recommend=wl,
                                                           add_rank_col=False),
        "all_items": lambda: model.recommend_to_items(targets[:50], dataset, k=len(items)),
    }
    expected = {name: fn() for name, fn in calls.items()}
    to_int = dataset.item_id_map.convert_to_internal

    def weight_score(target_ext, item_ext):
        return model.weight[to_int([target_ext])[0], to_int([item_ext])[0]]

    rectools_b200.install(device=0)
    try:
        u2i = model.recommend(dataset.user_id_map.external_ids[:100], dataset, k=5, filter_viewed=True)
        assert len(u2i) == 500
        for name, fn in calls.items():
            got = fn()
            eng = next(iter(integration._ENGINE_CACHE.values()))  # pylint: disable=protected-access
            assert eng.last_stats["path"] == 4, (name, eng.last_stats)
            _same_i2i(expected[name], got, weight_score)
        # u2i and i2i share the one engine of the weight matrix
        assert len(integration._ENGINE_CACHE) == 1  # pylint: disable=protected-access
    finally:
        rectools_b200.uninstall()

"""GPU: the wide mode for 128 < k <= 1024 -- one tensor-core pass with long append lists, the large-k re-score, row chunks
that bound the candidate buffers, and the exhaustive re-rank of a row list for whatever the pass could not certify.

Every call is compared with the exhaustive fp64 oracle (ids exactly, scores within rtol 3e-7); the statistics must show the
path taken (path 1, wide 1).  Two-stage candidate generation is the workload this serves: `CandidateGenerator` asks the
first-stage model for a few hundred items per user."""
import numpy as np
import pytest
from scipy import sparse

from oracle.topk_oracle import implicit_topk, neginf_score
from tests.helpers import synth_factors, synth_viewed_csr
from tests.tc_reference import Catalogue, check_snapshot

pytestmark = pytest.mark.gpu

N_ROWS, N_OBJ, D = 3_000, 60_000, 64


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


@pytest.fixture(scope="module")
def data():
    u, i = synth_factors(N_ROWS, N_OBJ, D, seed=31)
    csr = synth_viewed_csr(N_ROWS, N_OBJ, 100, seed=33)
    wl = np.sort(np.random.default_rng(34).choice(N_OBJ, N_OBJ // 2, replace=False)).astype(np.int32)
    return u, i, csr, wl


def _oracle(distance, sub32, objects, k, filt, whitelist):
    """Exhaustive fp64 top-k of the subject rows `sub32` (filt: their filter rows) in the engine's result definition
    (COSINE divides by the object norm only), padded like the engine: (ids, scores, counts)."""
    cat = Catalogue(objects, cosine=distance == "cosine", bf16=False, whitelist=whitelist)
    viewed = cat.viewed_positions(filt.indptr, filt.indices, len(sub32))
    norms = cat.norms[cat.pos2obj] if cat.cosine else None
    ids, sc = implicit_topk(cat.obj64_pos.astype(np.float32), np.ascontiguousarray(sub32, np.float32), k, norms, viewed, accum="f64")
    valid = sc > np.float32(neginf_score())
    return np.where(valid, cat.pos2obj[ids], -1), sc, valid.sum(axis=1)


def _check(ids, sc, cnt, oracle, sel, name):
    oid, osc, ocnt = oracle
    np.testing.assert_array_equal(cnt[sel], ocnt, err_msg=name)
    valid = np.arange(ids.shape[1])[None, :] < ocnt[:, None]
    np.testing.assert_array_equal(np.where(valid, ids[sel], -1), np.where(valid, oid, -1), err_msg=name)
    np.testing.assert_allclose(sc[sel][valid], osc[valid], rtol=3e-7, atol=1.5e-45, err_msg=name)


# ------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("k", [129, 256, 500, 1000, 1024])
@pytest.mark.parametrize("distance", ["dot", "cosine"])
@pytest.mark.parametrize("with_wl", [False, True])
def test_parity_with_the_fp64_oracle(lib, data, k, distance, with_wl):
    """Default flags and FORCE_TC both take the one-pass wide mode (n_rows x n_pos far above the tiny-problem size) and
    return full rows equal to the oracle on a sample of rows."""
    from rectools_b200 import Engine

    u, i, csr, wl = data
    whitelist = wl if with_wl else None
    eng = Engine(i, cosine=distance == "cosine")
    sel = np.arange(0, N_ROWS, 47)
    expected = _oracle(distance, u[sel], i, k, csr[sel], whitelist)
    for flags in (0, lib.Q_FORCE_TC):
        ids, sc, cnt = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, whitelist=whitelist, flags=flags)
        st = eng.last_stats
        name = f"{distance} k={k} wl={with_wl} flags={flags} {st}"
        assert st["path"] == 1 and st["wide"] == 1 and st["k_out"] == k, name
        assert (cnt == k).all(), name
        _check(ids, sc, cnt, expected, sel, name)
        print(f"\n[{name}]")
    eng.close()


def test_bf16_k500(lib, data):
    from rectools_b200 import Engine

    u, i, csr, _ = data
    eng = Engine(i, cosine=False, tc_mode="bf16")
    assert eng.info()["tc_dtype"] == lib.TC_BF16
    ids, sc, cnt = eng.topk(500, subjects=u, indptr=csr.indptr, indices=csr.indices)
    st = eng.last_stats
    assert st["path"] == 1 and st["wide"] == 1 and st["tc_dtype"] == lib.TC_BF16, st
    sel = np.arange(0, N_ROWS, 31)
    _check(ids, sc, cnt, _oracle("dot", u[sel], i, 500, csr[sel], None), sel, f"bf16 {st}")
    eng.close()


def test_path_choice_outside_the_wide_range(lib, data, monkeypatch):
    """k > 1024, a candidate count above half the catalogue, B200_WIDE=0 and FORCE_EXACT keep path 3; FORCE_TC is refused
    where the wide mode is not eligible."""
    from rectools_b200 import Engine

    u, i, csr, _ = data
    small = np.arange(0, 3_000, dtype=np.int32)  # T(1000) = 1664 > 1500
    eng = Engine(i, cosine=False)
    rows = u[:400]
    for k, wl, flags in ((1025, None, 0), (1000, small, 0), (300, None, lib.Q_FORCE_EXACT)):
        eng.topk(k, subjects=rows, whitelist=wl, flags=flags)
        assert eng.last_stats["path"] == 3, (k, eng.last_stats)
    for k, wl in ((1025, None), (1000, small)):
        with pytest.raises(NotImplementedError):
            eng.topk(k, subjects=rows, whitelist=wl, flags=lib.Q_FORCE_TC)
    monkeypatch.setenv("B200_WIDE", "0")
    eng.topk(300, subjects=u, indptr=csr.indptr, indices=csr.indices)
    assert eng.last_stats["path"] == 3 and eng.last_stats["wide"] == 0, eng.last_stats
    eng.close()


# ------------------------------------------------------------------------------------------------ short rows
def test_rows_with_fewer_survivors_than_k(lib, data):
    """Rows that viewed all but a few dozen objects: fewer than k survivors on the tensor-core path, counts and ids as
    the oracle's."""
    from rectools_b200 import Engine

    u, i, _, _ = data
    n_rows, k = 2_000, 300
    rng = np.random.default_rng(5)
    cols = []
    for r in range(n_rows):
        if r % 97 == 0:
            keep = rng.choice(N_OBJ, 40 + (r // 97) * 11, replace=False)  # 40 .. 260 survivors
            cols.append(np.setdiff1d(np.arange(N_OBJ), keep))
        else:
            cols.append(np.unique(rng.integers(0, N_OBJ, 100)))
    indptr = np.zeros(n_rows + 1, np.int64)
    indptr[1:] = np.cumsum([len(c) for c in cols])
    indices = np.concatenate(cols).astype(np.int32)
    csr = sparse.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(n_rows, N_OBJ))
    eng = Engine(i, cosine=False)
    ids, sc, cnt = eng.topk(k, subjects=u[:n_rows], indptr=indptr, indices=indices)
    st = eng.last_stats
    assert st["path"] == 1 and st["wide"] == 1, st
    short = np.arange(0, n_rows, 97)
    sel = np.union1d(short, np.arange(1, n_rows, 101))
    expected = _oracle("dot", u[sel], i, k, csr[sel], None)
    assert (expected[2][np.isin(sel, short)] < k).all()
    _check(ids, sc, cnt, expected, sel, f"short rows {st}")
    eng.close()


# ------------------------------------------------------------------------------------------------ failure route
def _planted_duplicates(seed=41, n_rows=1_500, n_obj=30_000, n_dup=2_000):
    """One object vector copied n_dup times across the catalogue, large enough to lead the ranking of many rows: the cut of
    those rows falls inside a block of exact ties that no append list can hold."""
    u, i = synth_factors(n_rows, n_obj, D, seed=seed)
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(D).astype(np.float32)
    v *= np.float32(5.0 / np.linalg.norm(v))
    i[np.sort(rng.choice(n_obj, n_dup, replace=False))] = v
    return u, i


@pytest.mark.parametrize("kind", ["T_just_above_k", "duplicates_at_the_cut"])
@pytest.mark.parametrize("with_ids", [False, True])
def test_failed_rows_take_the_row_list_exhaustive_rerank(lib, monkeypatch, kind, with_ids):
    """Rows the wide pass cannot certify (too few candidates, overflowing lists) are re-ranked by the exhaustive kernels
    over a row list: through a plain subject matrix and through resident subjects + subject ids (row map), host outputs
    patched row by row."""
    from rectools_b200 import Engine

    k = 200
    if kind == "T_just_above_k":
        monkeypatch.setenv("B200_WIDE_T", str(k + 1))
        u, i = synth_factors(2_000, 40_000, D, seed=43)
    else:
        u, i = _planted_duplicates()
    n_users, n_obj = len(u), len(i)
    csr_all = synth_viewed_csr(n_users, n_obj, 100, seed=44)
    eng = Engine(i, cosine=False)
    if with_ids:
        sids = np.random.default_rng(45).permutation(n_users)[: n_users - 7].astype(np.int64)
        eng.set_subjects(u)
        call_csr = csr_all[sids]
        ids, sc, cnt = eng.topk(k, subject_ids=sids, indptr=call_csr.indptr, indices=call_csr.indices)
    else:
        sids = np.arange(n_users, dtype=np.int64)
        call_csr = csr_all
        ids, sc, cnt = eng.topk(k, subjects=u, indptr=call_csr.indptr, indices=call_csr.indices)
    st = eng.last_stats
    name = f"{kind} ids={with_ids} {st}"
    print(f"\n[{name}]")
    # every row (the failed ones included) against the oracle
    _check(ids, sc, cnt, _oracle("dot", u[sids], i, k, call_csr, None), np.arange(len(sids)), name)
    assert st["path"] == 1 and st["wide"] == 1, name
    assert st["n_fallback_rows"] > 0 and st["n_exact_rows"] == st["n_fallback_rows"], name
    eng.close()


# ------------------------------------------------------------------------------------------------ chunking
def test_device_inputs_are_chunked_within_the_candidate_budget(lib, data, monkeypatch):
    """Device-resident inputs and outputs: a lowered candidate-buffer budget splits the call into row chunks; the results
    equal the one-chunk call and the oracle."""
    import torch

    from rectools_b200 import Engine

    u, i, csr, wl = data
    k = 500
    dev = torch.device("cuda:0")
    d_u = torch.from_numpy(u).to(dev)
    d_ip = torch.from_numpy(csr.indptr.astype(np.int64)).to(dev)
    d_ix = torch.from_numpy(csr.indices.astype(np.int32)).to(dev)
    d_wl = torch.from_numpy(wl).to(dev)
    eng = Engine(i, cosine=True)

    def call():
        o_ids = torch.empty((N_ROWS, k), dtype=torch.int32, device=dev)
        o_sc = torch.empty((N_ROWS, k), dtype=torch.float32, device=dev)
        o_cnt = torch.empty((N_ROWS,), dtype=torch.int32, device=dev)
        st = eng.topk_ptrs(N_ROWS, k, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), lib.Q_INPUTS_ON_DEVICE | lib.Q_OUTPUTS_ON_DEVICE,
                           subjects=d_u.data_ptr(), indptr=d_ip.data_ptr(), indices=d_ix.data_ptr(), whitelist=d_wl.data_ptr(),
                           n_whitelist=len(wl), stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy(), dict(st)

    ids0, sc0, cnt0, st0 = call()
    assert st0["n_chunks"] == 1 and st0["path"] == 1 and st0["wide"] == 1, st0
    monkeypatch.setenv("B200_WIDE_BUDGET_MB", "8")
    ids1, sc1, cnt1, st1 = call()
    print(f"\n[chunked {st1}]")
    assert st1["n_chunks"] > 1 and st1["path"] == 1 and st1["wide"] == 1, st1
    np.testing.assert_array_equal(ids0, ids1)
    np.testing.assert_array_equal(sc0, sc1)
    np.testing.assert_array_equal(cnt0, cnt1)
    sel = np.arange(0, N_ROWS, 29)
    _check(ids1, sc1, cnt1, _oracle("cosine", u[sel], i, k, csr[sel], wl), sel, f"chunked {st1}")
    eng.close()


# ------------------------------------------------------------------------------------------------ the pass itself
@pytest.mark.parametrize("k", [200, 1000])
@pytest.mark.parametrize("tc_mode", ["fp16", "bf16"])
def test_snapshot_of_the_large_k_pass(lib, monkeypatch, capsys, k, tc_mode):
    """tests/tc_reference.py on every row and list of the main pass: list contents, P1, P2, thresholds and the verdict,
    with append lists longer than the 512 slots of the k <= 128 re-score."""
    from rectools_b200 import Engine

    n_rows, n_obj = 600, 20_000
    u, i = synth_factors(n_rows, n_obj, D, seed=k)
    csr = synth_viewed_csr(n_rows, n_obj, 100, seed=k + 1)
    bf16 = tc_mode == "bf16"
    eng = Engine(i, cosine=False, tc_mode=tc_mode)
    monkeypatch.setenv("B200_TC_SNAPSHOT", "1")
    ids, sc, cnt = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, flags=lib.Q_FORCE_TC)
    st = dict(eng.last_stats)
    assert st["path"] == 1 and st["wide"] == 1, st
    snap = eng.candidate_snapshot()
    assert snap is not None and snap["wide"] == 1 and snap["kp"] == k and snap["k_cand"] == 32
    assert snap["n_lists"] * snap["cand_stride"] > 512
    cat = Catalogue(i, cosine=False, bf16=bf16)
    viewed = cat.viewed_positions(csr.indptr, csr.indices, n_rows)
    rep = check_snapshot(snap, cat, u, viewed)
    with capsys.disabled():
        print(f"\n[large-k snapshot k={k} {tc_mode}] stride={snap['cand_stride']} phase1={snap['phase1_tiles']}/{snap['tiles_per_split']} "
              f"max_count={int(snap['cand_counts'][:, :n_rows].sum(axis=0).max())} {rep.summary()} | {st['n_fallback_rows']} fallback rows")
    assert rep.ok, rep.summary()
    assert rep.n_fb == st["n_fallback_rows"]
    sel = np.arange(0, n_rows, 7)
    _check(ids, sc, cnt, _oracle("dot", u[sel], i, k, csr[sel], None), sel, f"snapshot k={k} {tc_mode}")
    eng.close()


# ------------------------------------------------------------------------------------------------ through the reference
def test_candidate_generator_through_the_unmodified_reference():
    """`CandidateGenerator(model, num_candidates=300, ...).generate_candidates(...)` -- the first stage of RecTools'
    two-stage `CandidateRankingModel` -- for PureSVD and an injected ALS model: after `install()` the frame equals the
    stock one and the engine took the wide mode."""
    from oracle import stage_reference

    if not stage_reference.available():
        pytest.skip("reference package not staged (oracle/_ref)")
    added = stage_reference.add_to_path()
    try:
        from rectools.models import PureSVDModel
        from rectools.models.ranking import CandidateGenerator

        import rectools_b200
        from rectools_b200 import integration
        from tests.ref_models import injected_als, synthetic_dataset
        from tests.test_gpu_models import _factors, _same_reco

        n_users, n_items = 6000, 3000
        dataset = synthetic_dataset(n_users, n_items, 30, seed=11)
        models = {
            "puresvd": PureSVDModel(factors=32, random_state=0).fit(dataset),
            "als": injected_als(_factors(n_users, 64, 12), _factors(n_items, 64, 13)),
        }
        users = np.random.default_rng(14).permutation(dataset.user_id_map.external_ids)[:5000]

        def generate(model):
            gen = CandidateGenerator(model, num_candidates=300, keep_ranks=True, keep_scores=True)
            gen.is_fitted_for_recommend = True  # the models are fitted already
            return gen.generate_candidates(users, dataset, filter_viewed=True, for_train=False)

        expected = {name: generate(m) for name, m in models.items()}
        rectools_b200.install(device=0)
        try:
            for name, model in models.items():
                got = generate(model)
                _same_reco(expected[name], got)
                stats = [e.last_stats for e in integration._ENGINE_CACHE.values()]  # pylint: disable=protected-access
                assert any(s.get("path") == 1 and s.get("wide") == 1 and s.get("k_out") == 300 for s in stats), (name, stats)
                assert len(got) == 300 * len(users), name
        finally:
            rectools_b200.uninstall()
    finally:
        stage_reference.remove_from_path(added)

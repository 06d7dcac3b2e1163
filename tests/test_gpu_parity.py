"""GPU parity tests: the CUDA path (through the C ABI, via B200Ranker / Engine) against the oracle and the golden
fixtures generated from the unmodified reference.  On continuous factors every engine result is held to the
rounding-interval checker of tests/score_interval.py (the engine defines scores as the fp64-accumulated dot rounded once
to fp32: no tolerance), and `rank()`'s flat output to the padded one bit for bit; the golden fixtures of the fp32
reference keep their tie window."""
import os

import numpy as np
import pytest
from scipy import sparse

from tests.helpers import (
    assert_same_ranking,
    golden_keys,
    load_rank_case,
    parse_key,
    synth_factors,
    synth_viewed_csr,
)
from tests.score_interval import check_topk, norm_interval, widen64

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    import rectools_b200

    return rectools_b200


# ------------------------------------------------------------------ reference known-answer vectors (test_rank.py:52-233)
SUBJECTS = np.array([[-4, 0, 3], [0, 1, 2]])
OBJECTS = np.array([[-4, 0, 3], [0, 2, 4], [1, 10, 100]])


@pytest.mark.parametrize(
    "distance, expected_recs, expected_scores",
    (
        ("dot", [2, 0, 1, 2, 1, 0], [296, 25, 12, 210, 10, 6]),
        ("cosine", [0, 2, 1, 1, 2, 0], [1, 0.5890328, 0.5366563, 1, 0.9344414, 0.5366563]),
        ("euclidean", [0, 1, 2, 1, 0, 2], [0, 4.58257569, 97.64220399, 2.23606798, 4.24264069, 98.41747812]),
    ),
)
@pytest.mark.parametrize("dense", [True, False])
def test_rank_known_answers(rb, distance, expected_recs, expected_scores, dense):
    subj = SUBJECTS if dense else sparse.csr_matrix(SUBJECTS)
    if not dense and distance != "dot":
        with pytest.raises(ValueError):
            rb.B200Ranker(distance, subj, OBJECTS)
        return
    ranker = rb.B200Ranker(distance, subj, OBJECTS)
    users, recs, scores = ranker.rank(subject_ids=[0, 1], k=3)
    np.testing.assert_equal(users, [0, 0, 0, 1, 1, 1])
    np.testing.assert_equal(recs, expected_recs)
    np.testing.assert_almost_equal(scores, expected_scores, decimal=5)


@pytest.mark.parametrize(
    "distance, expected_recs, expected_scores",
    (
        ("dot", [2, 1, 2, 0], [296, 12, 210, 6]),
        ("cosine", [2, 1, 2, 0], [0.5890328, 0.5366563, 0.9344414, 0.5366563]),
        ("euclidean", [1, 2, 0, 2], [4.58257569, 97.64220399, 4.24264069, 98.41747812]),
    ),
)
def test_rank_with_filter_known_answers(rb, distance, expected_recs, expected_scores):
    ui_csr = sparse.csr_matrix([[1, 0, 0], [0, 1, 0]])
    _, recs, scores = rb.B200Ranker(distance, SUBJECTS, OBJECTS).rank([0, 1], k=3, filter_pairs_csr=ui_csr)
    np.testing.assert_equal(recs, expected_recs)
    np.testing.assert_almost_equal(scores, expected_scores, decimal=5)


@pytest.mark.parametrize(
    "distance, expected_recs, expected_scores",
    (
        ("dot", [2, 0, 2, 0], [296, 25, 210, 6]),
        ("cosine", [0, 2, 2, 0], [1, 0.5890328, 0.9344414, 0.5366563]),
        ("euclidean", [0, 2, 0, 2], [0, 97.64220399, 4.24264069, 98.41747812]),
    ),
)
def test_rank_with_whitelist_known_answers(rb, distance, expected_recs, expected_scores):
    _, recs, scores = rb.B200Ranker(distance, SUBJECTS, OBJECTS).rank([0, 1], k=3, sorted_object_whitelist=np.array([0, 2]))
    np.testing.assert_equal(recs, expected_recs)
    np.testing.assert_almost_equal(scores, expected_scores, decimal=5)


def test_shape_mismatch_raises(rb):
    ranker = rb.B200Ranker("dot", SUBJECTS, OBJECTS)
    with pytest.raises(ValueError):
        ranker.rank([0, 1], k=3, filter_pairs_csr=sparse.csr_matrix([[1, 0, 0]]))


# ------------------------------------------------------------------ golden fixtures from the unmodified reference
@pytest.mark.parametrize("case", [0, 1, 2])
@pytest.mark.parametrize("force", ["default", "tc", "exact"])
def test_golden_rankers(rb, case, force):
    from rectools_b200 import _lib

    inp, out, csr = load_rank_case(case)
    rankers = {}
    n_checked = 0
    for key in golden_keys(out):
        impl, dist, k, use_filter, use_wl = parse_key(key)
        if impl == "torch" and dist == "euclidean":
            continue  # cdist-based scores / -inf masking differ from the implicit contract (see test_oracle_golden.py)
        if dist not in rankers:
            rankers[dist] = rb.B200Ranker(dist, inp["subjects"], inp["objects"])
        ranker = rankers[dist]
        n_pos = len(inp["whitelist"]) if use_wl else inp["objects"].shape[0]
        k_eff = n_pos if k is None else min(k, n_pos)
        flags = 0
        if force == "tc":
            if k_eff > 24 or n_pos < 128:
                continue
            flags = _lib.Q_FORCE_TC
        elif force == "exact":
            flags = _lib.Q_FORCE_EXACT
        sids, ids, scores, counts = ranker.rank_padded(
            inp["subject_ids"], k, csr if use_filter else None, inp["whitelist"] if use_wl else None, flags=flags
        )
        if force == "tc":
            assert ranker.last_stats["path"] == 1
        subj, fids, fscores = rb.flatten_padded(sids, ids, scores, counts)
        if dist == "cosine":
            fscores = fscores / ranker.subjects_norms[subj]
        elif dist == "euclidean":
            fscores = np.sqrt(np.maximum(ranker.subjects_dots[subj] - fscores, 0)).astype(np.float32)
        np.testing.assert_array_equal(subj, out[key + "|subjects"], err_msg=key)
        atol = 2e-4 if dist == "euclidean" else 2e-6
        assert_same_ranking(fids, fscores, out[key + "|ids"], out[key + "|scores"], tie_tol=2e-6, atol=atol, msg=key)
        n_checked += 1
    assert n_checked > 10 or (force == "tc" and case == 2)  # case 2 (64 objects) is below the tensor-core path's minimum


def test_golden_puresvd_c1(rb, golden_dir):
    """BASELINE config 1: factors of the reference's PureSVDModel(factors=32) on 6040x3706, K=10, filter_viewed."""
    g = np.load(os.path.join(golden_dir, "puresvd_c1.npz"))
    csr = sparse.csr_matrix(
        (np.ones(len(g["csr_indices"]), np.float32), g["csr_indices"], g["csr_indptr"]), shape=tuple(g["csr_shape"])
    )
    ranker = rb.B200Ranker("dot", g["user_factors"], g["item_factors"])
    for filt, pre in ((csr, "out_"), (None, "out_nf_")):
        subj, ids, scores = ranker.rank(g["subject_ids"], 10, filt)
        np.testing.assert_array_equal(subj, g[pre + "subjects"])
        assert_same_ranking(ids, scores, g[pre + "ids"], g[pre + "scores"], tie_tol=2e-6, msg=pre)


def _flat_is_padded(ranker, padded, flat, subjects, name):
    """`rank()`'s flat output is the padded call's entries, COSINE scores divided by `subjects_norms` in fp32, bit for
    bit; the subject norms are fp32 roundings of fp64 sums (inside the norm interval of the `subjects` rows)."""
    from rectools_b200.ranker import flatten_padded

    subj, fids, fsc = flatten_padded(*padded)
    if ranker.subjects_norms is not None:
        n_lo, n_hi = norm_interval(widen64(subjects))
        assert ((ranker.subjects_norms >= n_lo) & (ranker.subjects_norms <= n_hi)).all(), name
        fsc = (fsc / ranker.subjects_norms[subj]).astype(np.float32)
    np.testing.assert_array_equal(flat[0], subj, err_msg=f"{name}: rank() subjects")
    np.testing.assert_array_equal(flat[1], fids, err_msg=f"{name}: rank() ids")
    np.testing.assert_array_equal(np.asarray(flat[2], np.float32).view(np.int32), fsc.view(np.int32), err_msg=f"{name}: rank() scores")

# ------------------------------------------------------------------ seeded random inputs vs the fp64 oracle
@pytest.mark.parametrize(
    "n_users, n_items, d, k, per_user, distance, tc_mode",
    [
        (2048, 50_000, 128, 10, 100, "dot", "auto"),
        (2048, 50_000, 128, 10, 100, "cosine", "auto"),
        (1024, 30_000, 128, 10, 50, "dot", "bf16"),
        (777, 20_011, 64, 20, 30, "dot", "auto"),
        (300, 9_001, 200, 5, 10, "cosine", "auto"),
        (513, 12_345, 256, 20, 0, "dot", "auto"),
        (64, 5_000, 32, 100, 40, "dot", "auto"),  # K > 32: multi-pass exhaustive kernel
    ],
)
def test_random_vs_oracle(rb, n_users, n_items, d, k, per_user, distance, tc_mode):
    from rectools_b200 import _lib

    u, i = synth_factors(n_users, n_items, d, seed=n_users)
    csr = synth_viewed_csr(n_users, n_items, per_user) if per_user else None
    ranker = rb.B200Ranker(distance, u, i, tc_mode=tc_mode)
    sids = np.arange(n_users)
    for flags in ((_lib.Q_FORCE_TC if k <= 24 else 0), _lib.Q_FORCE_EXACT):
        if flags == _lib.Q_FORCE_EXACT and n_users * n_items > 3e7:
            sel = sids[:: max(1, n_users // 128)]
        else:
            sel = sids
        sub_csr = csr[sel] if csr is not None else None
        _, ids, scores, counts = ranker.rank_padded(sel, k, sub_csr, flags=flags)
        assert (counts == k).all()
        # engine scores are before the subject-norm division: the object side of COSINE only
        check_topk((ids, scores, counts), u[sel], i, k, cosine=distance == "cosine", filter_csr=sub_csr,
                   name=f"flags={flags} stats={ranker.last_stats}")
        if flags == _lib.Q_FORCE_TC:
            assert ranker.last_stats["path"] == 1
            assert ranker.last_stats["n_fallback_rows"] <= max(4, n_users // 50), ranker.last_stats


@pytest.mark.parametrize("mode", ["wide", "multipass"])
@pytest.mark.parametrize("distance, k, use_wl", [("dot", 100, False), ("cosine", 100, True), ("dot", 37, False), ("cosine", 128, False)])
def test_large_k_on_the_tensor_core_path(rb, monkeypatch, distance, k, use_wl, mode):
    """24 < k <= 128 on the tensor-core path (BASELINE config 3 shape: COSINE, K = 100, ~100 viewed).
    wide (default): ONE pass -- adaptive lists for the first part of the stream, then the frozen threshold + global append,
    block-per-row re-score; rows whose certificate fails take the multi-pass route.  multipass (B200_WIDE=0): certified passes
    of 20 results with the earlier results excluded like viewed objects.  Both must give the exact top-k in order."""
    from rectools_b200 import _lib

    if mode == "multipass":
        monkeypatch.setenv("B200_WIDE", "0")
    n_users, n_items, d = 1500, 30_000, 64
    u, i = synth_factors(n_users, n_items, d, seed=k)
    csr = synth_viewed_csr(n_users, n_items, 100)
    wl = np.sort(np.random.default_rng(4).choice(n_items, 9_000, replace=False)) if use_wl else None
    ranker = rb.B200Ranker(distance, u, i)
    sids = np.arange(n_users)
    _, ids, scores, counts = ranker.rank_padded(sids, k, csr, wl, flags=_lib.Q_FORCE_TC)
    st = ranker.last_stats
    assert st["path"] == 1 and (counts == k).all() and st["wide"] == (0 if mode == "multipass" else 1), st
    if mode != "multipass":
        assert st["n_tc_launches"] <= 1 + 12 * (st["n_fallback_rows"] > 0), st  # one main pass; re-rank passes only for failures
        assert st["n_fallback_rows"] <= n_users // 10, st
    sel = sids[::5]
    check_topk((ids[sel], scores[sel], counts[sel]), u[sel], i, k, cosine=distance == "cosine", filter_csr=csr[sel],
               whitelist=wl, name=str(st))


def test_wide_mode_overflow_and_short_streams(rb, monkeypatch):
    """Wide mode corner cases: a target far below what the catalogue offers (lists overflow -> rows re-ranked), duplicated
    top objects (ties at the cut), a catalogue of a few tiles (phase 1 covers most of the stream)."""
    from rectools_b200 import _lib

    n_users, n_items, d, k = 700, 6_000, 32, 60
    u, i = synth_factors(n_users, n_items, d, seed=3)
    i[1000:1100] = i[1000]  # 100 identical objects
    csr = synth_viewed_csr(n_users, n_items, 40)
    ranker = rb.B200Ranker("dot", u, i)
    sids = np.arange(n_users)
    for env in ({}, {"B200_WIDE_T": "400"}, {"B200_WIDE_T": "61"}):
        for k_, v_ in env.items():
            monkeypatch.setenv(k_, v_)
        _, ids, scores, counts = ranker.rank_padded(sids, k, csr, flags=_lib.Q_FORCE_TC)
        assert ranker.last_stats["wide"] == 1 and (counts == k).all()
        check_topk((ids, scores, counts), u, i, k, filter_csr=csr, name=f"{env} {ranker.last_stats}")


@pytest.mark.parametrize("splits", [None, "3"])
@pytest.mark.parametrize("carousel", [True, False], ids=["carousel", "no_carousel"])
def test_many_work_items_per_cta(rb, monkeypatch, splits, carousel):
    """More subject tiles than CTA pairs (persistent loop, accumulator / list / threshold hand-over between work items) and
    forced object splits, with every work item starting where the reference pair is in the object stream (the carousel)
    and at its first object tile."""
    from rectools_b200 import _lib

    if not carousel:
        monkeypatch.setenv("B200_TC_CAROUSEL", "0")
    if splits:
        monkeypatch.setenv("B200_TC_SPLITS", splits)
    n_users, n_items, d, k = 60_000, 12_345, 64, 10
    u, i = synth_factors(n_users, n_items, d, seed=77)
    csr = synth_viewed_csr(n_users, n_items, 30)
    ranker = rb.B200Ranker("dot", u, i)
    sids = np.arange(n_users)
    _, ids, scores, counts = ranker.rank_padded(sids, k, csr, flags=_lib.Q_FORCE_TC)
    assert ranker.last_stats["path"] == 1 and ranker.last_stats["epi_warps"] == 8
    sel = np.unique(np.concatenate([np.arange(0, n_users, 29), np.arange(n_users - 300, n_users)]))
    check_topk((ids[sel], scores[sel], counts[sel]), u[sel], i, k, filter_csr=csr[sel], name=str(ranker.last_stats))
    # determinism: a second call returns bit-identical arrays
    _, ids2, scores2, _ = ranker.rank_padded(sids, k, csr, flags=_lib.Q_FORCE_TC)
    np.testing.assert_array_equal(ids, ids2)
    np.testing.assert_array_equal(scores, scores2)


def test_edge_cases(rb):
    from rectools_b200 import _lib

    rng = np.random.default_rng(5)
    n_users, n_items, d = 40, 700, 24
    u = rng.standard_normal((n_users, d)).astype(np.float32)
    i = rng.standard_normal((n_items, d)).astype(np.float32)
    i[100:140] = i[100]  # 40 identical objects: ties must come out in ascending id order
    i[300:320] = 0.0  # zero vectors (score exactly 0, COSINE norm guard)
    u[7] = 0.0  # zero subject: every score ties at 0
    dense = np.zeros((n_users, n_items), dtype=np.float32)
    dense[3, :] = 1  # everything viewed -> no recommendations
    dense[4, : n_items - 3] = 1  # only 3 candidates left -> fewer than k rows
    dense[5, ::2] = 1
    csr = sparse.csr_matrix(dense)
    whitelist = np.sort(rng.choice(n_items, 333, replace=False))
    for distance in ("dot", "cosine"):
        ranker = rb.B200Ranker(distance, u, i)
        for wl in (None, whitelist):
            for k in (1, 10, 24, 33, 100, None):
                for flags in (0, _lib.Q_FORCE_TC, _lib.Q_FORCE_EXACT):
                    n_pos = n_items if wl is None else len(wl)
                    k_eff = n_pos if k is None else min(k, n_pos)
                    if flags == _lib.Q_FORCE_TC and k_eff > 128:
                        continue
                    sids = np.arange(n_users)[::-1].copy()
                    s1, r1, c1 = ranker.rank(sids, k, csr[sids], wl) if flags == 0 else (None, None, None)
                    _, ids, scores, counts = ranker.rank_padded(sids, k, csr[sids], wl, flags=flags)
                    msg = f"{distance} wl={wl is not None} k={k} flags={flags}"
                    check_topk((ids, scores, counts), u[sids], i, k, cosine=distance == "cosine", filter_csr=csr[sids],
                               whitelist=wl, name=msg, verbose=False)
                    if s1 is not None:
                        _flat_is_padded(ranker, (sids, ids, scores, counts), (s1, r1, c1), u, msg)
    # empty subject list / k larger than the catalogue
    ranker = rb.B200Ranker("dot", u, i[:5])
    s, r, c = ranker.rank([], k=3)
    assert len(s) == len(r) == len(c) == 0
    s, r, c = ranker.rank([0, 1], k=50)
    assert len(r) == 10
    with pytest.raises(ValueError):
        ranker.rank([0], k=0)


def test_near_ties_are_certified_or_re_ranked(rb):
    """Adversarial for the tensor-core candidate pass: 300 objects whose scores differ by ~1e-6 relative -- far below the
    fp16 operand resolution -- sit at the top of every row, so the approximate pass cannot order them.  The certificate
    must notice (rows go to the wider re-rank / the exhaustive kernel) and the returned ids must still equal the oracle."""
    from rectools_b200 import _lib

    rng = np.random.default_rng(9)
    n_users, n_items, d, k = 600, 20_000, 64, 10
    u = (rng.standard_normal((n_users, d)) / np.sqrt(d)).astype(np.float32)
    i = (0.2 * rng.standard_normal((n_items, d)) / np.sqrt(d)).astype(np.float32)
    base = u.mean(axis=0) + 0.5 * rng.standard_normal(d).astype(np.float32) / np.sqrt(d)
    hot = rng.choice(n_items, 300, replace=False)
    i[hot] = (3.0 * base[None, :] * (1.0 + 1e-6 * rng.standard_normal((300, 1)))).astype(np.float32)
    u = (u * 0.05 + base[None, :]).astype(np.float32)  # every subject scores the hot objects highest, within ~1e-6 of each other
    csr = synth_viewed_csr(n_users, n_items, 20)
    ranker = rb.B200Ranker("dot", u, i)
    sids = np.arange(n_users)
    _, ids, scores, counts = ranker.rank_padded(sids, k, csr, flags=_lib.Q_FORCE_TC)
    stats = ranker.last_stats
    assert stats["path"] == 1 and stats["n_fallback_rows"] > 0, stats  # the approximate pass alone could not decide
    check_topk((ids, scores, counts), u, i, k, filter_csr=csr, name=f"near ties {stats}")


def test_torch_ranker_signature_with_device_tensors(rb):
    """`TorchRanker`-style construction (rank_torch.py:59-67) with embeddings already on the GPU: device pointers are
    handed to the engine, results equal the oracle (and the reference's value-based filter semantics, rank_torch.py:143)."""
    import torch

    n_users, n_items, d, k = 700, 9_000, 48, 10
    u, i = synth_factors(n_users, n_items, d, seed=31)
    csr = synth_viewed_csr(n_users, n_items, 25)
    csr.data[::7] = 0.0  # explicit zeros do not filter in TorchRanker
    for distance in ("dot", "cosine"):
        ranker = rb.B200TorchRanker(distance, "cuda:0", torch.from_numpy(u), torch.from_numpy(i).to("cuda:0"), batch_size=128)
        sids = np.arange(n_users)
        flat = ranker.rank(sids, k, csr)
        eff = csr.copy()
        eff.eliminate_zeros()
        padded = ranker.rank_padded(sids, k, eff)
        check_topk(padded[1:], u, i, k, cosine=distance == "cosine", filter_csr=eff, name=f"torch ranker {distance}")
        _flat_is_padded(ranker, padded, flat, u, f"torch ranker {distance}")


def test_merge_matches_unsharded(rb):
    """Item-sharded ranking: per-shard top-k with global ids + b200_rank_merge == ranking the whole catalogue."""
    import torch

    from rectools_b200 import _lib

    n_users, n_items, d, k = 1000, 40_000, 64, 10
    u, i = synth_factors(n_users, n_items, d, seed=11)
    csr = synth_viewed_csr(n_users, n_items, 20)
    full = rb.B200Ranker("dot", u, i)
    _, ids_full, sc_full, cnt_full = full.rank_padded(np.arange(n_users), k, csr)
    shards = 3
    bounds = np.linspace(0, n_items, shards + 1).astype(int)
    all_ids, all_sc, all_cnt = [], [], []
    for s in range(shards):
        lo, hi = bounds[s], bounds[s + 1]
        eng = rb.Engine(i[lo:hi], cosine=False, id_offset=int(lo))
        ids, sc, cnt = eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices)
        assert ids[cnt > 0].min() >= lo and ids.max() < hi
        all_ids.append(ids)
        all_sc.append(sc)
        all_cnt.append(cnt)
        eng.close()
    dev = torch.device("cuda:0")
    t_ids = torch.from_numpy(np.stack(all_ids)).to(dev)
    t_sc = torch.from_numpy(np.stack(all_sc)).to(dev)
    t_cnt = torch.from_numpy(np.stack(all_cnt)).to(dev)
    o_ids = torch.empty((n_users, k), dtype=torch.int32, device=dev)
    o_sc = torch.empty((n_users, k), dtype=torch.float32, device=dev)
    o_cnt = torch.empty((n_users,), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    _lib.check(
        _lib.load().b200_rank_merge(
            0, torch.cuda.current_stream().cuda_stream, shards, n_users, k, t_ids.data_ptr(), t_sc.data_ptr(),
            t_cnt.data_ptr(), o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(),
        )
    )
    torch.cuda.synchronize()
    np.testing.assert_array_equal(o_ids.cpu().numpy(), ids_full)
    np.testing.assert_array_equal(o_sc.cpu().numpy(), sc_full)
    np.testing.assert_array_equal(o_cnt.cpu().numpy(), cnt_full)


@pytest.mark.parametrize("with_ids", [False, True])
def test_chunked_copy_compute_pipeline_matches_unchunked(rb, monkeypatch, with_ids):
    """Large host-buffer calls are staged / ranked / copied back in row chunks on two streams (B200_CHUNK_ROWS forces small
    chunks here): same arrays as the one-shot call, including a ragged last chunk, a CSR filter and a whitelist."""
    from rectools_b200 import _lib

    n_users, n_items, d, k = 9_001, 20_000, 64, 10
    u, i = synth_factors(n_users, n_items, d, seed=5)
    csr = synth_viewed_csr(n_users, n_items, 40)
    wl = np.arange(0, n_items, 3, dtype=np.int32)
    eng = rb.Engine(i, cosine=False)
    sids = np.random.default_rng(0).permutation(n_users).astype(np.int64)

    def call():
        if with_ids:
            sub = csr[sids]
            return eng.topk(k, subjects=u, subject_ids=sids, indptr=sub.indptr, indices=sub.indices, whitelist=wl, flags=_lib.Q_FORCE_TC)
        return eng.topk(k, subjects=u, indptr=csr.indptr, indices=csr.indices, whitelist=wl, flags=_lib.Q_FORCE_TC)

    ids0, sc0, cnt0 = call()
    assert eng.last_stats["n_chunks"] == 1
    monkeypatch.setenv("B200_CHUNK_ROWS", "2048")
    ids1, sc1, cnt1 = call()
    assert eng.last_stats["n_chunks"] == 5 and eng.last_stats["path"] == 1
    np.testing.assert_array_equal(ids0, ids1)
    np.testing.assert_array_equal(sc0, sc1)
    np.testing.assert_array_equal(cnt0, cnt1)
    rows = sids if with_ids else np.arange(n_users)
    sel = np.arange(0, n_users, 37)
    check_topk((ids1[sel], sc1[sel], cnt1[sel]), u[rows[sel]], i, k, filter_csr=csr[rows[sel]], whitelist=wl,
               name=f"chunks {eng.last_stats}")


@pytest.mark.parametrize("cosine", [False, True])
def test_implicit_gpu_shim_topk(rb, cosine):
    """`rectools_b200.implicit_gpu.KnnQuery().topk` (the stand-in for `implicit.gpu.KnnQuery().topk`, call shape of
    rank_implicit.py:175-182) against the oracle's restatement of implicit's top-k, incl. a row with fewer than k survivors."""
    from rectools_b200.implicit_gpu import COOMatrix, KnnQuery, Matrix

    u, i = synth_factors(300, 5_000, 64, seed=11)
    csr = synth_viewed_csr(300, 5_000, 25).tolil()
    csr[7, :] = 1.0  # everything viewed except three items
    csr[7, [5, 50, 500]] = 0.0
    csr = sparse.csr_matrix(csr)
    csr.eliminate_zeros()
    norms = None
    if cosine:
        norms = np.sqrt(np.einsum("ij,ij->i", i, i, dtype=np.float64)).astype(np.float32)
    ids, scores = KnnQuery().topk(
        items=Matrix(i), m=Matrix(u), k=10, item_norms=None if norms is None else Matrix(norms[None, :]),
        query_filter=COOMatrix(csr.tocoo()), item_filter=None,
    )
    counts = (ids >= 0).sum(axis=1).astype(np.int32)
    assert ids.shape == (300, 10) and counts[7] == 3 and (scores[7, 3:] <= -3.0e38).all() and (ids[7, 3:] == -1).all()
    # (the engine divides by its own fp32 norms, which are the caller's here: both are fp32 roundings of fp64 sums)
    check_topk((ids, scores, counts), u, i, 10, cosine=cosine, filter_csr=csr, name=f"implicit shim cosine={cosine}")


def test_k_none_and_k_above_128_materialised_scores(rb):
    """`k=None` (all objects, rank_implicit.py:233-234) and k > 128: the exhaustive scores are materialised once and the
    k / 32 selection passes stream them (path 3) -- whitelist, filter, COSINE, rows with fewer than k survivors."""
    n_users, n_items, d = 500, 6_000, 48
    u, i = synth_factors(n_users, n_items, d, seed=8)
    i[100:130] = i[100]
    csr = synth_viewed_csr(n_users, n_items, 60)
    wl = np.sort(np.random.default_rng(2).choice(n_items, 2_500, replace=False))
    sids = np.random.default_rng(3).permutation(n_users)[:300]
    for distance in ("dot", "cosine"):
        ranker = rb.B200Ranker(distance, u, i)
        for k, whitelist in ((None, wl), (300, None), (1000, wl)):
            flat = ranker.rank(sids, k, csr[sids], whitelist)
            assert ranker.last_stats["path"] == 3, ranker.last_stats
            padded = ranker.rank_padded(sids, k, csr[sids], whitelist)
            assert ranker.last_stats["path"] == 3, ranker.last_stats
            name = f"path 3 {distance} k={k} whitelist={whitelist is not None}"
            check_topk(padded[1:], u[sids], i, k, cosine=distance == "cosine", filter_csr=csr[sids], whitelist=whitelist, name=name)
            _flat_is_padded(ranker, padded, flat, u, name)

"""CPU: the case generators and expectations of tests/exact_cases.py against the oracle (`rank_oracle`, `flatten_padded`,
`merge_padded_numpy`), and the planted ties checked to straddle the boundary each one targets."""
import numpy as np
import pytest
from scipy import sparse

from oracle.topk_oracle import rank_oracle
from rectools_b200.ranker import flatten_padded, strip_sentinel_tail
from rectools_b200.sharded import merge_padded_numpy
from tests import exact_cases as ec

SM_COUNT = 132  # H100 SXM; the GPU tests use the engine's own count


@pytest.fixture(scope="module", params=["dot", "cosine"])
def cat(request):
    return request.param, ec.tie_catalogue(SM_COUNT, cosine=request.param == "cosine", n_obj=60_000, n_subjects=64)


def test_split_geometry_follows_run_exact():
    # 300 000 positions: 9375 tiles, at most 146 splits (tiles / 64)
    assert [ec.exact_splits(n, 300_000, 132) for n in (1, 3, 32, 33, 129)] == [146, 146, 146, 132, 53]
    assert ec.exact_splits(1, 5_000, 132) == 2 and ec.exact_splits(1, 1_000, 132) == 1
    e = ec.split_edges(129, 300_000, 132)
    assert len(e) == 52 and e[0] == 177 * 32 and (np.diff(e) == 177 * 32).all()
    assert len(ec.split_edges(1, 300_000, 132)) == 144  # 65 tiles per split: the last of the 146 is empty
    assert ec.dense_chunk_rows(300_000) == 864 and ec.sparse_chunk_rows(270_000) == 994


def test_planted_ties_straddle_their_boundaries(cat):
    distance, c = cat
    cosine = distance == "cosine"
    sc = ec.engine_scores(c.subjects[: len(c.plants)], c.objects, cosine)
    assert len(c.plants) == 10
    for p in c.plants:
        row = sc[p["row"]]
        if p["kind"] == "rank":
            best = np.sort(row)[::-1]
            assert ec.rank_straddle(best, p["at"]) == (p["left"], p["right"]), p
            assert (row[p["block"]] == best[p["at"] - 1]).all()
        else:
            assert ec.position_straddle(row, p["at"]) == (p["left"], p["right"]), p
            assert set(np.nonzero(row == row.max())[0]) == set(p["block"].tolist())
    # the block is invisible to every other row: its objects score 0 there
    others = np.setdiff1d(np.arange(len(c.subjects)), [p["row"] for p in c.plants])
    all_blocks = np.concatenate([p["block"] for p in c.plants])
    assert (ec.engine_scores(c.subjects[others], c.objects[all_blocks], cosine) == 0).all()


def test_integer_scores_tie_at_every_pass_boundary():
    """Natural (unplanted) rows of the DOT catalogue: the k0-th score is shared across every pass boundary for most rows."""
    c = ec.tie_catalogue(SM_COUNT, n_obj=60_000, n_subjects=64)
    rows = np.arange(ec.ZERO_ROW + 1, 64)
    best = -np.sort(-ec.engine_scores(c.subjects[rows], c.objects, False), axis=1)
    for k0 in (32, 64, 96, 128, 160):
        both = [min(ec.rank_straddle(b, k0)) >= 1 for b in best]
        assert np.mean(both) > 0.8, k0


@pytest.mark.parametrize("with_wl", [False, True])
@pytest.mark.parametrize("k", [1, 33, 100, None])
def test_expected_padded_is_the_oracle(cat, k, with_wl):
    distance, c = cat
    rng = np.random.default_rng(3)
    n = len(c.objects)
    sids = np.r_[np.arange(12), rng.integers(0, len(c.subjects), 9)]
    wl = np.sort(rng.choice(n, n // 3, replace=False)) if with_wl else None
    rows = [rng.integers(0, n + 50, rng.integers(0, 200)) for _ in sids]
    rows[3] = np.arange(n)  # everything filtered
    filt = ec.csr_from_rows(rows, n)
    ids, sc, cnt = ec.expected_padded(distance, c.subjects, c.objects, sids, k, filt, wl)
    n_pos = n if wl is None else len(wl)
    assert ids.shape == (len(sids), min(n_pos, k or n_pos))
    pad = np.arange(ids.shape[1])[None, :] >= cnt[:, None]
    assert (ids[pad] == -1).all() and (sc[pad] == ec.NEG_MAX).all() and cnt[3] == 0
    # the flattened padded rows are rank_oracle's answer (COSINE: before the subject-norm division)
    subj, fid, fsc = flatten_padded(sids, ids, sc, cnt)
    es, eid, esc = rank_oracle(distance, c.subjects, c.objects, sids, k, filt, wl, accum="f64")
    np.testing.assert_array_equal(subj, es)
    np.testing.assert_array_equal(fid, eid)
    if distance == "cosine":
        fsc = fsc / ec.calc_norms(c.subjects, "f64")[subj]
    np.testing.assert_array_equal(fsc, esc)


def test_filter_keeping_leaves_the_requested_survivors():
    rng = np.random.default_rng(0)
    wl = np.arange(0, 500, 3)
    f = ec.filter_keeping(rng, 500, [0, 1, 31, 32, 33], candidates=wl)
    for r, s in enumerate([0, 1, 31, 32, 33]):
        assert len(np.setdiff1d(wl, f[r].indices)) == s


def test_expected_merge_is_merge_padded_numpy_on_the_entries_read():
    rng = np.random.default_rng(1)
    ids, sc, cnt = ec.merge_case(rng, 3, 40, 33)
    o_ids, o_sc, o_cnt, _ = ec.expected_merge(ids, sc, cnt, 33)
    # no garbage (score 1e9 beyond a count) and no pad id ever reaches the output
    assert (o_sc < 1e8).all() and not (o_ids == ec.PAD_ID).any()
    for r in range(40):
        ent = [(-float(sc[li, r, e]), int(ids[li, r, e])) for li in range(3) for e in range(cnt[li, r]) if ids[li, r, e] != ec.PAD_ID]
        ent.sort()
        ent = ent[:33]
        assert o_cnt[r] == len(ent)
        assert [i for _, i in ent] == o_ids[r, : o_cnt[r]].tolist()
        assert (o_ids[r, o_cnt[r] :] == -1).all()
    # without pad ids it is merge_padded_numpy itself
    clean = np.where(ids == ec.PAD_ID, 10**6, ids)
    np.testing.assert_array_equal(ec.expected_merge(clean, sc, cnt, 33)[0], merge_padded_numpy(clean, sc, cnt, 33)[0])


def test_expected_merge_certificate():
    inf = np.float32(np.inf)
    ids = np.array([[[1, 2, 3]], [[4, 5, 6]]], np.int32)
    sc = np.array([[[5, 4, 1]], [[3, 2, 0]]], np.float32)
    cases = [  # (counts, bounds, k, fails)
        ([[3], [3]], [[-inf], [-inf]], 3, False),
        ([[1], [0]], [[-inf], [-inf]], 3, False),  # short row, no bound: accept
        ([[1], [0]], [[-inf], [-5.0]], 3, True),  # short row, finite bound: reject
        ([[3], [3]], [[3.0], [-inf]], 3, True),  # bound == 3rd score: reject
        ([[3], [3]], [[np.nextafter(np.float32(3), np.float32(0))], [-inf]], 3, False),  # one ulp below: accept
    ]
    for counts, bounds, k, fails in cases:
        _, _, _, f = ec.expected_merge(ids, sc, np.array(counts, np.int32), k, np.array(bounds, np.float32))
        assert (len(f) == 1) == fails, (counts, bounds)


def test_strip_sentinel_tail_follows_the_reference():
    """The wrapper's trailing strip (rank_implicit.py:107-118): real scores <= neginf_score at the end of a row go."""
    lo = np.float32(ec.neginf_score())
    ids = np.array([[4, 2, 9], [1, 3, 5], [7, 8, -1]], np.int32)
    sc = np.array([[1.0, lo, ec.NEG_MAX], [2.0, 1.0, 0.0], [ec.NEG_MAX, ec.NEG_MAX, ec.NEG_MAX]], np.float32)
    cnt = np.array([3, 3, 2], np.int32)
    strip_sentinel_tail(ids, sc, cnt)
    np.testing.assert_array_equal(cnt, [1, 3, 0])
    np.testing.assert_array_equal(ids, [[4, -1, -1], [1, 3, 5], [-1, -1, -1]])
    assert (sc[0, 1:] == ec.NEG_MAX).all()
    # the oracle agrees on the d = 1 catalogue of extreme values
    objects = np.array([[-ec.FLT_MAX], [1.0], [lo], [-1.0], [np.nextafter(lo, np.float32(0))]], np.float32)
    _, oid, osc = rank_oracle("dot", np.ones((1, 1), np.float32), objects, [0], 5, accum="f64")
    assert oid.tolist() == [1, 3, 4]


def test_sparse_subjects_densify_with_summed_duplicates():
    rng = np.random.default_rng(2)
    d, n_obj = 50, 301
    objects = ec.int_matrix(rng, n_obj, d)
    cols = rng.integers(0, d, 600)
    x = sparse.csr_matrix((rng.integers(-3, 4, 600).astype(np.float32) / 2, cols, [0, 600]), shape=(1, d))
    assert not x.has_canonical_format
    ids, sc, cnt = ec.expected_padded("dot", x, objects, [0], 10)
    dense = np.zeros(d)
    np.add.at(dense, cols, x.data.astype(np.float64))
    s = objects.astype(np.float64) @ dense
    order = np.lexsort((np.arange(n_obj), -s))[:10]
    np.testing.assert_array_equal(ids[0], order)
    np.testing.assert_array_equal(sc[0], s[order].astype(np.float32))

"""CPU: the candidate-pass checker of tests/tc_reference.py, tested before it is trusted on a GPU.  A snapshot built by a
pure-numpy model of a correct pass must pass every invariant, and each kind of defect the kernel could have must be
reported under its own invariant."""
import numpy as np
import pytest
from scipy import sparse

from tests.helpers import synth_factors
from tests.tc_reference import (
    Catalogue,
    SharedPass,
    check_snapshot,
    list_of_positions,
    model_snapshot,
    peer_word,
    round16,
    round_up_f32,
    scale_exp,
    subject_operands,
)


def _case(cosine=False, bf16=False, whitelist=False, nw=8, n_splits=2, seed=0):
    n_rows, n_obj, d, k = 37, 3000, 40, 10
    u, i = synth_factors(n_rows, n_obj, d, seed=seed)
    wl = np.sort(np.random.default_rng(seed).choice(n_obj, 2100, replace=False)) if whitelist else None
    cat = Catalogue(i, cosine=cosine, bf16=bf16, whitelist=wl)
    rng = np.random.default_rng(seed + 1)
    cols = np.sort(rng.choice(cat.n_pos, size=(n_rows, 30)), axis=1)  # viewed positions (duplicates possible)
    viewed = sparse.csr_matrix((np.ones(cols.size, np.float32), cols.reshape(-1), np.arange(n_rows + 1) * 30), shape=(n_rows, cat.n_pos))
    viewed.sum_duplicates()
    kc = 12 if nw == 8 else 8
    snap = model_snapshot(cat, u, viewed, k_cand=kc, kp=k, k_out=k, nw=nw, n_splits=n_splits)
    return cat, u, viewed, snap


def _copy(snap):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in snap.items()}


def test_emulation_primitives():
    # exponent: amax * 2^e in [2^13, 2^14), the frexp edge at exact powers of two, zero / non-finite -> 0
    amax = np.array([1.0, 2.0, 0.75, 2.0**-140, 3e38, 0.0, np.inf, np.nan], np.float32)
    e = scale_exp(amax)
    scaled = np.ldexp(amax[:5].astype(np.float64), e[:5])
    assert ((scaled >= 2**13) & (scaled < 2**14)).all()
    assert e[1] == 12 and e[0] == 13 and list(e[5:]) == [0, 0, 0]
    # fp16 rounding: nearest even, subnormals kept, beyond the subnormal range -> 0
    x = np.array([1 + 2**-11, 1 + 3 * 2**-11, 2**-24, 2**-26, 3 * 2**-25], np.float32)
    np.testing.assert_array_equal(round16(x, False), [1.0, 1 + 2**-9, 2**-24, 0.0, 2**-23])
    np.testing.assert_array_equal(round16(np.array([1 + 2**-8], np.float32), True), [1.0])
    # list partition: quarters alternate between the two column groups, splits take whole tiles
    lop = list_of_positions(1000, 2, 2)
    assert lop[0] == 0 and lop[64] == 1 and lop[128] == 0 and lop[511] == 1 and lop[512] == 2 and lop[999] == 3


@pytest.mark.parametrize(
    "kw", [{}, {"cosine": True, "whitelist": True}, {"bf16": True, "n_splits": 1}, {"nw": 16, "n_splits": 3}], ids=["dot", "cos-wl", "bf16", "nw16"]
)
def test_model_snapshot_passes_every_invariant(kw):
    cat, u, viewed, snap = _case(**kw)
    rep = check_snapshot(snap, cat, u, viewed)
    assert rep.ok, rep.summary()
    assert rep.frac_acc < 0.01 and rep.frac_eps < 0.5 and rep.i3_margin <= 0
    assert snap["cand_counts"][:, :37].max() == snap["k_cand"]


def _pick(cat, snap, viewed, want_viewed):
    """(row, list, position) with a position of the list's set that is viewed (or eligible and unlisted)."""
    lpr = snap["nw"] // 4
    lop = list_of_positions(cat.n_pos, lpr, snap["tiles_per_split"])
    vm = viewed.toarray() != 0
    for r in range(snap["n_sel"]):
        listed = set(cat.pos_of_obj[snap["cand_ids"][0, r, : snap["cand_counts"][0, r]]].tolist())
        for p in np.nonzero(lop == 0)[0]:
            if vm[r, p] == want_viewed and p not in listed:
                return r, 0, int(p)
    raise AssertionError("no such position")


def test_checker_reports_each_kind_of_defect():
    cat, u, viewed, snap = _case()
    assert check_snapshot(snap, cat, u, viewed).ok

    def bad(mutate, cls):
        s = _copy(snap)
        mutate(s)
        rep = check_snapshot(s, cat, u, viewed)
        assert rep.counts[cls] > 0, f"{cls} not reported: {rep.summary()}"
        return rep

    # a viewed object in a list
    r, l, p = _pick(cat, snap, viewed, True)
    bad(lambda s: s["cand_ids"].__setitem__((l, r, 0), cat.pos2obj[p]), "I1")
    # an object of the other column group
    lop = list_of_positions(cat.n_pos, 2, snap["tiles_per_split"])
    other = int(np.nonzero((lop == 1) & (viewed[0].toarray()[0] == 0))[0][0])
    bad(lambda s: s["cand_ids"].__setitem__((0, 0, 0), cat.pos2obj[other]), "I1")
    # an id listed twice
    def dup(s):
        s["cand_ids"][0, 1, 1] = s["cand_ids"][0, 1, 0]
        s["cand_scores"][0, 1, 1] = s["cand_scores"][0, 1, 0]
    bad(dup, "I1")
    # a threshold lowered below the score of a discarded object
    r, l, p = _pick(cat, snap, viewed, False)
    a = float((subject_operands(u[r : r + 1], False)[1] @ cat.i16_pos[p])[0])
    rep = bad(lambda s: s["cand_thr"].__setitem__((slice(None), r), np.float32(a - 0.05 * abs(a) - 1.0)), "I3")
    assert rep.i3_margin > 1
    # a score off by more than the accumulation bound
    def perturb(s):
        s["cand_scores"][1, 2, 3] += np.float32(0.01 * abs(s["cand_scores"][1, 2, 3]) + 1.0)
    bad(perturb, "I2")
    # constants: a wrong object exponent, an eps_rel 64x too small, a wrong row exponent
    bad(lambda s: s.__setitem__("obj_exp", s["obj_exp"] + 1), "const")
    bad(lambda s: s.__setitem__("eps_rel", np.float32(s["eps_rel"] / 64)), "const")
    bad(lambda s: s["row_exp"].__setitem__(5, s["row_exp"][5] + 1), "const")
    # a row the restated verdict rejects but the engine certified (and the reverse)
    rep = check_snapshot(snap, cat, u, viewed)
    if rep.rejected:
        bad(lambda s: s.__setitem__("fb_rows", np.empty(0, np.int32)), "I5")
    bad(lambda s: s.__setitem__("fb_rows", np.setdiff1d(np.arange(37), rep.rejected).astype(np.int32)[:1]), "I5")


# ------------------------------------------------------------------------------------------------ threshold-sharing passes
EPOCH, ROW0, MAX_ROWS = 5, 3, 50


def _bound(x, old=False):
    """The shard bound of rescore_select_kernel from x = max tau (exact units) + eps; `old`: the factor (1 + 2.4e-7) the
    kernel used before, which moves a negative bound down."""
    return round_up_f32(x * (1.0 + 2.4e-7) + 1e-37) if old else round_up_f32(x + 2.4e-7 * np.abs(x) + 1e-37)


def _shared_case(negative=False, old_bound=False):
    """A shared pass of 37 rows at call rows [3, 40) of a 50-row published array: rows = 0 mod 3 received a peer value
    (their 8th best A_ref) before the pass started, so every list adopted it; `negative`: every score is negative."""
    n_rows, n_obj, d, k = 37, 3000, 40, 10
    u, i = synth_factors(n_rows, n_obj, d, seed=3)
    if negative:
        u, i = -np.abs(u), np.abs(i)
    cat = Catalogue(i, cosine=False, bf16=False)
    rng = np.random.default_rng(4)
    cols = np.sort(rng.choice(cat.n_pos, size=(n_rows, 30)), axis=1)
    viewed = sparse.csr_matrix((np.ones(cols.size, np.float32), cols.reshape(-1), np.arange(n_rows + 1) * 30), shape=(n_rows, cat.n_pos))
    viewed.sum_duplicates()
    A = subject_operands(u, False)[1] @ cat.i16_pos.T
    floor = np.full(n_rows, -np.inf)
    floor[::3] = np.float32(-np.sort(-A[::3], axis=1)[:, 7])  # (no list can fill its 9 slots above it)
    snap = model_snapshot(cat, u, viewed, k_cand=9, kp=k, k_out=k, peer_floor=floor)
    snap["rows"] = np.arange(ROW0, ROW0 + n_rows, dtype=np.int32)
    tmax = snap["cand_thr"][:, :n_rows].astype(np.float64).max(axis=0)
    eps = float(cat.eps_rel()) * np.sqrt(np.einsum("ij,ij->i", u, u, dtype=np.float64)) * float(cat.max_obj_norm)
    x = np.ldexp(tmax, -(snap["row_exp"] + cat.obj_exp)) + eps
    bounds = np.where(tmax > -np.inf, _bound(x, old_bound), -np.inf).astype(np.float32)
    before = np.full(MAX_ROWS, peer_word(0, np.float32(-1.0)), np.uint64)
    after = before.copy()
    pub = np.isfinite(tmax)
    after[ROW0 : ROW0 + n_rows][pub] = peer_word(EPOCH, np.ldexp(tmax[pub], -cat.obj_exp))
    words = peer_word(EPOCH, np.ldexp(floor, -cat.obj_exp))[None, :]
    shared = SharedPass(bounds, EPOCH, words, np.full(n_rows, -np.inf), before, after, ROW0 + n_rows)
    return cat, u, viewed, snap, shared, A


@pytest.mark.parametrize("negative", [False, True], ids=["mixed", "negative"])
def test_model_shared_pass_passes_every_invariant(negative):
    cat, u, viewed, snap, shared, _ = _shared_case(negative)
    rep = check_snapshot(snap, cat, u, viewed, shared=shared)
    assert rep.ok, rep.summary()
    assert rep.n_adopted == 2 * 13 and rep.adopted_rows == list(range(0, 37, 3)) and rep.n_published == 37
    assert (shared.bounds < 0).all() == negative


def test_checker_reports_each_kind_of_shared_defect():
    cat, u, viewed, snap, shared, A = _shared_case()

    def bad(cls, snap_=snap, shared_=shared):
        rep = check_snapshot(snap_, cat, u, viewed, shared=shared_)
        assert rep.counts[cls] > 0, f"{cls} not reported: {rep.summary()}"

    # a threshold raised above everything a list of the call could hold (row 1 has no peer value)
    s = _copy(snap)
    s["cand_thr"][1, 1] = np.float32(A[1].max() + 0.01 * abs(A[1].max()) + 1.0)
    bad("I6", s)
    # the shard's bound of a negative row, computed with the factor (1 + 2.4e-7): 2-4 ulps below max tau + eps
    cat_n, u_n, viewed_n, snap_n, shared_n, _ = _shared_case(negative=True)
    assert check_snapshot(snap_n, cat_n, u_n, viewed_n, shared=shared_n).ok
    _, _, _, _, shared_old, _ = _shared_case(negative=True, old_bound=True)
    assert (shared_old.bounds < shared_n.bounds).all()
    rep = check_snapshot(snap_n, cat_n, u_n, viewed_n, shared=shared_old)
    assert rep.counts["I7"] == 37, rep.summary()
    # a bound of -inf for a row that discarded objects, and a finite bound for a row that discarded nothing
    bad("I7", snap, shared._replace(bounds=np.where(np.arange(37) == 4, -np.inf, shared.bounds).astype(np.float32)))
    # every row published one slot too far (the last one beyond the call's rows)
    after = shared.pub_before.copy()
    after[ROW0 + 1 : ROW0 + 38] = shared.pub_after[ROW0 : ROW0 + 37]
    bad("I8", snap, shared._replace(pub_after=after))
    # a published word with another epoch
    after = shared.pub_after.copy()
    after[ROW0 + 2] = peer_word(EPOCH + 1, np.float32(-1.0))
    bad("I8", snap, shared._replace(pub_after=after))
    # a value of the wrong epoch that a list adopted
    huge = np.float32(np.ldexp(A[1].max() * 4 + 1.0, -cat.obj_exp))
    words = shared.peer_words.copy()
    words[0, 1] = peer_word(EPOCH + 1, huge)
    s = _copy(snap)
    s["cand_thr"][:, 1] = np.float32(np.ldexp(np.float64(huge), cat.obj_exp))
    bad("I6", s, shared._replace(peer_words=words))
    # ... which is justified when it carries the call's epoch
    words[0, 1] = peer_word(EPOCH, huge)
    rep = check_snapshot(s, cat, u, viewed, shared=shared._replace(peer_words=words))
    assert rep.counts["I6"] == 0 and 1 in rep.adopted_rows
    # a pass that shares thresholds gives no verdict
    bad("I5", dict(_copy(snap), fb_rows=np.array([ROW0 + 2], np.int32)))

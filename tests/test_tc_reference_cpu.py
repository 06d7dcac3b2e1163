"""CPU: the candidate-pass checker of tests/tc_reference.py, tested before it is trusted on a GPU.  A snapshot built by a
pure-numpy model of a correct pass must pass every invariant, and each kind of defect the kernel could have must be
reported under its own invariant."""
import numpy as np
import pytest
from scipy import sparse

from tests.helpers import synth_factors
from tests.tc_reference import Catalogue, check_snapshot, list_of_positions, model_snapshot, round16, scale_exp


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
    from tests.tc_reference import subject_operands

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

"""CPU: the rounding-interval oracle of `tests/score_interval.py` checks itself.

* Containment: the correctly rounded fp32 value of the exact rational sum, and of fp64 sums simulated in the orders the
  kernels and BLAS use (sequential, 32 lanes strided with an xor-shuffle tree as in `select.cuh`, pairwise, reversed),
  lie in [lo, hi], for DOT and COSINE, on random rows, cancelling rows and subnormal elements.
* Midpoints: exact sums on an fp32 rounding midpoint, or one fp64 ulp off it, are ambiguous, and the checker accepts both
  roundings.
* Tightness: the cut-deciding scores of synthetic factors are almost never ambiguous.
* The checker passes an oracle-exact result and fails each planted fault."""
from fractions import Fraction

import numpy as np
import pytest
from scipy import sparse

from tests.helpers import synth_factors, synth_viewed_csr
from tests.score_interval import (COSINE_ZERO_NORM, NEG_MAX, check_topk, exact_pairs, from_keys, norm_interval, order_keys,
                                  rn32, row_lsb_exponent, score_interval, widen64)


# ------------------------------------------------------------------------------------------------ exact and simulated sums
def rn32_exact(x: Fraction) -> np.float32:
    """Round-to-nearest-even of a rational to fp32 (no double rounding through fp64)."""
    c = np.float32(float(x))
    best = None
    for v in (np.nextafter(c, np.float32(-np.inf)), c, np.nextafter(c, np.float32(np.inf))):
        e = abs(Fraction(float(v)) - x)
        if best is None or e < best[0] or (e == best[0] and (int(v.view(np.uint32)) & 1) == 0):
            best = (e, v)
    return best[1] + np.float32(0)


def exact_dots(u: np.ndarray, o: np.ndarray) -> list:
    fu = [[Fraction(float(x)) for x in row] for row in u]
    fo = [[Fraction(float(x)) for x in row] for row in o]
    return [[sum((a * b for a, b in zip(ru, ro)), Fraction(0)) for ro in fo] for ru in fu]


def _seq(p: np.ndarray) -> np.ndarray:
    acc = np.zeros(p.shape[:-1])
    for j in range(p.shape[-1]):
        acc = acc + p[..., j]
    return acc


def _lanes(p: np.ndarray) -> np.ndarray:
    """32 lanes: lane l sums terms l, l+32, ... in order (fma == add of the exact product), then the xor-shuffle tree."""
    d = p.shape[-1]
    lanes = [_seq(p[..., l::32]) if l < d else np.zeros(p.shape[:-1]) for l in range(32)]
    for o in (16, 8, 4, 2, 1):
        lanes = [lanes[l] + lanes[l ^ o] for l in range(32)]
    return lanes[0]


def _pairwise(p: np.ndarray) -> np.ndarray:
    if p.shape[-1] == 1:
        return p[..., 0]
    h = p.shape[-1] // 2
    return _pairwise(p[..., :h]) + _pairwise(p[..., h:])


ORDERS = {"sequential": _seq, "lanes32_xor": _lanes, "pairwise": _pairwise, "reversed": lambda p: _seq(p[..., ::-1])}


def _inputs(d: int, seed: int):
    rng = np.random.default_rng(seed)
    u = (rng.standard_normal((6, d)) / np.sqrt(d)).astype(np.float32)
    o = (rng.standard_normal((9, d)) / np.sqrt(d)).astype(np.float32)
    if d > 1:
        h = d // 2
        # cancelling pairs: o[0] against u[0] sums to (nearly) zero, terms of very different size
        u[0, :h], u[0, h : 2 * h] = u[0, :h], -u[0, :h]
        o[0, :h] = o[0, h : 2 * h] * (1 + np.float32(2.0**-20) * rng.standard_normal(h).astype(np.float32))
        o[1] = (o[1] * 10.0 ** rng.uniform(-8, 8, d)).astype(np.float32)  # terms over 16 decades
    u[1, ::2] *= np.float32(1e-40)  # subnormal elements
    u[2] *= np.float32(1e-39)  # an all-subnormal row
    o[2, 1::2] *= np.float32(1e-41)
    o[3] = 0.0  # a zero object (COSINE: norm 1e-10)
    return u, o


@pytest.mark.parametrize("d", [1, 7, 64, 129, 320])
def test_every_summation_order_is_inside(d):
    u, o = _inputs(d, d)
    u64, o64 = widen64(u), widen64(o)
    lo, hi = score_interval(u64, o64)
    exact = exact_dots(u, o)
    prod = u64[:, None, :] * o64[None, :, :]  # exact in fp64
    for r in range(len(u)):
        for c in range(len(o)):
            x = rn32_exact(exact[r][c])
            assert lo[r, c] <= x <= hi[r, c], (r, c, x, lo[r, c], hi[r, c])
    for order, fn in ORDERS.items():
        s = rn32(fn(prod))
        assert ((s >= lo) & (s <= hi)).all(), order
    # COSINE: the norm in every order is inside the norm interval, and so is every quotient
    n_lo, n_hi = norm_interval(o64)
    clo, chi = score_interval(u64, o64, (n_lo, n_hi))
    sq = o64 * o64
    for order, fn in ORDERS.items():
        nrm = np.sqrt(fn(sq)).astype(np.float32)
        nrm = np.where(nrm == 0, COSINE_ZERO_NORM, nrm)
        assert ((nrm >= n_lo) & (nrm <= n_hi)).all(), order
        s = rn32(fn(prod) / nrm.astype(np.float64)[None, :])
        assert ((s >= clo) & (s <= chi)).all(), order
    for r in range(len(u)):
        for c in range(len(o)):
            for n in {n_lo[c], n_hi[c]}:
                x = rn32_exact(exact[r][c] / Fraction(float(n)))
                assert clo[r, c] <= x <= chi[r, c], (r, c, x, clo[r, c], chi[r, c])


def test_rounding_midpoints_are_ambiguous_and_both_outcomes_pass():
    """1 + 2^-24 is the midpoint of 1 and 1 + 2^-23; add 0 / +1 / -1 fp64 ulps (2^-52), at scales 2^e and both signs.
    Two cancelling terms of 2^-60 leave the exact sum alone but round away in some orders (no exact fp64 sum)."""
    rows, objs = [], []
    for e in (-60, -3, 0, 17):
        for sign in (1.0, -1.0):
            for off in (0.0, 2.0**-52, -(2.0**-52)):
                rows.append(np.float32(sign * 2.0**e) * np.ones(5, np.float32))
                objs.append(np.array([1.0, 2.0**-24, off, 2.0**-60, -(2.0**-60)], np.float32))
    u, o = np.array(rows), np.array(objs)
    lo, hi = score_interval(widen64(u), widen64(o))
    for r in range(len(u)):
        x = Fraction(float(u[r, 0])) * sum(Fraction(float(v)) for v in o[r])
        ends = {float(np.float32(u[r, 0])), float(np.float32(u[r, 0]) * np.nextafter(np.float32(1), np.float32(2)))}
        assert {float(lo[r, r]), float(hi[r, r])} == ends, r
        assert lo[r, r] <= rn32_exact(x) <= hi[r, r]
        # a one-row, one-object call: both neighbours of the midpoint are accepted as the score
        for v in (lo[r, r], hi[r, r]):
            got = (np.zeros((1, 1), np.int32), np.array([[v]], np.float32), np.ones(1, np.int32))
            rep = check_topk(got, u[r : r + 1], o[r : r + 1], 1, max_ambiguous=1.0, verbose=False)
            assert rep.amb_returned == 1


def test_the_bound_is_tight_on_synthetic_factors():
    """Ambiguity comes from scores near zero (cancellation); at the scores a top-k cut can fall on (each row's top 1 %)
    fewer than 1e-5 are ambiguous, and over all pairs fewer than 1e-4."""
    u, i = synth_factors(1000, 20_000, 64, seed=5)
    u64, i64 = widen64(u), widen64(i)
    lo, hi = score_interval(u64, i64)
    amb = lo != hi
    top = lo >= np.sort(lo, axis=1)[:, -200][:, None]
    print(f"ambiguous: {int(amb.sum())} of {amb.size} pairs, {int(amb[top].sum())} of {int(top.sum())} in the top 1 %")
    assert amb.mean() < 1e-4 and amb[top].mean() < 1e-5
    clo, chi = score_interval(u64, i64, norm_interval(i64))
    assert (clo != chi).mean() < 1e-4


def test_16bit_sums_are_exact_in_every_order():
    """bf16 x bf16 terms have at most 16 significant bits: their fp64 sums are exact in every order, so the interval is the
    one correctly rounded value, midpoints included (where a Delta > 0 would make them ambiguous)."""
    import torch

    u, i = synth_factors(200, 3_000, 64, seed=6)
    u16 = torch.from_numpy(u).to(torch.bfloat16)
    i16 = torch.from_numpy(i).to(torch.bfloat16)
    lo, hi = score_interval(widen64(u16), widen64(i16))
    assert (lo == hi).all()
    prod = widen64(u16)[:20, None, :] * widen64(i16)[None, :50, :]
    for order, fn in ORDERS.items():
        np.testing.assert_array_equal(rn32(fn(prod)), lo[:20, :50], err_msg=order)
    x = [[rn32_exact(v) for v in row] for row in exact_dots(widen64(u16)[:4], widen64(i16)[:30])]
    np.testing.assert_array_equal(np.array(x, np.float32), lo[:4, :30])
    # one term below the quantum of the others breaks exactness only where the sum needs more than 53 bits
    assert not exact_pairs(np.array([[2.0**60]]), np.array([0]), np.array([0]))[0, 0]
    assert exact_pairs(np.array([[2.0**52]]), np.array([0]), np.array([0]))[0, 0]


def test_csr_terms_keep_their_quantum():
    """Duplicate CSR columns are separate terms: the quantum of a row is that of its stored values, not of their sums
    (2^-24 + 2^-24 would look like a multiple of 2^-23)."""
    x = sparse.csr_matrix((np.float32([2.0**-24, 2.0**-24, 1.0, 3.0]), [0, 0, 1, 2], [0, 3, 3, 4]), shape=(3, 4))
    np.testing.assert_array_equal(row_lsb_exponent(x), [-24, 1 << 20, 0])
    np.testing.assert_array_equal(row_lsb_exponent(x.toarray())[[0, 2]], [-23, 0])


# ------------------------------------------------------------------------------------------------ the checker and its faults
N_ROWS, N_OBJ, D, K, ID_OFF = 40, 3000, 48, 12, 500


def _oracle_result(u, objects, k, viewed, wl, id_off, cosine=False):
    """An oracle-exact padded result: numpy's fp64 scores rounded once, top-k by (score desc, id asc)."""
    wl_ = np.arange(len(objects)) if wl is None else wl
    o64 = widen64(objects[wl_])
    s = widen64(u) @ o64.T
    if cosine:
        s = s / np.sqrt(np.einsum("ij,ij->i", o64, o64)).astype(np.float32).astype(np.float64)[None, :]
    s = rn32(s)
    gid = wl_ + id_off
    k_out = min(k, len(wl_))
    ids = np.full((len(u), k_out), -1, np.int32)
    sc = np.full((len(u), k_out), NEG_MAX, np.float32)
    cnt = np.zeros(len(u), np.int32)
    for r in range(len(u)):
        ok = ~np.isin(gid, viewed.indices[viewed.indptr[r] : viewed.indptr[r + 1]])
        keys = np.sort(order_keys(s[r, ok], gid[ok]))[:k_out]
        i_, s_ = from_keys(keys)
        cnt[r] = len(keys)
        ids[r, : len(keys)], sc[r, : len(keys)] = i_, s_
    return ids, sc, cnt


@pytest.fixture(scope="module")
def call():
    u, i = synth_factors(N_ROWS, N_OBJ, D, seed=8)
    i[100] = i[2000]  # two objects tied in every row: ids 600 and 2500
    u[5] = 3 * i[2000] / np.linalg.norm(i[2000]) ** 2  # row 5 ranks the tied pair first
    wl = np.sort(np.random.default_rng(1).choice(N_OBJ, 2400, replace=False))
    wl = np.union1d(wl, [100, 2000])
    viewed = synth_viewed_csr(N_ROWS, N_OBJ + ID_OFF, 40, seed=3)
    return u, i, wl, viewed


def _check(call, got, viewed=None, subjects=None, **kw):
    u, i, wl, v = call
    return check_topk(got, u if subjects is None else subjects, i, K, filter_csr=v if viewed is None else viewed, whitelist=wl, id_offset=ID_OFF, **kw)


def test_checker_passes_the_oracle(call):
    u, i, wl, viewed = call
    got = _oracle_result(u, i, K, viewed, wl, ID_OFF)
    assert (got[0][5, :2] == [100 + ID_OFF, 2000 + ID_OFF]).all()
    rep = _check(call, got)
    assert rep.n_rows == N_ROWS and rep.n_returned == N_ROWS * K
    assert rep.n_checked == sum(len(wl) - np.isin(wl + ID_OFF, viewed.indices[viewed.indptr[r] : viewed.indptr[r + 1]]).sum() for r in range(N_ROWS))
    # a short row: everything but 5 objects viewed, so counts fall below k
    short = sparse.lil_matrix(viewed)
    short[9] = 0
    short[9, np.setdiff1d(wl, wl[:5]) + ID_OFF] = 1
    short = sparse.csr_matrix(short)
    got = _oracle_result(u, i, K, short, wl, ID_OFF)
    assert got[2][9] == 5
    _check(call, got, viewed=short)
    # COSINE, and a CSR of subjects with duplicate columns
    _check(call, _oracle_result(u, i, K, viewed, wl, ID_OFF, cosine=True), cosine=True)
    # each row's first 5 columns stored twice at half the value (exact): the same sums, with more terms
    cols = np.concatenate([np.r_[np.arange(5), np.arange(D)] for _ in range(N_ROWS)])
    vals = np.concatenate([np.r_[u[r, :5] / 2, u[r, :5] / 2, u[r, 5:]] for r in range(N_ROWS)]).astype(np.float32)
    dup = sparse.csr_matrix((vals, cols, np.arange(N_ROWS + 1) * (D + 5)), shape=u.shape)
    assert dup.nnz == N_ROWS * (D + 5) and not dup.has_canonical_format
    _check(call, _oracle_result(u, i, K, viewed, wl, ID_OFF), subjects=dup)


def _mutants(call):
    u, i, wl, viewed = call
    got = _oracle_result(u, i, K, viewed, wl, ID_OFF)
    lo, hi = score_interval(widen64(u[:1]), widen64(i[[got[0][0, 3] - ID_OFF]]))
    assert lo[0, 0] == hi[0, 0]

    def copy():
        return tuple(a.copy() for a in got)

    m = copy()
    m[1][0, 3] = np.nextafter(m[1][0, 3], np.float32(-np.inf))  # one score one ulp low (still in order)
    yield "score_1ulp", m, viewed, "outside their interval"
    m = copy()
    m[0][5, :2] = m[0][5, 1::-1]  # two fp32-equal scores, ids in the wrong order
    yield "tie_order", m, viewed, "order"
    m = copy()
    m[0][3, :-1], m[1][3, :-1] = got[0][3, 1:], got[1][3, 1:]  # the best object dropped, the row shifted up
    r3 = _oracle_result(u[3:4], i, K + 1, viewed[3], wl, ID_OFF)
    m[0][3, -1], m[1][3, -1] = r3[0][0, K], r3[1][0, K]
    yield "dropped_best", m, viewed, "leaves out"
    lil = sparse.lil_matrix(viewed)
    lil[2, got[0][2, 4]] = 1  # a returned id is viewed
    yield "viewed_returned", copy(), sparse.csr_matrix(lil), "filtered ids"
    m = copy()
    m[2][6] -= 1  # one entry fewer counted (its slot padded)
    m[0][6, -1], m[1][6, -1] = -1, NEG_MAX
    yield "count_low", m, viewed, "counts|leaves out"


@pytest.mark.parametrize("fault", ["score_1ulp", "tie_order", "dropped_best", "viewed_returned", "count_low"])
def test_checker_catches(call, fault):
    for name, got, viewed, msg in _mutants(call):
        if name == fault:
            with pytest.raises(AssertionError, match=msg):
                _check(call, got, viewed=viewed, verbose=False)
            return
    raise AssertionError(fault)

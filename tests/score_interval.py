"""The rounding-interval oracle: for every (subject, object) pair, the set of fp32 scores any fp64 summation order can give,
and a strict checker of padded top-k results against it (plain numpy, test infrastructure only).

The engine's score is `fp32(sum_j fp64(u_j) * fp64(i_j))` (COSINE: the fp64 sum divided by the fp32 object norm before
the one rounding), with the sum taken in an order each kernel chooses.  A numpy fp64 product gives one such order, so an
exact comparison with it is no valid test: two orders can land on either side of an fp32 rounding boundary.  Instead:

* `S = U64 @ I64^T` and `A = |U64| @ |I64|^T` in fp64.  Any recursive fp64 summation of n terms is within `gamma * A`
  of the exact sum, with `gamma = (n+2) u / (1 - (n+2) u)`, `u = 2^-53` (two terms above the textbook `gamma_{n-1}` pay
  for the rounding of `A` and of `S -/+ Delta` themselves).  `Delta = 2 gamma A` covers the engine's order and numpy's,
  so the engine's fp64 sum lies in `[S - Delta, S + Delta]`, and as `fp32_rn` (`astype(np.float32)`) is monotone, its
  score lies in `[lo, hi] = [fp32_rn(S - Delta), fp32_rn(S + Delta)]`.
* fma needs no special case: the product of two fp32 values (or fp16 / bf16 values, widened exactly) has at most 48
  significant bits and is exact in fp64, so `fma(a, b, acc) == acc + a*b` and the bound covers fma chains, shuffle
  trees and BLAS blocking alike.  (No product underflows: the smallest is 2^-298.)
* COSINE: the object norm is `fp32(sqrt(Q))` of an fp64 sum of squares, zero replaced by 1e-10f (`prep.cuh`,
  `row_stats_kernel`); its interval is `fp32_rn(sqrt(Q -/+ Delta_Q))`.  The score interval is `fp32_rn` of the min and
  max of the fp64 quotients `(S -/+ Delta) / n_{lo,hi}` at the four corners, each widened by 2 fp64 ulps.

Where every term is a multiple of a common power of two Q and `A < 2^53 Q` (16-bit factors usually, small integers
always), every partial sum is representable, every order gives the exact sum, and `Delta = 0`.

Almost always `lo == hi`: the check is bit-exact.  Where `lo != hi` the exact sum sits within `Delta` of an fp32
rounding boundary; the checker accepts either value and counts the entry as ambiguous.  The counts are reported so that
a bound grown loose cannot make the check vacuous."""
from __future__ import annotations

import typing as tp

import numpy as np
from scipy import sparse

U64 = 2.0**-53
NEG_MAX = np.float32(-np.finfo(np.float32).max)
COSINE_ZERO_NORM = np.float32(1e-10)
ELEMENTS_PER_BLOCK = 1 << 23


def gamma(n_terms: int) -> float:
    t = (int(n_terms) + 2) * U64
    return t / (1.0 - t)


def widen64(x: tp.Any) -> np.ndarray:
    """A numpy array or a CPU torch tensor of any float type (fp32, fp16, bf16) as fp64, exactly."""
    if hasattr(x, "double"):
        return x.double().numpy()
    return np.asarray(x).astype(np.float64)


def lsb_exponent(x: np.ndarray) -> np.ndarray:
    """Per row of `x` (fp32 values, in any float type): the exponent of the smallest unit in the last place among its
    nonzero elements, so that every element is an integer multiple of 2^e; a row of zeros gives a large value."""
    bits = np.ascontiguousarray(x, np.float32).view(np.int32) & np.int32(0x7FFFFFFF)
    ef = bits >> 23
    m = (bits & np.int32(0x7FFFFF)) | np.where(ef > 0, np.int32(1 << 23), np.int32(0))
    low = m & -m  # the lowest set bit of the significand, a power of two
    ctz = (low.astype(np.float32).view(np.int32) >> 23) - 127
    e = np.where(bits != 0, np.maximum(ef, 1) - 150 + ctz, np.int32(1 << 20))
    return e.min(axis=1).astype(np.int64) if e.shape[1] else np.full(e.shape[0], 1 << 20, np.int64)


def row_lsb_exponent(x: tp.Any) -> np.ndarray:
    """`lsb_exponent` of dense rows, or of the stored terms of each CSR row (duplicate columns are separate terms: their
    sum is never formed)."""
    if not sparse.issparse(x):
        return lsb_exponent(x)
    e = np.full(x.shape[0], 1 << 20, np.int64)
    nz = np.diff(x.indptr) > 0
    if nz.any():
        per_term = lsb_exponent(np.asarray(x.data, np.float32)[:, None])
        e[nz] = np.minimum.reduceat(per_term, x.indptr[:-1][nz])
    return e


def exact_pairs(a: np.ndarray, e_sub: np.ndarray, e_obj: np.ndarray) -> np.ndarray:
    """Pairs whose fp64 sum is exact in ANY order: every term is a multiple of Q = 2^(e_sub + e_obj) and every partial sum
    is at most A < 2^53 Q in magnitude, so each partial sum is representable.  (16-bit factors, small integers.)"""
    e_sub, e_obj = (np.clip(np.asarray(e, np.int64), -1100, 1100) for e in (e_sub, e_obj))
    if not e_sub.size or not e_obj.size or not (a < np.ldexp(1.0, int(min(e_sub.max() + e_obj.max() + 53, 1000)))).any():
        return np.zeros(a.shape, bool)  # (the common case for fp32 factors: no pair can be exact)
    return a < np.ldexp(1.0, np.clip(e_sub[:, None] + e_obj[None, :] + 53, -1000, 1000).astype(np.int32))


def rn32(x: np.ndarray) -> np.ndarray:
    """fp32 round-to-nearest of fp64 values, with -0.0 read as +0.0 (the sign of a zero score is not part of a result)."""
    return np.asarray(x).astype(np.float32) + np.float32(0)


def _widen_interval(lo: np.ndarray, hi: np.ndarray, ulps: int) -> tp.Tuple[np.ndarray, np.ndarray]:
    for _ in range(ulps):
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
    return lo, hi


def norm_interval(objects64: np.ndarray) -> tp.Tuple[np.ndarray, np.ndarray]:
    """The fp32 object norms any fp64 summation of the squares can give (zero -> 1e-10f), as (lo, hi) fp32 arrays."""
    q = np.einsum("ij,ij->i", objects64, objects64)
    dq = 2.0 * gamma(objects64.shape[1]) * q * (1.0 + 4.0 * U64)
    e = lsb_exponent(objects64)
    dq[q < np.ldexp(1.0, np.clip(2 * e + 53, -1000, 1000).astype(np.int32))] = 0.0  # (see `exact_pairs`)
    lo = np.sqrt(q - dq).astype(np.float32)
    hi = np.sqrt(q + dq).astype(np.float32)
    lo = np.where(lo == 0, COSINE_ZERO_NORM, lo)  # (zero -> 1e-10 is not monotone: order the two ends again)
    hi = np.where(hi == 0, COSINE_ZERO_NORM, hi)
    return np.minimum(lo, hi), np.maximum(lo, hi)


def score_interval(subjects: tp.Any, objects64: np.ndarray, norms: tp.Optional[tp.Tuple[np.ndarray, np.ndarray]] = None,
                   e_sub: tp.Optional[np.ndarray] = None, e_obj: tp.Optional[np.ndarray] = None) -> tp.Tuple[np.ndarray, np.ndarray]:
    """(lo, hi) fp32 [n, m] of every pair of `subjects` (fp64 [n, d], or a CSR [n, d] whose duplicate columns are separate
    terms) and `objects64` (fp64 [m, d]).  `norms`: the `norm_interval` of the objects, for COSINE.  `e_sub` / `e_obj`:
    their `lsb_exponent`s, when already known."""
    if sparse.issparse(subjects):
        sub = sparse.csr_matrix(subjects, dtype=np.float64)
        s = np.asarray(sub @ objects64.T)
        a = np.asarray(abs(sub) @ np.abs(objects64).T)
        n_terms = max(1, int(np.diff(sub.indptr).max())) if sub.shape[0] else 1
    else:
        s = subjects @ objects64.T
        a = np.abs(subjects) @ np.abs(objects64).T
        n_terms = max(1, objects64.shape[1])
    if e_sub is None:
        e_sub = row_lsb_exponent(subjects)
    exact = exact_pairs(a, e_sub, lsb_exponent(objects64) if e_obj is None else e_obj)
    delta = a
    delta *= 2.0 * gamma(n_terms) * (1.0 + 4.0 * U64)
    delta[exact] = 0.0
    lo64, hi64 = s - delta, s
    hi64 += delta
    if norms is not None:
        n_lo, n_hi = (n.astype(np.float64)[None, :] for n in norms)
        corners = (lo64 / n_lo, lo64 / n_hi, hi64 / n_lo, hi64 / n_hi)
        lo64, hi64 = _widen_interval(np.minimum.reduce(corners), np.maximum.reduce(corners), 2)
    return rn32(lo64), rn32(hi64)


def order_keys(scores: np.ndarray, ids: np.ndarray) -> np.ndarray:
    """uint64 keys whose ascending order is (score desc, id asc): the high word inverts the monotone map of the fp32 bit
    pattern, the low word is the id (-0.0 keys after +0.0: add +0.0 to the scores first to hold them equal)."""
    u = np.ascontiguousarray(scores, np.float32).view(np.uint32)
    mono = np.where(u >> 31, ~u, u | np.uint32(0x80000000)).astype(np.uint32)  # ascending in the score
    return ((~mono).astype(np.uint64) << np.uint64(32)) | np.asarray(ids).astype(np.uint64)


def from_keys(keys: np.ndarray) -> tp.Tuple[np.ndarray, np.ndarray]:
    ids = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    inv = ~(keys >> np.uint64(32)).astype(np.uint32)
    bits = np.where(inv >> 31, inv & np.uint32(0x7FFFFFFF), ~inv).astype(np.uint32)
    return ids, bits.view(np.float32)


# ------------------------------------------------------------------------------------------------ the strict checker
class Report:
    """What a check saw: eligible (row, object) pairs scored, returned entries, and the ambiguous ones (`lo != hi`):
    among the returned scores, among the objects left out whose interval reaches the k-th score (near the cut), and among
    all pairs."""

    def __init__(self, name: str) -> None:
        self.name = name
        self.n_rows = self.n_checked = self.n_returned = 0
        self.amb_returned = self.amb_cut = self.amb_all = 0

    @property
    def n_ambiguous(self) -> int:
        return self.amb_returned + self.amb_cut

    def summary(self) -> str:
        return (f"{self.name}: {self.n_rows} rows, {self.n_checked} entries checked, {self.n_returned} returned, ambiguous "
                f"{self.n_ambiguous} ({self.amb_returned} returned + {self.amb_cut} near the cut), {self.amb_all} of all")


def _filter_arrays(filter_csr: tp.Any, n_rows: int) -> tp.Tuple[np.ndarray, np.ndarray]:
    if filter_csr is None:
        return np.zeros(n_rows + 1, np.int64), np.empty(0, np.int64)
    if sparse.issparse(filter_csr):
        filter_csr = (filter_csr.indptr, filter_csr.indices)
    indptr, indices = (np.asarray(a, np.int64) for a in filter_csr)
    assert len(indptr) == n_rows + 1, "the filter needs one row per result row"
    return indptr - indptr[0], indices[indptr[0] : indptr[-1]]


def check_topk(
    got: tp.Tuple[np.ndarray, np.ndarray, np.ndarray],
    subjects: tp.Any,
    objects: tp.Any,
    k: tp.Optional[int],
    cosine: bool = False,
    filter_csr: tp.Any = None,
    whitelist: tp.Optional[np.ndarray] = None,
    id_offset: int = 0,
    name: str = "",
    max_ambiguous: float = 1e-4,
    verbose: bool = True,
) -> Report:
    """Check a padded engine result `got = (ids [n, k_out], scores, counts [n])` of every row against the score intervals.

    `subjects`: the batch rows, dense [n, d] (any float type) or a CSR [n, d]; `objects`: the engine's catalogue [N, d]
    (numpy or CPU torch, any float type); `filter_csr`: a CSR or (indptr, indices) of GLOBAL object ids per row (ids of
    other shards ignored); `whitelist`: sorted local object ids, the positions of the call; `id_offset`: added to local
    ids in the result.  Per row:
      1. counts == min(k_out, eligible positions), unfilled slots are id -1 / score -FLT_MAX;
      2. returned ids are eligible (in the shard, whitelisted, not filtered) and unique;
      3. each returned score lies in [lo, hi] of its id;
      4. the row is strictly ordered by (score desc, id asc);
      5. every eligible object not returned ranks after the k-th entry (s_k, id_k), judged by (lo, id).
    Asserts, and returns the `Report`; the ambiguous entries must stay below `max_ambiguous` of the checked ones."""
    ids, sc, cnt = (np.asarray(a) for a in got)
    n = ids.shape[0]
    n_obj = objects.shape[0]
    wl = None if whitelist is None else np.asarray(whitelist, np.int64)
    n_pos = n_obj if wl is None else len(wl)
    k_out = min(n_pos if k is None else int(k), n_pos)
    assert ids.shape == (n, k_out) and sc.shape == (n, k_out) and cnt.shape == (n,), f"{name}: shapes {ids.shape} {sc.shape} {cnt.shape}"
    dense_sub = not sparse.issparse(subjects)
    sub_all = widen64(subjects) if dense_sub else sparse.csr_matrix(subjects, dtype=np.float64)
    assert sub_all.shape[0] == n, f"{name}: {sub_all.shape[0]} subject rows for {n} result rows"
    rep = Report(name)
    rep.n_rows = n

    # ---- 1, 2, 4: padding, eligibility, uniqueness and order of the returned entries
    cnt = cnt.astype(np.int64)
    assert ((cnt >= 0) & (cnt <= k_out)).all(), f"{name}: counts out of range"
    valid = np.arange(k_out)[None, :] < cnt[:, None]
    assert (ids[~valid] == -1).all(), f"{name}: unfilled slots hold ids"
    assert (sc[~valid].view(np.uint32) == NEG_MAX.view(np.uint32)).all(), f"{name}: unfilled slots hold scores"
    local = ids.astype(np.int64) - int(id_offset)
    bad = valid & ((local < 0) | (local >= n_obj))
    assert not bad.any(), f"{name}: ids outside the shard at {np.argwhere(bad)[:5].tolist()}"
    if wl is None:
        pos_of_obj = None
        pos = np.where(valid, local, -1)
    else:
        pos_of_obj = np.full(n_obj, -1, np.int64)
        pos_of_obj[wl] = np.arange(len(wl))
        pos = np.where(valid, pos_of_obj[np.clip(local, 0, n_obj - 1)], -1)
        bad = valid & (pos < 0)
        assert not bad.any(), f"{name}: ids outside the whitelist at {np.argwhere(bad)[:5].tolist()}"
    srt = np.sort(np.where(valid, pos, -1 - np.arange(k_out)[None, :]), axis=1)
    dup = (srt[:, 1:] == srt[:, :-1]) & (srt[:, 1:] >= 0)
    assert not dup.any(), f"{name}: repeated ids in rows {np.nonzero(dup.any(axis=1))[0][:5].tolist()}"
    f_ptr, f_idx = _filter_arrays(filter_csr, n)
    for r in np.nonzero(np.diff(f_ptr) > 0)[0]:
        hit = np.isin(ids[r, : cnt[r]], f_idx[f_ptr[r] : f_ptr[r + 1]])
        assert not hit.any(), f"{name}: row {r} returns filtered ids {ids[r, : cnt[r]][hit][:5].tolist()}"
    keys = order_keys(np.where(valid, sc, NEG_MAX) + np.float32(0), np.where(valid, ids, 0).astype(np.int64))
    bad = valid[:, 1:] & (keys[:, 1:] <= keys[:, :-1])
    if bad.any():
        r, c = np.argwhere(bad)[0]
        raise AssertionError(f"{name}: row {r} out of (score desc, id asc) order at slot {c + 1}: "
                             f"({sc[r, c]!r}, {ids[r, c]}) then ({sc[r, c + 1]!r}, {ids[r, c + 1]})")
    # the k-th entry of each row; a row with fewer entries must hold every eligible object (-inf ranks after all)
    full = cnt == k_out
    s_k = np.where(full, sc[:, k_out - 1] if k_out else 0, -np.inf).astype(np.float32)
    id_k = np.where(full, ids[:, k_out - 1] if k_out else 0, -1).astype(np.int64)

    # ---- 3, 5: scores and completeness over blocks of positions
    pos2obj = np.arange(n_obj, dtype=np.int64) if wl is None else wl
    pb = max(1, min(n_pos, 1 << 18))
    rb = max(1, min(n, ELEMENTS_PER_BLOCK // pb))
    ret_lo = np.zeros((n, k_out), np.float32)
    ret_hi = np.zeros((n, k_out), np.float32)
    n_elig = np.zeros(n, np.int64)
    row_blocks = []
    for r0 in range(0, n, rb):
        r1 = min(r0 + rb, n)
        # the returned entries of these rows, by position
        rr, ss = np.nonzero(valid[r0:r1])
        rp = pos[r0:r1][rr, ss]
        o = np.argsort(rp, kind="stable")
        # the filtered pairs of these rows, as positions
        fr = np.repeat(np.arange(r1 - r0), np.diff(f_ptr[r0 : r1 + 1]))
        fl = f_idx[f_ptr[r0] : f_ptr[r1]] - int(id_offset)
        keep = (fl >= 0) & (fl < n_obj)
        fr, fl = fr[keep], fl[keep]
        fp = fl if pos_of_obj is None else pos_of_obj[fl]
        sub = sub_all[r0:r1]
        e_sub = row_lsb_exponent(sub)
        row_blocks.append((r0, r1, sub, e_sub, rr[o], ss[o], rp[o], fr[fp >= 0], fp[fp >= 0]))
    for p0 in range(0, n_pos, pb):
        p1 = min(p0 + pb, n_pos)
        obj64 = widen64(objects[p0:p1] if wl is None else objects[wl[p0:p1]])
        norms = norm_interval(obj64) if cosine else None
        e_obj = lsb_exponent(obj64)
        gid = pos2obj[p0:p1] + int(id_offset)
        for r0, r1, sub, e_sub, rr, ss, rp, fr, fp in row_blocks:
            lo, hi = score_interval(sub, obj64, norms, e_sub, e_obj)
            elig = np.ones(lo.shape, bool)
            m = (fp >= p0) & (fp < p1)
            elig[fr[m], fp[m] - p0] = False
            a, b = np.searchsorted(rp, [p0, p1])
            ret = np.zeros(lo.shape, bool)
            ret[rr[a:b], rp[a:b] - p0] = True
            ret_lo[r0 + rr[a:b], ss[a:b]] = lo[rr[a:b], rp[a:b] - p0]
            ret_hi[r0 + rr[a:b], ss[a:b]] = hi[rr[a:b], rp[a:b] - p0]
            out = elig & ~ret
            # (lo, id) before (s_k, id_k) in (score desc, id asc) order
            sk = s_k[r0:r1, None]
            viol = out & ((lo > sk) | ((lo == sk) & (gid[None, :] < id_k[r0:r1, None])))
            if viol.any():
                r, c = np.argwhere(viol)[0]
                rg = r0 + r
                raise AssertionError(
                    f"{name}: row {rg} leaves out id {gid[c]} with score in [{lo[r, c]!r}, {hi[r, c]!r}], which ranks before "
                    f"its last entry ({sc[rg, cnt[rg] - 1] if cnt[rg] else None!r}, {ids[rg, cnt[rg] - 1] if cnt[rg] else None}) "
                    f"(count {cnt[rg]} of k {k_out}; {int(viol.sum())} such pairs in this block)")
            amb = lo != hi
            n_elig[r0:r1] += elig.sum(axis=1)
            rep.amb_all += int((amb & elig).sum())
            rep.amb_cut += int((out & amb & (hi >= sk)).sum())

    # ---- 1, 3: counts and returned scores
    exp_cnt = np.minimum(n_elig, k_out)
    bad = np.nonzero(cnt != exp_cnt)[0]
    assert len(bad) == 0, f"{name}: counts {cnt[bad[:5]].tolist()} where {exp_cnt[bad[:5]].tolist()} positions are eligible (rows {bad[:5].tolist()})"
    bad = valid & ~((sc >= ret_lo) & (sc <= ret_hi))
    if bad.any():
        r, c = np.argwhere(bad)[0]
        raise AssertionError(f"{name}: {int(bad.sum())} scores outside their interval; row {r} slot {c} id {ids[r, c]}: "
                             f"{sc[r, c]!r} not in [{ret_lo[r, c]!r}, {ret_hi[r, c]!r}]")
    rep.n_checked = int(n_elig.sum())
    rep.n_returned = int(cnt.sum())
    rep.amb_returned = int((valid & (ret_lo != ret_hi)).sum())
    if verbose:
        print(rep.summary())
    assert rep.n_ambiguous <= max_ambiguous * max(rep.n_checked, 1), rep.summary()
    return rep

"""Plain numpy restatement of one tensor-core candidate pass, and a checker of the premises its certificate rests on.

The fused kernel (rectools_b200/csrc/fused_topk.cuh) scores 16-bit copies of the factors on the tensor cores and keeps,
per subject row and candidate list, the best APPROXIMATE scores.  The re-score kernels (select.cuh) recompute the
candidates exactly and accept a row when its kp-th exact score lies above every list's final threshold plus eps.  That
certificate is sound only if
  (P1) |approx - exact| <= eps = eps_rel * |u|_2 * max_i |i|_2, and
  (P2) a list's final threshold is at least the approximate score of every object the list discarded.
A row that breaks either premise can be certified with a wrong answer; a list that is merely worse than it should be
makes rows fail their certificate and take the (exact, slow) re-rank, which no end-to-end comparison notices.
`check_snapshot` tests the premises, the list contents and the verdict on every row and list of a pass captured with
B200_TC_SNAPSHOT (`Engine.candidate_snapshot`).  Nothing here calls the engine: it is numpy, in fp64 where it matters.

A pass of an item-sharded call that shares thresholds (B200_Q_SHARED_THRESHOLDS) gives no verdict: it reports a bound
per row instead, and its lists may prune with the other shards' published thresholds.  With `shared=SharedPass(...)`
the checker also tests that every threshold is justified by some shard's lists or a valid peer value (I6), restates
the bound in fp64 (I7) and checks what the pass published for the other shards (I8).  Published words are
(epoch << 32 | fp32 bits) in units of exact score * 2^row_exp, i.e. a shard's approximate units times 2^-obj_exp.
"""
from __future__ import annotations

import typing as tp

import numpy as np
from scipy import sparse

TILE_N = 256  # object positions per tile of the stream
QUART_N = 64  # positions per quarter (one MMA pass); quarter q of a tile belongs to column group q % lists-per-row
KBLK = 64  # d is padded to a multiple of this
PAD_ID = 0x7FFFFFFF
ACC_REL = 2.0**-21  # tensor-core accumulation bound per padded column (the d_pad term of eps_rel)
COSINE_MAX_NORM = np.float32(1.0000005)  # max_i |i|_2 of pre-normalised COSINE objects (prep.cuh)


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def scale_exp(amax: np.ndarray) -> np.ndarray:
    """fp16 operand scaling (prep.cuh `fp16_scale_exp`): e with amax * 2^e in [2^13, 2^14), i.e. 14 - frexp(amax).exp;
    0 when amax is 0 or not finite."""
    amax = np.asarray(amax, dtype=np.float32)
    ok = (amax > 0) & np.isfinite(amax)
    _, ex = np.frexp(np.where(ok, amax, np.float32(1)))
    return np.where(ok, 14 - ex, 0).astype(np.int32)


def round16(x32: np.ndarray, bf16: bool) -> np.ndarray:
    """fp32 -> fp16 / bf16, round to nearest even (subnormals included), returned widened to fp64."""
    x32 = np.ascontiguousarray(x32, dtype=np.float32)
    if bf16:
        import torch

        return torch.from_numpy(x32).to(torch.bfloat16).to(torch.float64).numpy()
    return x32.astype(np.float16).astype(np.float64)


def eps_rel(d: int, d_pad: int, bf16: bool) -> np.float32:
    """(2 rho + rho^2 + d_pad 2^-21 + sqrt(d) 2^-36) in fp32, rho = 2^-11 (fp16) / 2^-9 (bf16)."""
    rho = 2.0**-9 if bf16 else 2.0**-11
    return np.float32(2 * rho + rho * rho + d_pad * ACC_REL + np.sqrt(d) * 2.0**-36)


def norms_f32(x: np.ndarray) -> np.ndarray:
    """fp32 row norms accumulated in fp64 (prep.cuh `row_stats_kernel`), before the zero guard."""
    return np.sqrt(np.einsum("ij,ij->i", x, x, dtype=np.float64)).astype(np.float32)


def subject_operands(sub32: np.ndarray, bf16: bool) -> tp.Tuple[np.ndarray, np.ndarray]:
    """Per-row exponents and 16-bit subject rows (fp64 values, scaled units), as `convert_rows_kernel<T, true>`: both
    operand types are scaled."""
    sub32 = np.ascontiguousarray(sub32, dtype=np.float32)
    e = scale_exp(np.abs(sub32).max(axis=1) if sub32.shape[1] else np.zeros(len(sub32), np.float32))
    return e, round16(np.ldexp(sub32, e[:, None]).astype(np.float32), bf16)


class Catalogue:
    """The object side of a pass: 16-bit operand copy, exponent and norms of an engine's catalogue, seen through the
    positions of a call (whitelist entries, or every object)."""

    def __init__(self, objects: np.ndarray, cosine: bool, bf16: bool, whitelist: tp.Optional[np.ndarray] = None, id_off: int = 0):
        obj = np.ascontiguousarray(objects, dtype=np.float32)
        self.n_obj, self.d = obj.shape
        self.d_pad = round_up(self.d, KBLK)
        self.cosine, self.bf16, self.id_off = cosine, bf16, int(id_off)
        raw = norms_f32(obj)
        self.norms = np.where(raw == 0, np.float32(1e-10), raw).astype(np.float32)
        amax = np.abs(obj).max(axis=1) if self.d else np.zeros(self.n_obj, np.float32)
        if cosine:
            x = (obj / self.norms[:, None]).astype(np.float32)  # fp32 division, as the conversion kernel
            amax = (amax / self.norms).astype(np.float32)
            self.max_obj_norm = COSINE_MAX_NORM if (raw != 0).any() else np.float32(0)
        else:
            x = obj
            fin = raw[np.isfinite(raw)]
            self.max_obj_norm = np.float32(fin.max()) if fin.size else np.float32(0)
        fin = amax[np.isfinite(amax)]
        absmax = np.float32(fin.max()) if fin.size else np.float32(0)
        self.obj_exp = int(scale_exp(absmax))
        i16 = round16(np.ldexp(x, self.obj_exp).astype(np.float32), bf16)
        self.i16_norm_max = float(np.sqrt(np.einsum("ij,ij->i", i16, i16).max())) if self.n_obj else 0.0
        self.pos2obj = np.arange(self.n_obj, dtype=np.int64) if whitelist is None else np.asarray(whitelist, dtype=np.int64)
        self.n_pos = len(self.pos2obj)
        self.pos_of_obj = np.full(self.n_obj, -1, dtype=np.int64)
        self.pos_of_obj[self.pos2obj] = np.arange(self.n_pos)
        self.i16_pos = np.ascontiguousarray(i16[self.pos2obj])
        self.obj64_pos = obj[self.pos2obj].astype(np.float64)
        self.norm64_pos = self.norms[self.pos2obj].astype(np.float64) if cosine else None

    def eps_rel(self) -> np.float32:
        return eps_rel(self.d, self.d_pad, self.bf16)

    def exact(self, sub32: np.ndarray, pos: np.ndarray) -> np.ndarray:
        """Exact scores (fp64, before the final fp32 rounding) of subject rows sub32[i] with positions pos[i]."""
        s = np.einsum("ij,ij->i", np.asarray(sub32, np.float64), self.obj64_pos[pos])
        return s if self.norm64_pos is None else s / self.norm64_pos[pos]

    def viewed_positions(self, indptr: np.ndarray, indices: np.ndarray, n_rows: int) -> sparse.csr_matrix:
        """filter_pairs_csr (GLOBAL object ids; ids of other shards / beyond the catalogue ignored) -> [n_rows, n_pos] mask."""
        indptr = np.asarray(indptr, dtype=np.int64)
        rows = np.repeat(np.arange(n_rows), np.diff(indptr))
        local = np.asarray(indices, dtype=np.int64)[indptr[0] : indptr[-1]] - self.id_off
        keep = (local >= 0) & (local < self.n_obj)
        rows, local = rows[keep], local[keep]
        pos = self.pos_of_obj[local]
        keep = pos >= 0
        m = sparse.csr_matrix((np.ones(int(keep.sum()), np.float32), (rows[keep], pos[keep])), shape=(n_rows, self.n_pos))
        m.sum_duplicates()
        return m


def list_of_positions(n_pos: int, lists_per_row: int, tiles_per_split: int) -> np.ndarray:
    """List l = split * lists_per_row + g owns the positions of its split's tiles whose quarter q has q % lists_per_row == g."""
    p = np.arange(n_pos, dtype=np.int64)
    split = (p // TILE_N) // tiles_per_split
    g = ((p // QUART_N) % 4) % lists_per_row
    return split * lists_per_row + g


class Report:
    """Violations per invariant (a few examples each) and the observed margins."""

    CLASSES = ("const", "I1", "I2", "I3", "I4", "I5", "I6", "I7", "I8")

    def __init__(self) -> None:
        self.violations: tp.Dict[str, tp.List[str]] = {c: [] for c in self.CLASSES}
        self.counts: tp.Dict[str, int] = {c: 0 for c in self.CLASSES}
        self.frac_acc = 0.0  # max |cand - A_ref| / (d_pad 2^-21 |u16| max|i16|)
        self.frac_eps = 0.0  # max |approx - exact| / eps
        self.i3_margin = -np.inf  # max (best discarded A_ref - tau) / accumulation bound
        self.n_rows = self.n_lists = self.n_overflow = self.n_fb = self.n_rejected = self.n_tolerated = 0
        self.rejected: tp.List[int] = []  # batch rows the restated verdict rejects
        # shared mode: lists of rows with a valid peer value / of those, lists whose final tau IS that value (converted);
        # rows of the pass whose published slot was written
        self.n_peer_lists = self.n_adopted = self.n_published = 0
        self.adopted_rows: tp.List[int] = []  # batch rows with at least one list that adopted the peer value

    def add(self, cls: str, msg: str, n: int = 1) -> None:
        self.counts[cls] += n
        if len(self.violations[cls]) < 8:
            self.violations[cls].append(msg)

    @property
    def ok(self) -> bool:
        return not any(self.counts.values())

    def summary(self) -> str:
        bad = {c: n for c, n in self.counts.items() if n}
        return (
            f"rows={self.n_rows} lists={self.n_lists} frac_acc={self.frac_acc:.3g} frac_eps={self.frac_eps:.3g} "
            f"i3_margin={self.i3_margin:.3g} overflow={self.n_overflow} fb={self.n_fb} rejected={self.n_rejected} "
            f"tolerated={self.n_tolerated} adopted={self.n_adopted}/{self.n_peer_lists} published={self.n_published}"
            + (f" VIOLATIONS={bad} {self.violations}" if bad else "")
        )


class SharedPass(tp.NamedTuple):
    """What a threshold-sharing pass adds to its snapshot (all rows in the pass's batch order).

    bounds      [n_sel] fp32   the pass's `out_bounds`
    epoch                      the call's peer_epoch
    peer_words  [n_peers, n_sel] uint64  each peer's word of the row, as the pass could read it (arrays are static while
                               a pass runs when shards run one after another)
    justify     [n_sel] fp64   published units: the largest `list_justification` of the OTHER shards of the call (-inf: none)
    pub_before / pub_after  [max_rows] uint64  this shard's published array before / after the call (None: not checked)
    n_call_rows                rows of the whole call (slots [0, n_call_rows) may be written, the rest must stay untouched)
    """

    bounds: np.ndarray
    epoch: int
    peer_words: np.ndarray
    justify: np.ndarray
    pub_before: tp.Optional[np.ndarray] = None
    pub_after: tp.Optional[np.ndarray] = None
    n_call_rows: int = 0


def peer_word(epoch: int, value: np.ndarray) -> np.ndarray:
    """(epoch << 32 | fp32 bits) words of published values."""
    bits = np.asarray(value, np.float32).view(np.uint32).astype(np.uint64)
    return (np.uint64(epoch) << np.uint64(32)) | bits


def split_words(words: np.ndarray) -> tp.Tuple[np.ndarray, np.ndarray]:
    """(epochs uint32, fp32 values) of published words."""
    w = np.asarray(words, np.uint64)
    return (w >> np.uint64(32)).astype(np.uint32), (w & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.float32)


def round_up_f32(x: np.ndarray) -> np.ndarray:
    """Smallest fp32 >= x (fp64 in), elementwise; +inf above the fp32 range."""
    x = np.asarray(x, np.float64)
    with np.errstate(over="ignore"):
        f = x.astype(np.float32)
    low = f.astype(np.float64) < x
    return np.where(low, np.nextafter(f, np.float32(np.inf)), f).astype(np.float32)


def _kth_per_list(A: np.ndarray, elig: np.ndarray, pos_of_list: tp.List[np.ndarray], kc: int) -> np.ndarray:
    """[rows] max over lists of the kc-th best eligible A of the list (-inf where no list has kc eligible positions)."""
    out = np.full(A.shape[0], -np.inf)
    for cols in pos_of_list:
        if len(cols) < kc:
            continue
        v = np.where(elig[:, cols], A[:, cols], -np.inf)
        out = np.maximum(out, -np.partition(-v, kc - 1, axis=1)[:, kc - 1])
    return out


def list_justification(snap: tp.Dict[str, tp.Any], cat: "Catalogue", sub32: np.ndarray, viewed: sparse.csr_matrix, block: int = 256) -> np.ndarray:
    """[n_sel] in published units: per row, the largest (K'-th best eligible A_ref of a list + accumulation bound) over the
    pass's lists, times 2^-obj_exp.  No list of the pass can hold a threshold above it without a peer's help."""
    n_sel = int(snap["n_sel"])
    sub32 = np.ascontiguousarray(sub32, dtype=np.float32)
    lpr = int(snap["nw"]) // 4
    lop = list_of_positions(cat.n_pos, lpr, max(1, int(snap["tiles_per_split"])))
    pos_of_list = [np.nonzero(lop == l)[0] for l in range(int(snap["n_lists"]))]
    _, u16 = subject_operands(sub32, cat.bf16)
    acc_bound = cat.d_pad * ACC_REL * np.sqrt(np.einsum("ij,ij->i", u16, u16)) * cat.i16_norm_max
    out = np.empty(n_sel)
    for r0 in range(0, n_sel, block):
        r1 = min(n_sel, r0 + block)
        A = u16[r0:r1] @ cat.i16_pos.T
        elig = viewed[r0:r1].toarray() == 0
        out[r0:r1] = _kth_per_list(A, elig, pos_of_list, int(snap["k_cand"])) + acc_bound[r0:r1]
    return np.ldexp(out, -cat.obj_exp)


def _sorted_kth(scores: np.ndarray, ids: np.ndarray, k: int) -> float:
    order = np.lexsort((ids, -scores.astype(np.float64)))
    return float(scores[order[k - 1]])


def check_snapshot(
    snap: tp.Dict[str, tp.Any],
    cat: Catalogue,
    sub32: np.ndarray,
    viewed: sparse.csr_matrix,
    excluded: tp.Optional[sparse.csr_matrix] = None,
    prev: tp.Optional[tp.Tuple[np.ndarray, np.ndarray, np.ndarray]] = None,
    block: int = 256,
    shared: tp.Optional[SharedPass] = None,
) -> Report:
    """Check one pass.  `sub32` [n_sel, d] fp32 subject rows and `viewed` [n_sel, n_pos] (Catalogue.viewed_positions) in
    the pass's batch order; `excluded` [n_sel, n_pos]: positions returned by earlier passes (k0 > 0); `prev` (k0 > 0):
    per batch row (score, LOCAL id, rows with at least k0 results) of output entry k0 - 1, the bound of this pass;
    `shared`: the pass shared thresholds (I5 becomes "no verdict", I6-I8 apply)."""
    rep = Report()
    n_sel, n_pos = int(snap["n_sel"]), cat.n_pos
    nl, stride, kc = int(snap["n_lists"]), int(snap["cand_stride"]), int(snap["k_cand"])
    wide, k0, kp = bool(snap["wide"]), int(snap["k0"]), int(snap["kp"])
    rep.n_rows, rep.n_lists = n_sel, nl
    sub32 = np.ascontiguousarray(sub32, dtype=np.float32)
    assert sub32.shape == (n_sel, cat.d) and viewed.shape == (n_sel, n_pos)

    # ---- constants and geometry the kernel ran with
    lpr = int(snap["nw"]) // 4
    n_obj_tiles = (n_pos + TILE_N - 1) // TILE_N
    expect = {
        "bf16": int(cat.bf16), "obj_exp": cat.obj_exp, "id_off": cat.id_off, "n_pos": n_pos, "n_obj_tiles": n_obj_tiles,
        "n_lists": int(snap["n_splits"]) * lpr, "rows_pad": round_up(n_sel, 2 * 128),
        "tiles_per_split": (n_obj_tiles + int(snap["n_splits"]) - 1) // int(snap["n_splits"]),
    }
    for key, val in expect.items():
        if int(snap[key]) != int(val):
            rep.add("const", f"{key}={snap[key]} expected {val}")
    ref_eps = cat.eps_rel()
    if abs(float(snap["eps_rel"]) - float(ref_eps)) > float(np.spacing(ref_eps)):
        rep.add("const", f"eps_rel={snap['eps_rel']!r} expected {ref_eps!r}")
    if abs(float(snap["max_obj_norm"]) - float(cat.max_obj_norm)) > 2 * float(np.spacing(cat.max_obj_norm)):
        rep.add("const", f"max_obj_norm={snap['max_obj_norm']!r} expected {cat.max_obj_norm!r}")
    if not wide and not 1 <= kc <= stride:
        rep.add("const", f"k_cand={kc} cand_stride={stride}")
    row_exp_ref, u16 = subject_operands(sub32, cat.bf16)
    row_exp = np.asarray(snap["row_exp"][:n_sel], dtype=np.int64)
    bad = np.nonzero(row_exp != row_exp_ref)[0]
    if len(bad):
        rep.add("const", f"row_exp differs in {len(bad)} rows, e.g. row {bad[0]}: {row_exp[bad[0]]} vs {row_exp_ref[bad[0]]}", len(bad))

    lop = list_of_positions(n_pos, lpr, max(1, int(snap["tiles_per_split"])))
    pos_of_list = [np.nonzero(lop == l)[0] for l in range(nl)]
    u_norm = np.sqrt(np.einsum("ij,ij->i", sub32, sub32, dtype=np.float64))
    acc_bound = cat.d_pad * ACC_REL * np.sqrt(np.einsum("ij,ij->i", u16, u16)) * cat.i16_norm_max  # scaled units
    eps = float(ref_eps) * u_norm * float(cat.max_obj_norm)
    scale = np.ldexp(1.0, -(row_exp + int(snap["obj_exp"])))  # approximate units -> exact units

    counts = np.asarray(snap["cand_counts"])[:, :n_sel]
    thr = np.asarray(snap["cand_thr"])[:, :n_sel].astype(np.float64)
    overflow = counts > stride
    rep.n_overflow = int(overflow.any(axis=0).sum())
    n_listed = np.minimum(counts, stride)
    if not wide and (counts > kc).any():
        rep.add("I1", f"adaptive lists longer than K'={kc}: {int((counts > kc).sum())}", int((counts > kc).sum()))
    if (counts < 0).any() or np.isnan(thr).any() or (thr == np.inf).any():
        rep.add("I4", "negative count, NaN or +inf threshold")

    # exact fp32 scores of every listed candidate (input of the restated verdict)
    cand_rows: tp.List[tp.List[tp.Tuple[np.ndarray, np.ndarray]]] = [[] for _ in range(n_sel)]
    justify = np.full(n_sel, -np.inf)  # approximate units: the largest K'-th best eligible A_ref of a list + accumulation bound

    for r0 in range(0, n_sel, block):
        r1 = min(n_sel, r0 + block)
        A = u16[r0:r1] @ cat.i16_pos.T  # fp64 dot of the 16-bit operands, scaled units
        vmask = viewed[r0:r1].toarray() != 0
        xmask = excluded[r0:r1].toarray() != 0 if excluded is not None else np.zeros_like(vmask)
        listed = np.zeros_like(vmask)
        slot = np.arange(stride)[None, None, :]
        emask = slot < n_listed[:, r0:r1, None]  # [lists, rows, slots]
        l_idx, rr, e_idx = np.nonzero(emask)
        ids = np.asarray(snap["cand_ids"])[l_idx, r0 + rr, e_idx].astype(np.int64)
        sc = np.asarray(snap["cand_scores"])[l_idx, r0 + rr, e_idx].astype(np.float64)
        in_range = (ids >= 0) & (ids < cat.n_obj)
        pos = np.where(in_range, cat.pos_of_obj[np.clip(ids, 0, max(cat.n_obj - 1, 0))], -1)
        good = pos >= 0
        if (~good).any():
            i = np.nonzero(~good)[0][0]
            rep.add("I1", f"id {ids[i]} (row {r0 + rr[i]}, list {l_idx[i]}) is not an object position", int((~good).sum()))
        l_idx, rr, ids, sc, pos = l_idx[good], rr[good], ids[good], sc[good], pos[good]
        # I1: list membership, filter, exclusion, uniqueness
        wrong = lop[pos] != l_idx
        if wrong.any():
            i = np.nonzero(wrong)[0][0]
            rep.add("I1", f"row {r0 + rr[i]}: id {ids[i]} (position {pos[i]}) in list {l_idx[i]}, belongs to list {lop[pos[i]]}", int(wrong.sum()))
        vw = vmask[rr, pos]
        if vw.any():
            i = np.nonzero(vw)[0][0]
            rep.add("I1", f"row {r0 + rr[i]}: viewed id {ids[i]} in list {l_idx[i]}", int(vw.sum()))
        xw = xmask[rr, pos]
        if xw.any():
            i = np.nonzero(xw)[0][0]
            rep.add("I1", f"row {r0 + rr[i]}: id {ids[i]} returned by an earlier pass is listed again", int(xw.sum()))
        key = (rr * n_pos + pos) if len(rr) else np.empty(0, np.int64)
        uniq, first, cnt = np.unique(key, return_index=True, return_counts=True)
        if (cnt > 1).any():
            i = first[np.nonzero(cnt > 1)[0][0]]
            rep.add("I1", f"row {r0 + rr[i]}: id {ids[i]} listed {cnt.max()} times", int((cnt - 1).sum()))
        listed[rr, pos] = True
        # I2 (P1): approximate scores against the 16-bit emulation and against the exact scores
        a_ref = A[rr, pos]
        ab = acc_bound[r0 + rr]
        d_acc = np.abs(sc - a_ref)
        f_acc = np.where(ab > 0, d_acc / np.where(ab > 0, ab, 1), np.where(d_acc > 0, np.inf, 0))
        exact = cat.exact(sub32[r0 + rr], pos)
        d_eps = np.abs(sc * scale[r0 + rr] - exact)
        ep = eps[r0 + rr]
        f_eps = np.where(ep > 0, d_eps / np.where(ep > 0, ep, 1), np.where(d_eps > 0, np.inf, 0))
        if len(sc):
            rep.frac_acc = max(rep.frac_acc, float(f_acc.max()))
            rep.frac_eps = max(rep.frac_eps, float(f_eps.max()))
        for f, what in ((f_acc, "|cand - A_ref| > d_pad 2^-21 |u16| max|i16|"), (f_eps, "|approx - exact| > eps")):
            if (f > 1).any():
                i = int(np.argmax(f))
                rep.add("I2", f"row {r0 + rr[i]} id {ids[i]}: {what} ({f[i]:.3g} of the bound)", int((f > 1).sum()))
        exact32 = exact.astype(np.float32)
        order = np.argsort(rr, kind="stable")
        splits = np.searchsorted(rr[order], np.arange(r1 - r0 + 1))
        for i in range(r1 - r0):
            sel = order[splits[i] : splits[i + 1]]
            cand_rows[r0 + i].append((exact32[sel], ids[sel]))
        justify[r0:r1] = _kth_per_list(A, ~(vmask | xmask), pos_of_list, kc) + acc_bound[r0:r1]
        # I3 (P2) and I4: every discarded eligible position lies below the list's final threshold
        elig = ~(vmask | xmask | listed)
        for l in range(nl):
            cols = pos_of_list[l]
            if len(cols) == 0:
                continue
            best = np.where(elig[:, cols], A[:, cols], -np.inf).max(axis=1)
            t = thr[l, r0:r1]
            live = ~overflow[l, r0:r1] & np.isfinite(best)
            over = live & (best > t + acc_bound[r0:r1])
            with np.errstate(invalid="ignore", divide="ignore"):
                m = (best - t) / acc_bound[r0:r1]
            m = m[live & np.isfinite(m)]
            if len(m):
                rep.i3_margin = max(rep.i3_margin, float(m.max()))
            if over.any():
                i = np.nonzero(over)[0][0]
                rep.add("I3", f"row {r0 + i} list {l}: a discarded object scores {best[i]:.9g} > tau {t[i]:.9g}", int(over.sum()))
            if t.size:
                empty = (t == -np.inf) & np.isfinite(best)
                if empty.any():
                    i = np.nonzero(empty)[0][0]
                    rep.add("I4", f"row {r0 + i} list {l}: tau = -inf but an eligible object is not listed", int(empty.sum()))
            if not wide:
                full = counts[l, r0:r1] >= kc
                for i in np.nonzero(full)[0]:
                    k = n_listed[l, r0 + i]
                    mn = float(np.asarray(snap["cand_scores"])[l, r0 + i, :k].min())
                    if not thr[l, r0 + i] >= mn:
                        rep.add("I4", f"row {r0 + i} list {l}: full list with tau {thr[l, r0 + i]} < its minimum {mn}")

    if shared is not None:
        _check_shared(rep, snap, shared, thr, overflow, justify, row_exp, eps)
        return rep

    # ---- I5: the verdict of rescore_select_kernel / rescore_wide_kernel, restated in fp64
    pass_row = {int(r): i for i, r in enumerate(np.asarray(snap["rows"]))}
    fb = set()
    for r in np.asarray(snap["fb_rows"]).tolist():
        if r not in pass_row:
            rep.add("I5", f"failure row {r} is not a row of the pass")
        else:
            fb.add(pass_row[r])
    rep.n_fb = len(fb)
    thr_max = thr.max(axis=0) if nl else np.full(n_sel, -np.inf)
    row_over = overflow.any(axis=0)
    rejected = set()
    for i in range(n_sel):
        if prev is not None and not prev[2][i]:
            continue  # exhausted by earlier passes: no verdict
        if not (thr_max[i] > -np.inf or row_over[i]):
            continue  # nothing was discarded: nothing to certify
        parts = cand_rows[i]
        s = np.concatenate([p[0] for p in parts]) if parts else np.empty(0, np.float32)
        ids = np.concatenate([p[1] for p in parts]) if parts else np.empty(0, np.int64)
        if prev is not None:
            bs, bi = np.float32(prev[0][i]), int(prev[1][i])
            keep = (s < bs) | ((s == bs) & (ids > bi))
            s, ids = s[keep], ids[keep]
        tol = 0.0
        if row_over[i] or len(s) < kp:
            ok, margin = False, -np.inf
        else:
            e_k = _sorted_kth(s, ids, kp)
            bound = np.ldexp(thr_max[i], -int(row_exp[i] + int(snap["obj_exp"]))) + eps[i] + 1.2e-7 * abs(e_k)
            margin = e_k - bound
            ok = margin > 0
            tol = float(np.spacing(np.float32(e_k)))
        if not ok:
            rejected.add(i)
        if (not ok) != (i in fb):
            if abs(margin) <= tol:
                rep.n_tolerated += 1
            else:
                what = "certified by the engine, rejected by the restated check" if not ok else "sent to the fallback, passes the restated check"
                rep.add("I5", f"row {i} (call row {int(snap['rows'][i])}): {what}, margin {margin:.3g}")
    rep.n_rejected = len(rejected)
    rep.rejected = sorted(rejected)
    return rep


def _check_shared(rep: Report, snap: tp.Dict[str, tp.Any], sh: SharedPass, thr: np.ndarray, overflow: np.ndarray, justify: np.ndarray,
                  row_exp: np.ndarray, eps: np.ndarray) -> None:
    """I5-I8 of a threshold-sharing pass (see SharedPass); `thr` [lists, n_sel] final thresholds, `justify` / `thr` in
    approximate units, `eps` in exact units."""
    n_sel, obj_exp = int(snap["n_sel"]), int(snap["obj_exp"])
    rows = np.asarray(snap["rows"], np.int64)[:n_sel]
    # I5: no local verdict in this mode -- the merge's global certificate decides
    if len(snap["fb_rows"]):
        rep.add("I5", f"{len(snap['fb_rows'])} rows sent to the fallback by a pass that shares thresholds", len(snap["fb_rows"]))
    # I6: every threshold is justified by a list of some shard of the call or by a valid peer value
    ep, val = split_words(np.asarray(sh.peer_words, np.uint64).reshape(-1, n_sel))
    valid = (ep == np.uint32(sh.epoch)) & ~np.isnan(val)
    peer = np.where(valid, val.astype(np.float64), -np.inf).max(axis=0) if len(ep) else np.full(n_sel, -np.inf)
    peer_conv = np.ldexp(peer, obj_exp)  # the pass's approximate units (ldexpf in the kernel: exact in the fp32 range)
    allowed = np.maximum(np.maximum(justify, np.ldexp(np.asarray(sh.justify, np.float64), obj_exp)), peer_conv)
    over = thr > allowed[None, :]
    if over.any():
        l, i = (int(v[0]) for v in np.nonzero(over))
        rep.add("I6", f"row {i} list {l}: tau {thr[l, i]:.9g} above every justification {allowed[i]:.9g} (own lists "
                f"{justify[i]:.9g}, other shards {np.ldexp(sh.justify[i], obj_exp):.9g}, peers {peer_conv[i]:.9g})", int(over.sum()))
    has_peer = np.isfinite(peer_conv)
    adopted = has_peer[None, :] & (thr == peer_conv.astype(np.float32)[None, :])
    rep.n_peer_lists = int(has_peer.sum()) * thr.shape[0]
    rep.n_adopted = int(adopted.sum())
    rep.adopted_rows = np.nonzero(adopted.any(axis=0))[0].tolist()
    # I7: the bound, restated in fp64: smallest fp32 >= x = max tau (exact units) + eps, at most a few ulps above it
    bounds = np.asarray(sh.bounds, np.float32)[:n_sel]
    tmax = thr.max(axis=0) if thr.shape[0] else np.full(n_sel, -np.inf)
    row_over = overflow.any(axis=0)
    with np.errstate(invalid="ignore", over="ignore"):
        x = np.ldexp(tmax, -(row_exp + obj_exp)) + eps
        lo = round_up_f32(x - 1e-12 * np.abs(x))  # (eps: the kernel sums |u|^2 in another order)
        hi = round_up_f32(x + 2.0**-21 * np.abs(x) + 1e-36)
    none = ~row_over & (tmax == -np.inf)
    expect_inf = row_over | (~none & (lo == np.inf))
    bad = np.zeros(n_sel, bool)
    bad |= none & (bounds != -np.inf)
    bad |= expect_inf & (bounds != np.inf)
    live = ~none & ~expect_inf
    bad |= live & ~((bounds >= lo) & (bounds <= hi))
    for i in np.nonzero(bad)[0][:1]:
        rep.add("I7", f"row {i}: bound {bounds[i]!r}, expected [{lo[i]!r}, {hi[i]!r}] (max tau {tmax[i]!r}, x = {x[i]!r})", int(bad.sum()))
    # I8: the published array -- the call's epoch, at the absolute row, never above the row's final max tau * 2^-obj_exp
    if sh.pub_after is None:
        return
    before, after = np.asarray(sh.pub_before, np.uint64), np.asarray(sh.pub_after, np.uint64)
    touched = after != before
    outside = touched.copy()
    outside[: sh.n_call_rows] = False
    if outside.any():
        rep.add("I8", f"slot {int(np.nonzero(outside)[0][0])} outside the call's {sh.n_call_rows} rows was written", int(outside.sum()))
    t_ep, t_val = split_words(after)
    wrong_ep = touched & (t_ep != np.uint32(sh.epoch))
    if wrong_ep.any():
        rep.add("I8", f"slot {int(np.nonzero(wrong_ep)[0][0])} written with epoch {int(t_ep[np.nonzero(wrong_ep)[0][0]])}", int(wrong_ep.sum()))
    mine = touched[rows]
    rep.n_published = int(mine.sum())
    with np.errstate(invalid="ignore"):
        above = mine & ~(t_val[rows].astype(np.float64) <= np.ldexp(tmax, -obj_exp))
    if above.any():
        i = int(np.nonzero(above)[0][0])
        rep.add("I8", f"row {i} (slot {rows[i]}): published {t_val[rows[i]]!r} > max tau * 2^-obj_exp {np.ldexp(tmax[i], -obj_exp)!r}", int(above.sum()))


def model_snapshot(
    cat: Catalogue, sub32: np.ndarray, viewed: sparse.csr_matrix, k_cand: int, kp: int, k_out: int, nw: int = 8, n_splits: int = 1,
    peer_floor: tp.Optional[np.ndarray] = None,
) -> tp.Dict[str, tp.Any]:
    """What a correct adaptive pass may leave behind, built without the engine: the same partition of the stream, each list
    holding its K' best eligible positions by A_ref, every list's threshold the maximum of the row's full-list minima,
    the failure rows those of the restated verdict.  `peer_floor` [n_sel] (approximate units, -inf: none): a shared pass
    whose lists adopted a peer threshold from the start -- lists keep only positions above it, thresholds are at least
    it, and there is no verdict.  Input of the checker's own tests."""
    n_sel = len(sub32)
    row_exp, u16 = subject_operands(sub32, cat.bf16)
    lpr = nw // 4
    n_obj_tiles = (cat.n_pos + TILE_N - 1) // TILE_N
    tps = (n_obj_tiles + n_splits - 1) // n_splits
    nl, stride, rows_pad = n_splits * lpr, 32, round_up(n_sel, 256)
    lop = list_of_positions(cat.n_pos, lpr, tps)
    scores = np.zeros((nl, rows_pad, stride), np.float32)
    ids = np.full((nl, rows_pad, stride), PAD_ID, np.int32)
    counts = np.zeros((nl, rows_pad), np.int32)
    thr = np.full((nl, rows_pad), -np.inf, np.float32)
    A = u16 @ cat.i16_pos.T
    vm = viewed.toarray() != 0
    for r in range(n_sel):
        minima = []
        for l in range(nl):
            cols = np.nonzero((lop == l) & ~vm[r])[0]
            if peer_floor is not None:
                cols = cols[A[r, cols] > peer_floor[r]]
            top = cols[np.argsort(-A[r, cols], kind="stable")[:k_cand]]
            counts[l, r] = len(top)
            scores[l, r, : len(top)] = A[r, top]
            ids[l, r, : len(top)] = cat.pos2obj[top]
            if len(top) == k_cand:
                minima.append(np.float32(A[r, top].min()))
        thr[:, r] = max(minima) if minima else -np.inf
        if peer_floor is not None:
            thr[:, r] = np.maximum(thr[:, r], np.float32(peer_floor[r]))
    snap = {
        "valid": 1, "launch": 1, "nw": nw, "n_lists": nl, "n_splits": n_splits, "tiles_per_split": tps, "n_obj_tiles": n_obj_tiles,
        "cand_stride": stride, "n_pos": cat.n_pos, "rows_pad": rows_pad, "n_sel": n_sel, "k_out": k_out, "k_cand": k_cand, "k0": 0,
        "kp": kp, "wide": 0, "phase1_tiles": 0x7FFFFFFF, "bf16": int(cat.bf16), "obj_exp": cat.obj_exp, "eps_rel": cat.eps_rel(),
        "max_obj_norm": cat.max_obj_norm, "id_off": cat.id_off, "cand_scores": scores, "cand_ids": ids, "cand_counts": counts,
        "cand_thr": thr, "row_exp": row_exp, "rows": np.arange(n_sel, dtype=np.int32), "fb_rows": np.empty(0, np.int32),
    }
    if peer_floor is None:
        snap["fb_rows"] = np.asarray(check_snapshot(snap, cat, sub32, viewed).rejected, dtype=np.int32)
    snap["n_fb"] = len(snap["fb_rows"])
    return snap

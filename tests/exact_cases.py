"""Case generators and expectations for the exhaustive kernels (plain numpy, no GPU).

The exhaustive half of the engine -- `exact_topk_kernel` + `merge_select_kernel` (path 0 and every re-rank),
`dense_scores_kernel` + `scores_topk_kernel` (path 3), `sparse_scores_kernel` (path 2) and `b200_rank_merge*` -- branches at
pass boundaries (k0 = 32, 64, ...), at 32-object tiles, at the object splits of `run_exact` and at the row chunks of paths 2 / 3.
Continuous random scores almost never tie there.  The generators below use INTEGER-valued factors (entries in [-3, 3],
small d): every fp64 dot is an exact small integer, so one score value is shared by tens to hundreds of objects and ties land
on every boundary.  COSINE divides by the object norm, which breaks integer ties, so its catalogues are drawn from a small
pool of distinct rows: duplicated rows tie exactly after the division too.

Planted blocks use a private column per planted subject row: only that row has a non-zero entry there, so the block is
invisible (score 0) to every other row and several plants coexist in one catalogue.

The result definition is the engine's (include/b200_rank.h): fp64-accumulated dot rounded once to fp32, COSINE divided by
the fp32 object norm but NOT by the subject norm, order (score desc, id asc), unfilled slots id -1 / score -FLT_MAX.
"""
from __future__ import annotations

import typing as tp

import numpy as np
from scipy import sparse

from oracle.topk_oracle import calc_norms, implicit_topk, neginf_score
from rectools_b200.sharded import merge_padded_numpy

FLT_MAX = np.float32(np.finfo(np.float32).max)
NEG_MAX = np.float32(-FLT_MAX)
PAD_ID = 0x7FFFFFFF
EX_ROWS = 32  # rows per block of exact_topk_kernel (select.cuh)
CHUNK_BYTES = 1 << 30  # score-row budget of a path-2 / path-3 row chunk (engine.cu: run_sparse, run_dense_large_k)


# ------------------------------------------------------------------------------------------------ geometry of the kernels
def exact_splits(n_rows: int, n_pos: int, sm_count: int) -> int:
    """Object splits of one `run_exact` call (engine.cu): clamp(ceil(2 sm / blocks_x), 1, tiles / 64, 1024)."""
    tiles = (n_pos + 31) // 32
    blocks_x = (n_rows + EX_ROWS - 1) // EX_ROWS
    s = (2 * sm_count + blocks_x - 1) // blocks_x
    return int(min(max(1, min(s, tiles // 64)), 1024))


def split_edges(n_rows: int, n_pos: int, sm_count: int) -> np.ndarray:
    """First position of every non-empty split after the first (exact_topk_kernel: ceil(tiles / splits) tiles each)."""
    tiles = (n_pos + 31) // 32
    s = exact_splits(n_rows, n_pos, sm_count)
    per = (tiles + s - 1) // s
    return np.array([j * per * 32 for j in range(1, s) if j * per < tiles], dtype=np.int64)


def dense_chunk_rows(n_pos: int) -> int:
    """Rows per chunk of path 3 (`run_dense_large_k`): 2^30 / (4 n_pos), rounded down to 32, at least 32."""
    return max(32, (CHUNK_BYTES // max(4 * n_pos, 1)) // 32 * 32)


def sparse_chunk_rows(n_pos: int) -> int:
    """Rows per chunk of path 2 (`run_sparse`): 2^30 / (4 n_pos), at least 1."""
    return max(1, CHUNK_BYTES // max(4 * n_pos, 1))


# ------------------------------------------------------------------------------------------------ generators
def int_matrix(rng: np.random.Generator, n: int, d: int, lo: int = -3, hi: int = 3) -> np.ndarray:
    """Integer-valued fp32 factors, entries uniform in [lo, hi]."""
    return rng.integers(lo, hi + 1, size=(n, d)).astype(np.float32)


def pooled_matrix(rng: np.random.Generator, n: int, d: int, n_pool: int, lo: int = -3, hi: int = 3) -> np.ndarray:
    """`n` rows drawn from `n_pool` distinct integer rows (COSINE catalogues: duplicates tie after the norm division)."""
    pool = int_matrix(rng, n_pool, d, lo, hi)
    return pool[rng.integers(0, n_pool, size=n)]


def engine_scores(subjects: np.ndarray, objects: np.ndarray, cosine: bool) -> np.ndarray:
    """Scores in the engine's definition: fp32(sum fp64 products) (COSINE: / fp32 object norm), [n_subjects, n_objects]."""
    s = np.asarray(subjects, np.float64) @ np.asarray(objects, np.float64).T
    if cosine:
        s = s / calc_norms(np.asarray(objects, np.float32), "f64").astype(np.float64)[None, :]
    return s.astype(np.float32)


def _plant(objects: np.ndarray, subjects: np.ndarray, row: int, col: int, junk_col: int, above: np.ndarray, block: np.ndarray,
           cosine: bool) -> None:
    """Make `above` (any positions) the objects ranked first for subject `row` and `block` the exact tie right after them.
    Column `col` is private to `row` (zero for every other subject and every unplanted object); `junk_col` is a column no
    subject uses (COSINE: it lowers the block's cosine below the above-objects' without changing any other score)."""
    assert np.all(subjects[np.arange(len(subjects)) != row, col] == 0) and np.all(subjects[:, junk_col] == 0)
    assert np.all(objects[:, col] == 0), "private column already used"
    nat = np.abs(subjects[row]).sum() * 3 if not cosine else np.sqrt((subjects[row].astype(np.float64) ** 2).sum())
    for rows, (v_col, v_junk) in ((above, (3.0, 0.0)), (block, (2.0, 1.0) if cosine else (2.0, 0.0))):
        objects[rows] = 0
        objects[rows, col] = v_col
        objects[rows, junk_col] = v_junk
    # private strength C: DOT block = 2C, COSINE block = 2C / sqrt(5); both above every natural score (<= 3 |u|_1 or |u|_2)
    subjects[row, col] = float(int(nat) + 1 if not cosine else int(nat * np.sqrt(5) / 2) + 2)


def tie_across_rank(objects: np.ndarray, subjects: np.ndarray, row: int, col: int, junk_col: int, k0: int, left: int, right: int,
                    rng: np.random.Generator, free: np.ndarray, cosine: bool = False) -> np.ndarray:
    """Plant, for subject `row`, k0 - left objects above a block of left + right exact ties: the block straddles rank k0
    with `left` ties before it and `right` after it.  Positions are drawn from the `free` mask (updated).  Returns the
    block's object ids."""
    pos = rng.choice(np.nonzero(free)[0], size=k0 - left + left + right, replace=False)
    free[pos] = False
    above, block = pos[: k0 - left], pos[k0 - left :]
    _plant(objects, subjects, row, col, junk_col, above, block, cosine)
    return np.sort(block)


def tie_across_position(objects: np.ndarray, subjects: np.ndarray, row: int, col: int, junk_col: int, edge: int, left: int, right: int,
                        free: np.ndarray, cosine: bool = False) -> np.ndarray:
    """Plant, for subject `row`, a block of exact ties that is the row's best: positions [edge - left, edge + right) (a
    32-object tile edge, a split edge of `run_exact`, the start of the last tile, ...).  Returns the block's object ids."""
    block = np.arange(edge - left, min(edge + right, len(objects)))
    assert free[block].all(), "planted ranges overlap"
    free[block] = False
    _plant(objects, subjects, row, col, junk_col, np.empty(0, np.int64), block, cosine)
    return block


class TieCatalogue(tp.NamedTuple):
    objects: np.ndarray   # [n_obj, d] fp32
    subjects: np.ndarray  # [n_subjects, d] fp32; rows 0 .. len(plants) - 1 planted, row ZERO_ROW all zero
    plants: tp.List[tp.Dict[str, tp.Any]]  # row, kind ("rank" / "position"), at (k0 or edge), left, right, block ids


ZERO_ROW = 10


def tie_catalogue(sm_count: int, cosine: bool = False, n_obj: int = 300_000, n_subjects: int = 1_500, d_nat: int = 8, seed: int = 0
                  ) -> TieCatalogue:
    """Integer catalogue with ties everywhere plus ten planted blocks (one private column each, d = d_nat + 11):
    rank ties across k0 = 32, 64, 96, 128, 160 and position ties across the first, second and third split edge of a 1-, 33- and
    129-row call
    (`sm_count`: the engine's), a tile edge and the start of the last tile.  n_obj = 300 000 makes path 3 cut 864-row chunks."""
    rng = np.random.default_rng(seed)
    n_plants = 10
    d = d_nat + n_plants + 1
    junk = d - 1
    objects = np.zeros((n_obj, d), np.float32)
    objects[:, :d_nat] = pooled_matrix(rng, n_obj, d_nat, 3_000) if cosine else int_matrix(rng, n_obj, d_nat)
    subjects = np.zeros((n_subjects, d), np.float32)
    subjects[:, :d_nat] = int_matrix(rng, n_subjects, d_nat)
    subjects[ZERO_ROW] = 0
    free = np.ones(n_obj, bool)
    specs = [  # (row, kind, at, left, right)
        (0, "position", int(split_edges(1, n_obj, sm_count)[0]), 9, 7),
        (1, "rank", 32, 3, 4),
        (2, "rank", 64, 1, 30),
        (3, "rank", 96, 20, 2),
        (4, "rank", 128, 5, 5),
        (5, "rank", 160, 7, 9),
        (6, "position", (n_obj - 1) // 32 * 32, 6, 32),
        (7, "position", 32 * 1000, 10, 10),
        (8, "position", int(split_edges(129, n_obj, sm_count)[2]), 12, 12),
        (9, "position", int(split_edges(33, n_obj, sm_count)[1]), 4, 20),
    ]
    plants = []
    for row, kind, at, left, right in specs:  # position plants first: their ranges are fixed
        if kind == "position":
            block = tie_across_position(objects, subjects, row, d_nat + row, junk, at, left, right, free, cosine)
            plants.append(dict(row=row, kind=kind, at=at, left=left, right=int(min(right, n_obj - at)), block=block))
    for row, kind, at, left, right in specs:
        if kind == "rank":
            block = tie_across_rank(objects, subjects, row, d_nat + row, junk, at, left, right, rng, free, cosine)
            plants.append(dict(row=row, kind=kind, at=at, left=left, right=right, block=block))
    return TieCatalogue(objects, subjects, sorted(plants, key=lambda p: p["row"]))


def rank_straddle(sorted_scores: np.ndarray, k0: int) -> tp.Tuple[int, int]:
    """(ties of the score at rank k0 - 1 among ranks < k0, ties of it among ranks >= k0) of one best-first score row."""
    v = sorted_scores[k0 - 1]
    return int((sorted_scores[:k0] == v).sum()), int((sorted_scores[k0:] == v).sum())


def position_straddle(scores_by_pos: np.ndarray, edge: int) -> tp.Tuple[int, int]:
    """(positions < edge, positions >= edge) holding the row's best score."""
    top = scores_by_pos.max()
    hit = np.nonzero(scores_by_pos == top)[0]
    return int((hit < edge).sum()), int((hit >= edge).sum())


def filter_keeping(rng: np.random.Generator, n_obj: int, survivors: tp.Sequence[int], candidates: tp.Optional[np.ndarray] = None
                   ) -> sparse.csr_matrix:
    """One filter row per entry of `survivors`: every object of `candidates` (default: all) except that many is filtered."""
    cand = np.arange(n_obj) if candidates is None else np.asarray(candidates)
    rows = []
    for s in survivors:
        keep = rng.choice(len(cand), size=min(s, len(cand)), replace=False)
        rows.append(np.delete(cand, keep))
    return csr_from_rows(rows, n_obj)


def csr_from_rows(rows: tp.Sequence[np.ndarray], n_cols: int) -> sparse.csr_matrix:
    """A filter CSR whose row r lists rows[r] as given (sorted, duplicates kept -- the kernels look ids up, never sum them)."""
    indptr = np.zeros(len(rows) + 1, np.int64)
    indptr[1:] = np.cumsum([len(r) for r in rows])
    indices = np.concatenate([np.sort(np.asarray(r, np.int64)) for r in rows]) if len(rows) else np.empty(0, np.int64)
    width = max(n_cols, int(indices.max()) + 1 if len(indices) else 0)
    return sparse.csr_matrix((np.ones(len(indices), np.float32), indices.astype(np.int32), indptr), shape=(len(rows), width))


# ------------------------------------------------------------------------------------------------ expectations
def expected_padded(distance: str, subjects: tp.Any, objects: np.ndarray, subject_ids: tp.Sequence[int], k: tp.Optional[int],
                    filter_csr: tp.Optional[sparse.csr_matrix] = None, whitelist: tp.Optional[np.ndarray] = None, batch: int = 256
                    ) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The oracle's answer in the engine's padded form: `(ids int32 [n, k_out], scores fp32, counts int32)`.

    `implicit_topk(accum="f64")` over the whitelisted positions with the filter rows masked, the ids mapped back through
    the whitelist, then the reference's trailing strip (scores <= `neginf_score()`, rank_implicit.py:107-118) turned into
    counts: every slot >= count is id -1 / score -FLT_MAX.  COSINE scores are divided by the object norm only.
    `subjects` may be a CSR matrix (sparse subjects: densified, duplicate columns summed, as the reference does)."""
    if sparse.issparse(subjects):
        subjects = np.asarray(subjects.todense())
    subjects = np.asarray(subjects, np.float32)
    objects = np.asarray(objects, np.float32)
    sids = np.asarray(subject_ids, np.int64)
    wl = None if whitelist is None else np.asarray(whitelist, np.int64)
    pos_obj = objects if wl is None else objects[wl]
    n_pos = len(pos_obj)
    k_out = min(n_pos if k is None else int(k), n_pos)
    filt = None
    if filter_csr is not None:
        csr = sparse.csr_matrix(filter_csr)
        if wl is not None:  # filter columns -> whitelist positions (ids beyond the CSR width are unfiltered)
            wl_in = wl[wl < csr.shape[1]]
            filt = sparse.csr_matrix(csr[:, wl_in])
            filt = sparse.csr_matrix((filt.data, filt.indices, filt.indptr), shape=(csr.shape[0], n_pos))
        else:
            filt = csr
    norms = calc_norms(pos_obj, "f64") if distance == "cosine" else None
    if k_out == 0:
        return np.empty((len(sids), 0), np.int32), np.empty((len(sids), 0), np.float32), np.zeros(len(sids), np.int32)
    ids, sc = implicit_topk(pos_obj, subjects[sids], k_out, norms, filt, accum="f64", batch=batch)
    valid = sc > np.float32(neginf_score())
    counts = valid.sum(axis=1).astype(np.int32)
    assert (valid == (np.arange(k_out)[None, :] < counts[:, None])).all()  # (best-first rows: the strip is a suffix)
    if wl is not None:
        ids = wl[ids].astype(np.int32)
    return np.where(valid, ids, -1).astype(np.int32), np.where(valid, sc, NEG_MAX).astype(np.float32), counts


def merge_case(rng: np.random.Generator, n_lists: int, n_rows: int, k: int) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Lists [n_lists, n_rows, k] for `b200_rank_merge`: counts 0 .. k per list (row 0 empty, row 1 about k / 3 entries in
    all, below a later pass's k0), integer scores tied within and across lists, ids unique per row but not ordered by list,
    some B200_PAD_ID entries inside a count, and high-scoring garbage in every slot beyond a count."""
    ids = rng.integers(0, 1 << 20, size=(n_lists, n_rows, k)).astype(np.int32)  # garbage ids
    sc = rng.integers(-4, 5, size=(n_lists, n_rows, k)).astype(np.float32) + np.float32(1e9)  # garbage scores, high
    cnt = rng.integers(0, k + 1, size=(n_lists, n_rows)).astype(np.int32)
    cnt[:, 0] = 0
    if n_rows > 1:
        cnt[:, 1] = np.bincount(rng.integers(0, n_lists, max(1, k // 3)), minlength=n_lists).clip(0, k)
    for r in range(n_rows):
        perm = rng.permutation(n_lists * k * 4)[: n_lists * k].reshape(n_lists, k)
        for li in range(n_lists):
            c = cnt[li, r]
            ids[li, r, :c] = perm[li, :c]
            sc[li, r, :c] = np.sort(rng.integers(-3, 4, c).astype(np.float32))[::-1]
            if c > 2 and rng.random() < 0.3:
                ids[li, r, rng.integers(0, c)] = PAD_ID
    return ids, sc, cnt


def merge_inputs_valid(ids: np.ndarray, scores: np.ndarray, counts: np.ndarray) -> tp.Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Lists [n_lists, n_rows, L] as `b200_rank_merge` reads them: entries < count whose id is neither B200_PAD_ID nor
    negative, compacted to the front of each list (the rest: -1 / -FLT_MAX)."""
    n_lists, n_rows, L = ids.shape
    keep = (np.arange(L)[None, None, :] < np.asarray(counts)[:, :, None]) & (ids != PAD_ID) & (ids >= 0)
    order = np.argsort(~keep, axis=2, kind="stable")
    c_ids = np.where(np.take_along_axis(keep, order, 2), np.take_along_axis(ids, order, 2), -1).astype(np.int32)
    c_sc = np.where(np.take_along_axis(keep, order, 2), np.take_along_axis(scores, order, 2), NEG_MAX).astype(np.float32)
    return c_ids, c_sc, keep.sum(axis=2).astype(np.int32)


def expected_merge(ids: np.ndarray, scores: np.ndarray, counts: np.ndarray, k: int, bounds: tp.Optional[np.ndarray] = None):
    """`merge_padded_numpy` over the entries the merge reads, plus (with `bounds` [n_lists, n_rows]) the certificate of
    `b200_rank_merge_certified` restated in fp64: a row is accepted iff every bound is -inf, or it has at least k valid
    entries and its k-th merged score is strictly greater than the largest bound.
    Returns (ids, scores, counts, fail_rows sorted ascending)."""
    c_ids, c_sc, c_cnt = merge_inputs_valid(ids, scores, counts)
    o_ids, o_sc, o_cnt = merge_padded_numpy(c_ids, c_sc, c_cnt, k)
    fail = np.empty(0, np.int64)
    if bounds is not None:
        b = np.asarray(bounds, np.float64).max(axis=0)
        n_valid = c_cnt.sum(axis=0)
        e_k = np.where(n_valid >= k, o_sc[:, k - 1].astype(np.float64), -np.inf)
        ok = (b == -np.inf) | ((n_valid >= k) & (e_k > b))
        fail = np.nonzero(~ok)[0]
    return o_ids, o_sc, o_cnt, fail

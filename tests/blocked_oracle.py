"""A top-k oracle over blocks of objects, for catalogues too large to widen to fp64 at once (test infrastructure only).

`blocked_oracle` gives the engine's answer in padded form: fp64 dots rounded once to fp32 (COSINE: divided by the fp32
object norm), filtered pairs at -FLT_MAX, a running top-k per row merged by (score desc, id asc).  Its fp64 sums come from
BLAS, so on continuous factors a score may land on the other side of an fp32 rounding boundary than the engine's; the
GPU tests hold results to `tests/score_interval.py` instead.  `tests/test_large_catalogue_oracle_cpu.py` pins it against
`rank_oracle` on integer factors, where every score is exact."""
import numpy as np

from oracle.topk_oracle import NEG_SENTINEL, calc_norms, neginf_score
from tests.score_interval import NEG_MAX, from_keys, order_keys

BLOCK_OBJECTS = 1 << 20


def _rows_f32(objects, sel) -> np.ndarray:
    """Rows `sel` (a slice or ids) of a numpy matrix or a CPU torch tensor (any float type, widened exactly) as fp32."""
    if hasattr(objects, "float"):
        import torch

        return objects[sel if isinstance(sel, slice) else torch.from_numpy(sel)].float().numpy()
    return np.asarray(objects[sel], np.float32)


def blocked_oracle(distance, subjects, objects, k, filter_csr=None, whitelist=None, block=BLOCK_OBJECTS, row_block=64):
    """The engine's answer in padded form (`ec.expected_padded`'s), computed over blocks of `block` positions: fp64 dot
    rounded once to fp32 (COSINE: / the fp32 object norm), filtered pairs at -FLT_MAX, a running top-k per row merged by
    (score desc, id asc), then the trailing sentinel strip as counts (slots beyond: id -1 / score -FLT_MAX).
    `subjects` [n, d] are the batch rows; `filter_csr` [n, >= ids] filters by object id; `whitelist` (sorted) restricts
    the positions.  Returns (ids int32 [n, k_out], scores fp32, counts int32)."""
    subjects = np.asarray(subjects, np.float64)
    n = subjects.shape[0]
    wl = None if whitelist is None else np.asarray(whitelist, np.int64)
    n_pos = objects.shape[0] if wl is None else len(wl)
    k_out = min(n_pos if k is None else int(k), n_pos)
    run = np.empty((n, 0), np.uint64)
    for p0 in range(0, n_pos, block):
        p1 = min(p0 + block, n_pos)
        ids = np.arange(p0, p1, dtype=np.int64) if wl is None else wl[p0:p1]
        blk = _rows_f32(objects, slice(p0, p1) if wl is None else ids)
        blk64 = blk.astype(np.float64)
        norms = calc_norms(blk, "f64").astype(np.float64) if distance == "cosine" else None
        parts = []
        for r0 in range(0, n, row_block):
            r1 = min(r0 + row_block, n)
            s = subjects[r0:r1] @ blk64.T
            if norms is not None:
                s = s / norms[None, :]
            s = s.astype(np.float32) + np.float32(0)  # (-0.0 -> +0.0: the sign of an exact zero is not part of the result)
            if filter_csr is not None:
                for r in range(r0, r1):
                    cols = filter_csr.indices[filter_csr.indptr[r] : filter_csr.indptr[r + 1]]
                    if wl is None:
                        s[r - r0, cols[(cols >= p0) & (cols < p1)] - p0] = NEG_SENTINEL
                    else:
                        s[r - r0, np.isin(ids, cols)] = NEG_SENTINEL
            keys = order_keys(s, np.broadcast_to(ids, s.shape))
            if k_out < keys.shape[1]:
                keys = np.partition(keys, k_out - 1, axis=1)[:, :k_out]
            parts.append(np.sort(keys, axis=1))
        cand = np.concatenate(parts, axis=0)
        # two sorted runs per row: the stable sort (timsort) merges them
        run = np.sort(np.concatenate([run, cand], axis=1), axis=1, kind="stable")[:, :k_out]
    ids, sc = from_keys(run)
    valid = sc > np.float32(neginf_score())
    counts = valid.sum(axis=1).astype(np.int32)
    assert (valid == (np.arange(k_out)[None, :] < counts[:, None])).all()
    return np.where(valid, ids, -1).astype(np.int32), np.where(valid, sc, NEG_MAX).astype(np.float32), counts

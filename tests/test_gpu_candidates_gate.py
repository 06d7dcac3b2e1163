"""GPU: the threshold gate of the fused kernel's accumulator hand-off, on a pass built to make it disagree with itself.

The MMA warp group stages a warp's 16 rows of a quarter only if one of their scores lies above that row's threshold;
otherwise that part of the staging buffer keeps an earlier quarter, and the epilogue lanes of those rows must not scan it.
An epilogue warp reads 32 rows: lanes 0-15 come from one MMA warp, lanes 16-31 from the next.  Here the subjects come in
alternating 16-row blocks aimed at two disjoint object clusters, the clusters fill alternate object tiles, and each tile of
a cluster scores above every earlier one for the rows aimed at it and below zero for the others.  With the carousel off
and one object split (the stream ascends from tile 0), every tile after the first two has one half of every epilogue
warp staged with new best scores and the other half gated -- a half that was staged with its own best scores one tile
before.  A lane that scanned its stale rows would take those scores with the positions of the current tile: list entries
whose score does not belong to their id, which the snapshot check (tests/tc_reference.py) reports.  The pass is checked
with check_snapshot and the final top-k with the rounding-interval checker, as in tests/test_gpu_candidates.py."""
import numpy as np
import pytest

from tests.tc_reference import TILE_N
from tests.test_gpu_candidates import K, _run

pytestmark = pytest.mark.gpu

BLOCK = 16  # rows of one MMA warp in an m-half


@pytest.fixture(scope="module")
def lib():
    from rectools_b200 import _lib

    return _lib


def _alternating_clusters(n_rows, n_tiles, d, seed):
    """Rows of block b (16 rows each) aim at cluster b % 2; tile t holds cluster t % 2 with scores rising by tile."""
    rng = np.random.default_rng(seed)
    n_obj = n_tiles * TILE_N
    tile = np.arange(n_obj) // TILE_N
    cluster = tile % 2
    objects = np.zeros((n_obj, d), np.float32)
    # own-cluster score (1 + t + [0, 0.5)) x row scale: every tile of a cluster above all of its earlier ones
    objects[np.arange(n_obj), cluster] = (1.0 + tile + 0.5 * rng.random(n_obj)).astype(np.float32)
    objects[:, 2:] = (0.1 * rng.standard_normal((n_obj, d - 2))).astype(np.float32)  # scores do not see these columns
    aim = (np.arange(n_rows) // BLOCK) % 2
    subjects = np.zeros((n_rows, d), np.float32)
    scale = rng.uniform(0.5, 2.0, n_rows).astype(np.float32)
    subjects[np.arange(n_rows), aim] = scale
    subjects[np.arange(n_rows), 1 - aim] = -scale  # the other cluster scores below zero
    return subjects, objects, aim, cluster, tile


def test_gate_halves_disagree_tile_after_tile(lib, monkeypatch, capsys):
    from rectools_b200 import Engine

    monkeypatch.setenv("B200_TC_CAROUSEL", "0")
    monkeypatch.setenv("B200_TC_SPLITS", "1")  # one stream of all 64 tiles: 31 tiles where a staged half is gated
    n_rows, n_tiles, d = 768, 64, 64
    u, i, aim, cluster, tile = _alternating_clusters(n_rows, n_tiles, d, seed=5)

    # the premise, in fp64: for every row, each own-cluster tile scores above every earlier tile, the other cluster below 0
    s = u.astype(np.float64) @ i.astype(np.float64).T
    own = aim[:, None] == cluster[None, :]
    assert (s[own] > 0).all() and (s[~own] < 0).all()
    for a in (0, 1):
        rows = aim == a
        t_own = np.arange(a, n_tiles, 2)
        lo = np.array([s[rows][:, tile == t].min(axis=1) for t in t_own])
        hi = np.array([s[rows][:, tile == t].max(axis=1) for t in t_own])
        assert (lo[1:] > hi[:-1]).all()

    eng = Engine(i, cosine=False)
    _, reps = _run(eng, lib, monkeypatch, capsys, "gate_alternating_halves", u, K, i, False)
    snap = reps[0][0]
    assert snap["n_splits"] == 1 and snap["tiles_per_split"] == n_tiles
    eng.close()

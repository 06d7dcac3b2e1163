"""CPU (gloo, world_size 2 and 3): the item-sharded exchange logic of `ShardedB200Ranker` -- shard ranges, global ids,
whitelist split, padding of short shards, all-gather + merge -- with the oracle standing in for the per-shard CUDA
engine.  The CUDA side of the same path is covered by test_gpu_parity.py::test_merge_matches_unsharded."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from scipy import sparse

from rectools_b200.sharded import ShardedB200Ranker, merge_padded_numpy, shard_bounds, split_whitelist
from tests.helpers import synth_factors, synth_viewed_csr
from tests.sharded_cases import OracleShard


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out, item_shards=None):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        u, i = synth_factors(40, 203, 16, seed=5)
        csr = synth_viewed_csr(40, 203, 20)
        whitelist = np.sort(np.random.default_rng(1).choice(203, 70, replace=False))
        results = {}
        for dist_name in ("dot", "cosine"):
            ranker = ShardedB200Ranker(dist_name, u, i, local_factory=OracleShard, item_shards=item_shards)
            for k, filt, wl in ((5, None, None), (7, csr, None), (4, csr, whitelist), (80, None, whitelist)):
                sids = np.arange(40)[::-1].copy()
                res = ranker.rank(sids, k, None if filt is None else filt[sids], wl)
                results[(dist_name, k, filt is not None, wl is not None)] = [np.asarray(x) for x in res]
        if rank == 0:
            out.put(results)
        dist.barrier()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize(
    "world, item_shards",
    [(2, None), (3, None), (2, 1), (4, 2), (3, 1)],
    ids=["items2", "items3", "subjects2", "grid2x2", "subjects3-ragged"],
)
def test_sharded_matches_unsharded_oracle(world, item_shards):
    """Item sharding (north star), subject sharding and the item x subject grid all return the unsharded result on every
    rank: shard ranges, global ids, whitelist split, short shards, ragged subject slices, both all-gathers, the merge."""
    from oracle.topk_oracle import rank_oracle

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, out, item_shards)) for r in range(world)]
    for p in procs:
        p.start()
    results = out.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    u, i = synth_factors(40, 203, 16, seed=5)
    csr = synth_viewed_csr(40, 203, 20)
    whitelist = np.sort(np.random.default_rng(1).choice(203, 70, replace=False))
    sids = np.arange(40)[::-1].copy()
    for (dist_name, k, has_f, has_wl), (s, ids, sc) in results.items():
        es, eid, esc = rank_oracle(dist_name, u, i, sids, k, csr[sids] if has_f else None, whitelist if has_wl else None, accum="f64")
        np.testing.assert_array_equal(s, es)
        np.testing.assert_array_equal(ids, eid, err_msg=str((dist_name, k, has_f, has_wl)))
        np.testing.assert_allclose(sc, esc, rtol=1e-6, atol=1e-7)


def test_shard_helpers():
    assert shard_bounds(10, 4) == [(0, 3), (3, 6), (6, 9), (9, 10)]
    assert shard_bounds(2, 4) == [(0, 1), (1, 2), (2, 2), (2, 2)]
    np.testing.assert_array_equal(split_whitelist([1, 3, 5, 7, 9], 3, 8), [0, 2, 4])
    assert len(split_whitelist([1, 2], 5, 9)) == 0


def _worker_tiny(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        u, i = synth_factors(9, 50, 8, seed=2)
        results = {}
        ranker = ShardedB200Ranker("dot", u, i, local_factory=OracleShard)
        for n in (1, 2, 5, 9):  # fewer rows than ranks, rows not divisible by the ranks: padded slices of the all-to-all
            res = ranker.rank(np.arange(n), 4)
            results[n] = [np.asarray(x) for x in res]
        if rank == 0:
            out.put(results)
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_slice_exchange_with_tiny_and_ragged_batches():
    from oracle.topk_oracle import rank_oracle

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_tiny, args=(r, 4, port, out)) for r in range(4)]
    for p in procs:
        p.start()
    results = out.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    u, i = synth_factors(9, 50, 8, seed=2)
    for n, (s, ids, sc) in results.items():
        es, eid, esc = rank_oracle("dot", u, i, np.arange(n), 4, accum="f64")
        np.testing.assert_array_equal(s, es)
        np.testing.assert_array_equal(ids, eid, err_msg=f"n={n}")
        np.testing.assert_allclose(sc, esc, rtol=1e-6, atol=1e-7)


def test_sharded_argument_checks_single_process():
    """ADVICE r1: the sharded ranker range-checks subject ids and the whitelist like `B200Ranker` does."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()))
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        u, i = synth_factors(6, 30, 4, seed=1)
        ranker = ShardedB200Ranker("dot", u, i, local_factory=OracleShard)
        with pytest.raises(IndexError):
            ranker.rank([0, 6], 3)
        with pytest.raises(ValueError, match="sorted"):
            ranker.rank([0], 3, sorted_object_whitelist=np.array([5, 2]))
        with pytest.raises(IndexError):
            ranker.rank([0], 3, sorted_object_whitelist=np.array([2, 30]))
        with pytest.raises(ValueError, match="filter_pairs_csr"):
            ranker.rank([0, 1], 3, sparse.csr_matrix((3, 30), dtype=np.float32))
        s, ids, sc = ranker.rank([2, 0], 3)
        assert len(ids) == 6
    finally:
        dist.destroy_process_group()

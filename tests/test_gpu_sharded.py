"""GPU: the item-sharded exchange on real engines.

* one GPU: the threshold-sharing PROTOCOL without peers -- per-shard passes with `B200_Q_SHARED_THRESHOLDS` (no local verdict,
  per-row bounds out), packed buffers, `b200_rank_merge_certified`, re-rank of the rows the global certificate rejects --
  must equal the unsharded ranking;
* two or more GPUs: `ShardedB200Ranker` under torchrun (NCCL), with and without threshold sharing over NVLink peer memory,
  host and device inputs, item sharding / subject sharding / grid (scripts/dist_gpu_check.py, the case table of
  tests/sharded_cases.py).  The same table runs on one GPU in tests/test_gpu_sharded_processes.py."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle.topk_oracle import rank_oracle
from tests.helpers import synth_factors, synth_viewed_csr

pytestmark = pytest.mark.gpu
ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def test_shared_threshold_protocol_on_one_gpu(rb):
    import torch

    from rectools_b200 import _lib
    from rectools_b200.sharded import EngineShard, Packed, shard_bounds

    n_users, n_items, d, k, shards = 5000, 60_000, 64, 10, 3
    u, i = synth_factors(n_users, n_items, d, seed=13)
    i[20_000:20_030] = i[20_000]  # exact duplicates inside one shard: ties at the cut for the rows that like them
    u[:40] = (u[:40] * 0.05 + 3.0 * i[20_000][None, :]).astype(np.float32)
    csr = synth_viewed_csr(n_users, n_items, 30)
    dev = torch.device("cuda:0")
    d_users = torch.from_numpy(u).to(dev)
    d_indptr = torch.from_numpy(csr.indptr.astype(np.int64)).to(dev)
    d_indices = torch.from_numpy(csr.indices.astype(np.int32)).to(dev)
    bufs = []
    local = None
    for s, (lo, hi) in enumerate(shard_bounds(n_items, shards)):
        local = EngineShard(i[lo:hi], False, lo, 0, "auto")
        pk = Packed(torch, n_users, k, dev)
        st = local.local_topk(n_users, k, pk, shared_epoch=7, subjects=d_users.data_ptr(), indptr=d_indptr.data_ptr(),
                              indices=d_indices.data_ptr(), flags=_lib.Q_INPUTS_ON_DEVICE | _lib.Q_FORCE_TC)
        assert st["path"] == 1 and st["n_fallback_rows"] == 0  # no local verdict in this mode
        assert torch.isfinite(pk.bounds).any()
        bufs.append(pk.buf)
    g = torch.cat(bufs)
    o_ids, o_sc, o_cnt, fail_rows, fail_count = local.merge(g, shards, n_users, k, certified=True)
    torch.cuda.synchronize()
    n_fail = int(fail_count.item())
    assert 0 < n_fail < n_users // 4  # the planted ties (at least) cannot be certified
    rows = np.sort(fail_rows[:n_fail].cpu().numpy())
    assert set(range(40)) <= set(rows.tolist())
    ids, sc, cnt = o_ids.cpu().numpy(), o_sc.cpu().numpy(), o_cnt.cpu().numpy()
    ok = np.setdiff1d(np.arange(n_users), rows)
    sel = ok[::3]
    _, oid, osc = rank_oracle("dot", u, i, sel, k, csr[sel], accum="f64")
    np.testing.assert_array_equal(ids[sel].reshape(-1), oid)
    np.testing.assert_allclose(sc[sel].reshape(-1), osc, rtol=3e-7, atol=1e-9)
    assert (cnt[sel] == k).all()


@pytest.mark.parametrize("n_gpus", [2])
def test_sharded_ranker_under_torchrun(n_gpus, tmp_path):
    import torch

    from tests.sharded_cases import check_results, free_port

    if torch.cuda.device_count() < n_gpus:
        pytest.skip(f"needs {n_gpus} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n_gpus}", "--master-addr", "127.0.0.1",
           "--master-port", str(free_port()), os.path.join(ROOT, "scripts", "dist_gpu_check.py"), "--out", str(tmp_path)]
    res = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    sys.stdout.write(res.stdout[-4000:])
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    report = check_results(str(tmp_path), f"items{n_gpus}", ["edges", "tiny", "certificate"], "engine")
    assert "bit-identical" in report

"""GPU: `ShardedB200Ranker`, unmodified, on real engines with one GPU -- several ranks, one device.

Every rank is a process with its own CUDA context and its own engine on device 0; gloo carries the collectives and the
published-threshold arrays are opened across the processes through CUDA IPC (`b200_rank_peer_export` / `_import`), so the
PEERS kernels of different processes read each other's arrays.  tests/sharded_cases.py holds the case table, the worker and
the launcher; this file starts the ranks (`--backend gloo --one-device --provider engine`), asserts that every rank wrote
bit-identical results, and compares rank 0 with the fp64 oracle on every row of every call.

Collectives: this torch's gloo takes CUDA tensors for `all_to_all_single`, `all_gather_into_tensor` and `all_gather`
directly; the worker probes them at start, falls back to pinned-host staging for one that is refused, and prints which is
in use (asserted below, so a change of either kind is noticed).

What still needs two GPUs: NCCL itself, NVLink peer access and `cudaIpcMemLazyEnablePeerAccess` across devices
(tests/test_gpu_sharded.py::test_sharded_ranker_under_torchrun, same case table)."""
import json
import os

import pytest

from tests import sharded_cases as sc

pytestmark = pytest.mark.gpu


def _run(config, cases, tmp_path, capsys):
    world, _ = sc.CONFIGS[config]
    out = str(tmp_path)
    text = sc.launch(world, ["--backend", "gloo", "--one-device", "--provider", "engine", "--configs", config, "--cases", ",".join(cases)],
                     out, timeout=600)
    report = sc.check_results(out, config, cases, "engine")
    with capsys.disabled():
        print("\n" + text + report)
    with open(os.path.join(out, "rank0.json"), encoding="utf-8") as f:
        return json.load(f)


@pytest.mark.parametrize("config", list(sc.CONFIGS))
def test_sharded_ranker_on_one_gpu(config, tmp_path, capsys):
    """One launch per configuration (a CUDA context per rank is the expensive part), three cases.

    `edges`, `tiny`: world 2 and 3 with item shards, 4 as a 2 x 2 grid, 3 with subject sharding; DOT / COSINE with and without threshold
    sharing, EUCLIDEAN through `rank`: ragged and empty shards, k_loc < k, empty and short local whitelists, batches of 1, 2,
    world - 1, world + 1 and 37 rows, k = 1 .. 1025 and None, everything-viewed rows, exact duplicates in different shards and
    at shard boundaries, a tie of the k-th and (k+1)-th across two shards, zero-norm vectors.

    `certificate`: 40 equal objects, 35 subjects aimed at them, spread over the slices of the all-to-all, the last row of the batch and
    rows with empty filter rows among them.  With sharing on, the fused kernel ranks (path 1), the global certificate rejects
    at least the planted rows and they are re-ranked: through `rank` (CSR sub-matrix), `rank_device` with CUDA tensors
    (gathered filter rows) and with host arrays.  Three consecutive `rank_device` calls of n, n/2 and n rows on one ranker
    (epochs), a call with more rows than `max_rows` and a ranker whose arrays hold one row (both unshared, both right), bf16
    operands, uneven subject-group slices.  On pure item sharding also: each rank checks the fused kernel's snapshot of one
    shared call (I1-I4, I7) and the global I6 against the justifications gathered from the other processes, and prints the
    fraction of thresholds adopted from a peer process (not asserted: it depends on how the processes are time-sliced); then
    a second `enable_sharing` is refused, rank 0 destroys its engines while the others still map their arrays, and a new
    ranker in the same group ranks correctly."""
    info = _run(config, ["edges", "tiny", "certificate"], tmp_path, capsys)
    assert all(v == "cuda" for v in info["collectives"].values()), info["collectives"]
    stats = info["stats"]
    item_sharded = sc.CONFIGS[config][1] != 1
    shared = [k for k, v in stats.items() if v.get("n_uncertified_rows") is not None]
    assert bool(shared) == item_sharded and all(stats[k]["sharing"] for k in shared)
    first = stats[f"{config}|certificate|rank/shared"]
    assert first["sharing"] == item_sharded
    if item_sharded:
        assert first["path"] == 1 and first["n_uncertified_rows"] >= first["planted_in_group"] > 0
        assert stats[f"{config}|certificate|device_cuda/2-half"]["n_uncertified_rows"] >= 1
    if sc.CONFIGS[config][1] is None:
        assert stats[f"{config}|certificate|device_cuda/over-max_rows"]["n_uncertified_rows"] is None
        assert stats[f"{config}|certificate|device_cuda/one-row-arrays"]["n_uncertified_rows"] is None
        assert 0.0 <= stats[f"{config}|certificate|snapshot"]["adopted_fraction"] <= 1.0
        assert stats[f"{config}|certificate|after-close"]["n_uncertified_rows"] >= len(sc.PLANTED)

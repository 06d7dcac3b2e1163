"""`ShardedB200Ranker` on W ranks, whatever the backend: one case table, a worker that runs it, a launcher that starts the
ranks and never leaves one behind, and the every-row comparison with the fp64 oracle.

    python -m tests.sharded_cases --backend gloo --one-device --provider engine --out DIR     (under RANK / WORLD_SIZE / MASTER_*)

* `--backend nccl`: one device per rank (torchrun, scripts/dist_gpu_check.py).  `--backend gloo --one-device`: every rank holds
  an engine on device 0; CUDA IPC handles open across processes of one device, so threshold sharing is the real thing.
* `--provider oracle` plugs `OracleShard` in: the case generators, expectations, comparisons and the process handling run on
  a machine without a GPU (tests/test_sharded_cases_cpu.py).
* gloo collectives on CUDA tensors are probed once per process group; one that is refused is rebound on the
  `torch.distributed` module to a wrapper that stages through pinned host tensors (`ShardedB200Ranker` looks the functions
  up through `self.dist` at call time).  The worker prints which of the two is in use.

Every rank writes the padded result of every call to `--out`; the parent (`check_results`) asserts the ranks agree bit for
bit and compares rank 0 with `oracle.topk_oracle` at accum="f64" on every row.  Nothing here waits for a peer's kernel:
kernels of different processes on one GPU are time-sliced, stale thresholds are only weaker bounds."""
from __future__ import annotations

import argparse
import dataclasses
import datetime
import json
import os
import socket
import subprocess
import sys
import time
import typing as tp

import numpy as np
from scipy import sparse

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.topk_oracle import implicit_topk, rank_oracle  # noqa: E402
from rectools_b200.sharded import merge_padded_numpy, shard_bounds, split_whitelist  # noqa: E402
from tests.helpers import assert_same_ranking, synth_factors, synth_viewed_csr  # noqa: E402

FLT_MAX = np.finfo(np.float32).max
# name -> (world, item_shards): pure item sharding, the item x subject grid, pure subject sharding with ragged slices
CONFIGS: tp.Dict[str, tp.Tuple[int, tp.Optional[int]]] = {"items2": (2, None), "items3": (3, None), "grid2x2": (4, 2), "subjects3": (3, 1)}


class OracleShard:
    """Local top-k provider with the EngineShard interface, backed by the numpy oracle (test infrastructure only)."""

    def __init__(self, objects, cosine, lo):
        self.objects, self.cosine, self.lo = objects, cosine, lo
        self.subjects = None

    def set_subjects(self, subjects):
        self.subjects = subjects

    def local_topk(self, subject_ids, k, indptr, indices, whitelist_local):
        import torch

        n = len(subject_ids)
        objs = self.objects if whitelist_local is None else self.objects[whitelist_local]
        n_pos = objs.shape[0]
        k_loc = min(k, n_pos)
        ids = np.full((n, k_loc), -1, dtype=np.int32)
        sc = np.full((n, k_loc), -FLT_MAX, dtype=np.float32)
        cnt = np.zeros(n, dtype=np.int32)
        if k_loc == 0 or n == 0:
            return torch.from_numpy(ids), torch.from_numpy(sc), torch.from_numpy(cnt)
        filt = None
        if indptr is not None:
            # global column ids -> local positions of this shard (and of the whitelist)
            rows = np.repeat(np.arange(n), np.diff(indptr))
            cols = np.asarray(indices, dtype=np.int64) - self.lo
            keep = (cols >= 0) & (cols < self.objects.shape[0])
            rows, cols = rows[keep], cols[keep]
            if whitelist_local is not None:
                pos = np.searchsorted(whitelist_local, cols)
                ok = (pos < len(whitelist_local)) & (whitelist_local[np.minimum(pos, len(whitelist_local) - 1)] == cols)
                rows, cols = rows[ok], pos[ok]
            filt = sparse.csr_matrix((np.ones(len(rows), np.float32), (rows, cols)), shape=(n, n_pos))
        norms = None
        if self.cosine:
            norms = np.sqrt((objs.astype(np.float64) ** 2).sum(1)).astype(np.float32)
            norms[norms == 0] = 1e-10
        tid, tsc = implicit_topk(objs, self.subjects[subject_ids], k_loc, norms, filt, accum="f64")
        valid = tsc > -1e38
        cnt[:] = valid.sum(1)
        loc = tid if whitelist_local is None else np.asarray(whitelist_local)[tid]
        ids[valid] = (loc + self.lo)[valid]
        sc[valid] = tsc[valid]
        return torch.from_numpy(ids), torch.from_numpy(sc), torch.from_numpy(cnt)

    def merge(self, ids, sc, cnt, k):
        import torch

        o = merge_padded_numpy(ids.numpy(), sc.numpy(), cnt.numpy(), k)
        return tuple(torch.from_numpy(x) for x in o)


# ------------------------------------------------------------------------------------------------------- the case table
@dataclasses.dataclass(frozen=True)
class RankerSpec:
    distance: str = "dot"
    share: bool = False
    with_subjects: bool = True
    max_rows: tp.Optional[int] = None
    tc_mode: str = "auto"


@dataclasses.dataclass
class Call:
    """One ranking call of a case.  kind "rank": `sids` + a CSR with one row per id; "device_cuda" / "device_host":
    `rank_device` with the subject matrix `sub` of the whole batch, cut into the subject groups' slices `group_rows`.
    `planted`: batch rows the global certificate must reject when the call shares thresholds; `expect_shared`: None = not
    asserted."""

    key: str
    ranker: RankerSpec
    kind: str = "rank"
    sids: tp.Optional[np.ndarray] = None
    sub: tp.Optional[np.ndarray] = None
    k: tp.Optional[int] = 10
    csr: tp.Optional[sparse.csr_matrix] = None
    wl: tp.Optional[np.ndarray] = None
    group_rows: tp.Optional[tp.List[tp.Tuple[int, int]]] = None
    planted: tp.Optional[np.ndarray] = None
    expect_shared: tp.Optional[bool] = None


@dataclasses.dataclass
class Case:
    name: str
    edge: str
    u: np.ndarray
    i: np.ndarray
    calls: tp.List[Call]
    proof: tp.List[str]  # what the data shows about the edge (asserted while it is generated)
    extra: tp.Optional[str] = None  # engine-only steps after the calls: "snapshot" / "lifetime"


def _csr_from_rows(rows: tp.List[np.ndarray], n_cols: int) -> sparse.csr_matrix:
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    indices = np.concatenate(rows).astype(np.int32) if rows else np.empty(0, np.int32)
    return sparse.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(len(rows), n_cols))


EDGE_KS = (1, 6, 10, 24, 25, 33, 100, 1025)


def edges_case(world: int, item_shards: tp.Optional[int], provider: str) -> Case:
    """A 1301 x 16 catalogue (prime: no world size divides it) and 37 subjects with every small edge of the exchange."""
    I = world if item_shards is None else item_shards
    n_users, n_items, d = 37, 1301, 16
    u, i = synth_factors(n_users, n_items, d, seed=5)
    b = shard_bounds(n_items, I)
    dup = np.unique(np.concatenate([[lo, lo + 3, lo + 5, lo + 8, lo + 13, hi - 1] for lo, hi in b]))
    i[dup] = i[0]
    u[:5] = (0.05 * u[:5] + 3.0 * i[0][None, :]).astype(np.float32)
    i[7] = 0  # zero-norm object
    u[9] = 0  # zero-norm subject
    rng = np.random.default_rng(11)
    rows = [np.sort(rng.choice(n_items, 20, replace=False)) for _ in range(n_users)]
    rows[5] = np.arange(n_items)  # everything viewed
    rows[6] = np.arange(b[-1][0], b[-1][1]) if I > 1 else np.arange(600, n_items)  # ids of one other shard only
    rows[7] = np.empty(0, np.int64)
    csr_all = _csr_from_rows(rows, n_items)
    sids = np.arange(n_users)[::-1].copy()
    csr = csr_all[sids]
    lo0, hi0 = b[0]
    wl_empty = np.arange(lo0, hi0, 2)  # every other shard's local whitelist is empty
    wl_short = np.sort(np.concatenate([np.arange(lo0, hi0, 3)] + [np.arange(lo, min(lo + 3, hi)) for lo, hi in b[1:]]))
    # ---- proof from the data
    proof = [f"n_items={n_items} % world {world} = {n_items % world}, shards {b}"]
    assert n_items % world != 0 and all(n_items % s for s in (2, 3, 4))
    s_all = u.astype(np.float64) @ i.astype(np.float64).T
    order = np.lexsort((np.arange(n_items), -s_all[0]))
    assert set(order[: len(dup)].tolist()) == set(dup.tolist()) and len(np.unique(s_all[0][dup])) == 1
    shard_of = lambda x: int(np.searchsorted([hi for _, hi in b], x, side="right"))
    if I > 1:
        assert {shard_of(x) for x in dup} == set(range(I)) and all(lo in dup and hi - 1 in dup for lo, hi in b)
        assert shard_of(order[5]) != shard_of(order[6])  # k = 6: the k-th and the (k+1)-th tie across two shards
        proof.append(f"{len(dup)} exact duplicates in {I} shards, at every shard's first and last id; subject 0 ranks them first; "
                     f"its 6th ({order[5]}, shard {shard_of(order[5])}) and 7th ({order[6]}, shard {shard_of(order[6])}) tie")
        assert max(hi - lo for lo, hi in b) < 1025 < n_items
        proof.append(f"k=1025 > every shard ({max(hi - lo for lo, hi in b)} objects): k_loc < k on every rank")
        assert all(len(split_whitelist(wl_empty, lo, hi)) == 0 for lo, hi in b[1:]) and len(split_whitelist(wl_empty, lo0, hi0)) > 0
        assert all(0 < len(split_whitelist(wl_short, lo, hi)) < 10 for lo, hi in b[1:])
        proof.append(f"whitelist A leaves shards 1.. no position; whitelist B leaves them {[len(split_whitelist(wl_short, lo, hi)) for lo, hi in b[1:]]} (< k=10)")
    assert csr_all[5].nnz == n_items and csr_all[7].nnz == 0 and (I == 1 or (csr_all[6].indices >= b[0][1]).all())
    proof.append("subject 5 has viewed everything, subject 6 only ids outside shard 0, subject 7 nothing; subject 9 and object 7 are zero vectors")
    # ---- calls
    calls = []
    shares = (False,) if provider == "oracle" else (True, False)
    for dist_name in ("dot", "cosine", "euclidean"):
        for share in shares:
            if share and dist_name == "euclidean":
                continue
            spec = RankerSpec(dist_name, share)
            tag = f"{dist_name}/share={int(share)}"
            for k in EDGE_KS:
                calls.append(Call(f"{tag}/k={k}", spec, sids=sids, k=k, csr=csr, expect_shared=(share and I > 1 and k <= 24) if share else False))
            for n in sorted({1, 2, world - 1, world + 1}):
                calls.append(Call(f"{tag}/n={n}", spec, sids=sids[:n], k=10, csr=csr[:n]))
            calls.append(Call(f"{tag}/wlA", spec, sids=sids, k=10, csr=csr, wl=wl_empty))
            calls.append(Call(f"{tag}/wlB", spec, sids=sids, k=10, csr=None, wl=wl_short))
            calls.append(Call(f"{tag}/wlB/k=None", spec, sids=sids, k=None, csr=csr, wl=wl_short))
            calls.append(Call(f"{tag}/wlA/k=None", spec, sids=sids, k=None, csr=None, wl=wl_empty))
    return Case("edges", "ragged shards, duplicates across shards, k_loc < k, empty local whitelists, tiny batches, k up to 1025, "
                "EUCLIDEAN and zero norms", u, i, calls, proof)


def tiny_case(world: int, item_shards: tp.Optional[int], provider: str) -> Case:
    """A catalogue smaller than the number of item shards: the last shard is empty."""
    I = world if item_shards is None else item_shards
    n_items = {1: 3, 2: 1, 3: 4}.get(I, 2)
    u, i = synth_factors(9, n_items, 8, seed=2)
    b = shard_bounds(n_items, I)
    proof = [f"n_items={n_items}: shards {b}"]
    if I > 1:
        assert b[-1][0] == b[-1][1]
        proof.append(f"shard {I - 1} is empty")
    rows = [np.empty(0, np.int64) for _ in range(9)]
    rows[0] = np.arange(n_items)
    csr = _csr_from_rows(rows, n_items)
    calls = []
    for dist_name in ("dot", "cosine"):
        for share in (False,) if provider == "oracle" else (True, False):
            spec = RankerSpec(dist_name, share)
            calls.append(Call(f"{dist_name}/share={int(share)}/k=3", spec, sids=np.arange(9), k=3))
            calls.append(Call(f"{dist_name}/share={int(share)}/viewed", spec, sids=np.arange(9), k=3, csr=csr))
    return Case("tiny", "a catalogue with fewer objects than item shards", u, i, calls, proof)


N_BIG, ITEMS_BIG = 600, 100_003
PLANTED = np.concatenate([np.arange(12), np.arange(295, 306), np.arange(588, 600)])


def _big_data():
    u, i = synth_factors(N_BIG, ITEMS_BIG, 64, seed=21)
    i[50_000:50_040] = i[50_000]  # ties at the cut for the subjects below: rows the global certificate must reject
    # twelve objects of ONE candidate list (ids 50 048 .. 50 059 share a 64-wide quarter of the tile stream) that the same
    # subjects score above everything else, all different: a shared pass keeps at most K' < 10 of them, so the merged row is
    # wrong until the re-rank replaces it -- a re-ranked row scattered to the wrong index cannot go unnoticed
    i[50_048:50_060] = i[50_000][None, :] * (1.5 - 0.02 * np.arange(12, dtype=np.float32))[:, None]
    u[PLANTED] = (u[PLANTED] * 0.05 + 3.0 * i[50_000][None, :]).astype(np.float32)
    keep = np.ones(N_BIG)
    keep[[3, 300, N_BIG - 1]] = 0  # planted rows with an empty filter row, the last row of the batch among them
    csr = sparse.csr_matrix(sparse.diags(keep) @ synth_viewed_csr(N_BIG, ITEMS_BIG, 40))
    csr.eliminate_zeros()
    csr.sort_indices()
    return u, i, csr


def _group_rows(world: int, item_shards: tp.Optional[int], n: int) -> tp.List[tp.Tuple[int, int]]:
    """Slices of a `rank_device` batch: uneven on purpose when there are several subject groups."""
    groups = 1 if item_shards is None else world // item_shards
    cuts = {1: [0, n], 2: [0, n * 7 // 12, n], 3: [0, n * 5 // 12, n * 9 // 12, n]}[groups]
    return [(cuts[g], cuts[g + 1]) for g in range(groups)]


def certificate_case(world: int, item_shards: tp.Optional[int], provider: str) -> Case:
    """40 equal objects and 35 subjects aimed at them: with threshold sharing the global certificate rejects those rows and
    they are re-ranked; host inputs (`rank`) and device / host matrices (`rank_device`), consecutive calls, sharing limits."""
    I = world if item_shards is None else item_shards
    groups = world // I
    u, i, csr = _big_data()
    n_group = -(-N_BIG // groups)  # rows of `rank`'s subject group 0
    per = -(-n_group // I)
    slices = sorted({int(r) // per for r in PLANTED if r < n_group})
    proof = [f"{len(PLANTED)} planted rows {PLANTED[0]}..{PLANTED[11]}, {PLANTED[12]}..{PLANTED[22]}, {PLANTED[23]}..{PLANTED[-1]}; "
             f"all-to-all slices of {per} rows: group 0's planted rows fall into slices {slices}"]
    assert csr[3].nnz == 0 and csr[N_BIG - 1].nnz == 0 and N_BIG - 1 in PLANTED and 3 in PLANTED
    if I > 1 and groups == 1:
        assert len(slices) > 1 and any(r % per == 0 for r in PLANTED) and any(r % per == per - 1 for r in PLANTED)
        proof.append("planted rows sit at the last row of one slice and the first of the next; rows 3 and 599 (planted) have empty filter rows")
    sids = np.arange(N_BIG)
    shared = I > 1
    gr = _group_rows(world, item_shards, N_BIG)
    big = max(b - a for a, b in gr) * groups  # max_rows is split evenly over the subject groups: room for the longest slice
    calls = [Call("rank/shared", RankerSpec("dot", True), sids=sids, csr=csr, planted=PLANTED, expect_shared=shared)]
    if provider == "engine":
        dev = RankerSpec("dot", True, with_subjects=False, max_rows=big)
        half = _group_rows(world, item_shards, N_BIG // 2)
        calls += [
            Call("device_cuda/1", dev, "device_cuda", sub=u, csr=csr, group_rows=gr, planted=PLANTED, expect_shared=shared),
            # other subjects in the rows of the call before: with the same epoch their stale words would count as thresholds
            Call("device_cuda/2-half", dev, "device_cuda", sub=u[N_BIG // 2 :], csr=csr[N_BIG // 2 :], group_rows=half,
                 planted=PLANTED[PLANTED >= N_BIG // 2] - N_BIG // 2, expect_shared=shared),
            Call("device_cuda/3", dev, "device_cuda", sub=u, csr=csr, group_rows=gr, planted=PLANTED, expect_shared=shared),
            Call("device_host", dev, "device_host", sub=u, csr=csr, group_rows=gr, planted=PLANTED, expect_shared=shared),
            Call("rank/shared/again", RankerSpec("dot", True), sids=sids[::-1].copy(), csr=csr[sids[::-1]], planted=N_BIG - 1 - PLANTED,
                 expect_shared=shared),
        ]
        if groups == 1 and I > 1:
            calls += [
                # more rows than the published arrays hold: the call runs unshared
                Call("device_cuda/over-max_rows", RankerSpec("dot", True, False, N_BIG // 2), "device_cuda", sub=u, csr=csr, group_rows=gr,
                     expect_shared=False),
                # no subjects and no max_rows at construction: the arrays hold one row
                Call("device_cuda/one-row-arrays", RankerSpec("dot", True, False, None), "device_cuda", sub=u, csr=csr, group_rows=gr,
                     expect_shared=False),
                Call("device_cuda/one-row-arrays/n=1", RankerSpec("dot", True, False, None), "device_cuda", sub=u[:1], csr=csr[:1],
                     group_rows=[(0, 1)], expect_shared=True),
                # (bf16 plans longer lists, which hold the ten planted objects: rejections are not guaranteed, the result is)
                Call("device_cuda/bf16", RankerSpec("dot", True, False, N_BIG, "bf16"), "device_cuda", sub=u, csr=csr, group_rows=gr,
                     expect_shared=True),
                Call("rank/cosine", RankerSpec("cosine", True), sids=sids, csr=csr, expect_shared=True),
            ]
    return Case("certificate", "rows the global certificate rejects, spread over slices; re-rank from host and device inputs; epochs; "
                "sharing limits", u, i, calls, proof, extra="snapshot+lifetime" if provider == "engine" and groups == 1 and I > 1 else None)


CASES: tp.Dict[str, tp.Callable[[int, tp.Optional[int], str], Case]] = {"edges": edges_case, "tiny": tiny_case, "certificate": certificate_case}


# ------------------------------------------------------------------------------------------------------- the worker
def _stage_collectives(torch, dist, device) -> tp.Dict[str, str]:
    """Probe the collectives `sharded.py` calls on CUDA tensors; rebind a refused one to a pinned-host staging wrapper."""
    world = dist.get_world_size()
    used = {}

    def probe(name, fn):
        try:
            fn()
            torch.cuda.synchronize()
            used[name] = "cuda"
        except (RuntimeError, NotImplementedError, ValueError) as e:  # refused before any communication, on every rank alike
            used[name] = f"host-staged ({str(e).splitlines()[0][:80]})"
            return False
        return True

    t = torch.arange(world, dtype=torch.int32, device=device)
    if not probe("all_to_all_single", lambda: dist.all_to_all_single(torch.empty_like(t), t)):
        orig_a2a = dist.all_to_all_single

        def all_to_all_single(output, input, *args, **kw):  # pylint: disable=redefined-builtin
            if not input.is_cuda:
                return orig_a2a(output, input, *args, **kw)
            o = torch.empty(output.shape, dtype=output.dtype, pin_memory=True)
            orig_a2a(o, input.cpu(), *args, **kw)
            output.copy_(o)
            return None

        dist.all_to_all_single = all_to_all_single
    if not probe("all_gather_into_tensor", lambda: dist.all_gather_into_tensor(torch.empty(world * world, dtype=torch.int32, device=device), t)):
        orig_agt = dist.all_gather_into_tensor

        def all_gather_into_tensor(output, input, *args, **kw):  # pylint: disable=redefined-builtin
            if not input.is_cuda:
                return orig_agt(output, input, *args, **kw)
            o = torch.empty(output.shape, dtype=output.dtype, pin_memory=True)
            orig_agt(o, input.cpu(), *args, **kw)
            output.copy_(o)
            return None

        dist.all_gather_into_tensor = all_gather_into_tensor
    if not probe("all_gather", lambda: dist.all_gather([torch.empty_like(t) for _ in range(world)], t)):
        orig_ag = dist.all_gather

        def all_gather(tensors, tensor, *args, **kw):
            if not tensor.is_cuda:
                return orig_ag(tensors, tensor, *args, **kw)
            host = [torch.empty(x.shape, dtype=x.dtype) for x in tensors]
            orig_ag(host, tensor.cpu(), *args, **kw)
            for dst, src in zip(tensors, host):
                dst.copy_(src)
            return None

        dist.all_gather = all_gather
    return used


class Worker:
    def __init__(self, args):
        import torch
        import torch.distributed as dist

        self.torch, self.dist, self.args = torch, dist, args
        self.rank, self.world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
        self.engine = args.provider == "engine"
        self.device = None
        if self.engine:
            if args.one_device and args.backend != "gloo":
                raise SystemExit("--one-device needs --backend gloo: NCCL refuses two ranks on one device")
            index = 0 if args.one_device else int(os.environ.get("LOCAL_RANK", self.rank))
            torch.cuda.set_device(index)
            self.device = torch.device("cuda", index)
        kw = dict(device_id=self.device) if args.backend == "nccl" else {}
        dist.init_process_group(args.backend, rank=self.rank, world_size=self.world, timeout=datetime.timedelta(seconds=120), **kw)
        self.collectives = {}
        if self.engine and args.backend == "gloo":
            self.collectives = _stage_collectives(torch, dist, self.device)
        self.arrays: tp.Dict[str, np.ndarray] = {}
        self.stats: tp.Dict[str, tp.Any] = {}

    def say(self, msg):
        if self.rank == 0:
            print(msg, flush=True)

    def make_ranker(self, case: Case, spec: RankerSpec, item_shards):
        from rectools_b200.sharded import ShardedB200Ranker

        kw = dict(item_shards=item_shards, share_thresholds=spec.share, max_rows=spec.max_rows)
        if self.engine:
            kw.update(tc_mode=spec.tc_mode)
        else:
            kw.update(local_factory=OracleShard)
        return ShardedB200Ranker(spec.distance, case.u if spec.with_subjects else None, case.i, **kw)

    def run_call(self, ranker, call: Call, prefix: str):
        torch = self.torch
        key = f"{prefix}|{call.key}"
        if call.kind == "rank":
            seen = {}
            inner = type(ranker).rank_padded

            def spy(*a, **kw):
                out = inner(ranker, *a, **kw)
                seen["padded"] = [t.cpu().numpy().copy() for t in out[1:]]
                return out

            ranker.rank_padded = spy
            try:
                flat = ranker.rank(call.sids, call.k, call.csr, call.wl)
            finally:
                del ranker.rank_padded
            padded = seen["padded"]
            for name, a in zip(("fsub", "fids", "fsc"), flat):
                self.arrays[f"{key}|{name}"] = np.asarray(a)
            my_rows = shard_bounds(len(call.sids), ranker.subject_groups)[ranker.group_idx]
        else:
            a, b = call.group_rows[ranker.group_idx]
            sub = np.ascontiguousarray(call.sub[a:b])
            ip = np.ascontiguousarray(call.csr.indptr[a : b + 1].astype(np.int64) - int(call.csr.indptr[a]))
            ix = np.ascontiguousarray(call.csr.indices[int(call.csr.indptr[a]) : int(call.csr.indptr[b])].astype(np.int32))
            if call.kind == "device_cuda":
                sub, ip, ix = (torch.from_numpy(x).to(self.device) for x in (sub, ip, ix))
            out = ranker.rank_device(sub, call.k, ip, ix)
            torch.cuda.synchronize()
            padded = [t.cpu().numpy() for t in out]
            my_rows = (a, b)
        for name, a_ in zip(("ids", "sc", "cnt"), padded):
            self.arrays[f"{key}|{name}"] = a_
        st = dict(ranker.last_stats)
        info = {"sharing": bool(getattr(ranker.local, "sharing", False)), "path": st.get("path"), "n_uncertified_rows": st.get("n_uncertified_rows")}
        if self.engine and call.expect_shared is not None and my_rows[1] > my_rows[0]:
            assert ("n_uncertified_rows" in st) == call.expect_shared, (key, st, call.expect_shared)
            if call.expect_shared:
                assert ranker.local.sharing
                if call.planted is not None:
                    mine = int(((call.planted >= my_rows[0]) & (call.planted < my_rows[1])).sum())
                    info["planted_in_group"] = mine
                    assert st["path"] == 1 and st["n_uncertified_rows"] >= mine, (key, st, mine)
                    # thresholds of another call or of other rows reject far more than the planted ties
                    assert st["n_uncertified_rows"] <= mine + (my_rows[1] - my_rows[0]) // 10, (key, st, mine)
        self.stats[key] = info
        self.say(f"  {key}: sharing={info['sharing']} path={info['path']} n_uncertified_rows={info['n_uncertified_rows']}"
                 + (f" (planted in this group: {info['planted_in_group']})" if "planted_in_group" in info else ""))

    # ---- engine-only steps
    def snapshot_step(self, case: Case, ranker, prefix: str):
        """One shared `rank_device` call under B200_TC_SNAPSHOT=1: every rank checks its own pass (I1-I4, I7) and the global
        form of I6 -- no threshold above the largest justification of any list of any shard -- with the justifications
        gathered from the other processes."""
        from tests.tc_reference import Catalogue, SharedPass, check_snapshot, list_justification

        torch, dist = self.torch, self.dist
        u, _, csr = case.u, case.i, _big_data()[2]
        lo, hi = ranker.lo, ranker.hi
        cat = Catalogue(case.i[lo:hi], cosine=False, bf16=False, id_off=lo)
        seen = {}
        shard = ranker.local
        inner = type(shard).local_topk

        def spy(n_rows, k, out, shared_epoch=0, **inputs):
            st = inner(shard, n_rows, k, out, shared_epoch=shared_epoch, **inputs)
            if shared_epoch and "snap" not in seen:  # (the re-rank's call would replace the snapshot)
                seen["snap"] = shard.engine.candidate_snapshot()
                seen["bounds"] = out.bounds.cpu().numpy().copy()
            return st

        shard.local_topk = spy
        os.environ["B200_TC_SNAPSHOT"] = "1"
        try:
            d_in = [torch.from_numpy(np.ascontiguousarray(x)).to(self.device) for x in (u, csr.indptr.astype(np.int64), csr.indices.astype(np.int32))]
            out = ranker.rank_device(d_in[0], 10, d_in[1], d_in[2])
            torch.cuda.synchronize()
        finally:
            del os.environ["B200_TC_SNAPSHOT"]
            del shard.local_topk
        for name, t in zip(("ids", "sc", "cnt"), out):
            self.arrays[f"{prefix}|snapshot|{name}"] = t.cpu().numpy()
        snap = seen["snap"]
        assert snap is not None and snap["launch"] == 1
        rows = snap["rows"].astype(np.int64)
        viewed = cat.viewed_positions(csr.indptr, csr.indices, N_BIG)[rows]
        own = list_justification(snap, cat, u[rows], viewed)
        gathered: tp.List[tp.Any] = [None] * self.world
        dist.all_gather_object(gathered, (rows, own))
        assert all((g[0] == rows).all() for g in gathered)
        others = np.max([g[1] for r, g in enumerate(gathered) if r != self.rank], axis=0)
        sp = SharedPass(seen["bounds"][rows], ranker.epoch, np.zeros((0, len(rows)), np.uint64), others)
        rep = check_snapshot(snap, cat, u[rows], viewed, shared=sp)
        thr = snap["cand_thr"][:, : len(rows)].astype(np.float64)
        adopted = thr > np.ldexp(own, int(snap["obj_exp"]))[None, :]
        print(f"  {prefix}|snapshot rank {self.rank}: K'={snap['k_cand']} lists={thr.shape[0]} {rep.summary()} "
              f"thresholds above the rank's own justification (adopted from a peer process): {int(adopted.sum())}/{adopted.size} = "
              f"{adopted.mean():.3f}", flush=True)
        assert rep.ok, rep.summary()
        self.stats[f"{prefix}|snapshot"] = {"adopted_fraction": float(adopted.mean()), "k_cand": int(snap["k_cand"])}

    def lifetime_step(self, case: Case, rankers: tp.Dict[RankerSpec, tp.Any], prefix: str, item_shards):
        """Several rankers lived side by side in this group (an export and an import each).  A second `enable_sharing` on a
        shard is refused; rank 0 destroys its engines while the others still map their arrays; a new ranker then works."""
        dist = self.dist
        first = rankers[RankerSpec("dot", True)]
        assert sum(bool(r.local.sharing) for r in rankers.values()) >= 2
        try:
            first.local.enable_sharing(dist, first.exchange_group, N_BIG)
            raise AssertionError("a second enable_sharing was accepted")
        except ValueError as e:
            assert "already exported" in str(e), e
        assert first.local.sharing
        if self.rank != 0:
            dist.barrier()
        for r in rankers.values():
            r.local.engine.close()
        if self.rank == 0:
            dist.barrier()
        rankers.clear()
        spec = RankerSpec("dot", True)
        ranker = self.make_ranker(case, spec, item_shards)
        csr = _big_data()[2]
        self.run_call(ranker, Call("after-close", spec, sids=np.arange(N_BIG), csr=csr, planted=PLANTED, expect_shared=True), prefix)

    def run(self):
        args, dist = self.args, self.dist
        configs = args.configs.split(",") if args.configs else [c for c, (w, _) in CONFIGS.items() if w == self.world]
        try:
            if args.die_on_rank is not None:  # the launcher's failure handling: one rank fails, the others never finish by themselves
                if self.rank == args.die_on_rank:
                    sys.exit(3)
                time.sleep(3600)
            for config in configs:
                world, item_shards = CONFIGS[config]
                assert world == self.world, f"{config} needs {world} ranks"
                for name in args.cases.split(","):
                    case = CASES[name](world, item_shards, args.provider)
                    self.say(f"[{config}/{name}] world={world} item_shards={item_shards or world} backend={args.backend} provider={args.provider} "
                             f"one_device={args.one_device} collectives={self.collectives or 'cpu tensors'}\n  edge: {case.edge}\n  "
                             + "\n  ".join(case.proof))
                    prefix = f"{config}|{name}"
                    rankers: tp.Dict[RankerSpec, tp.Any] = {}
                    for call in case.calls:
                        if call.ranker not in rankers:
                            rankers[call.ranker] = self.make_ranker(case, call.ranker, item_shards)
                            if self.engine and not call.ranker.with_subjects and call.ranker.max_rows is None and item_shards is None:
                                assert rankers[call.ranker].local.max_shared_rows == 1
                        self.run_call(rankers[call.ranker], call, prefix)
                    if case.extra:
                        self.snapshot_step(case, rankers[RankerSpec("dot", True, False, N_BIG)], prefix)
                        self.lifetime_step(case, rankers, prefix, item_shards)
                    rankers.clear()
            os.makedirs(args.out, exist_ok=True)
            np.savez(os.path.join(args.out, f"rank{self.rank}.npz"), **self.arrays)
            with open(os.path.join(args.out, f"rank{self.rank}.json"), "w", encoding="utf-8") as f:
                json.dump({"stats": self.stats, "collectives": self.collectives, "configs": configs}, f)
            dist.barrier()
            if args.check and self.rank == 0:
                for config in configs:
                    print(check_results(args.out, config, args.cases.split(","), args.provider), flush=True)
        finally:
            dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------------- the parent
def expected_padded(case: Case, call: Call):
    """fp64 oracle of one call: flat `(subjects, ids, scores)` as `rank` returns them and the padded `(ids, counts)`."""
    if call.kind == "rank":
        flat = rank_oracle(call.ranker.distance, case.u, case.i, call.sids, call.k, call.csr, call.wl, accum="f64")
        sids = call.sids
    else:
        sids = np.arange(len(call.sub))
        flat = rank_oracle("dot", call.sub, case.i, sids, call.k, call.csr, None, accum="f64")
    n_pos = case.i.shape[0] if call.wl is None else len(call.wl)
    k_out = min(n_pos if call.k is None else call.k, n_pos)
    assert len(np.unique(sids)) == len(sids)
    cnt = np.array([(flat[0] == s).sum() for s in sids], dtype=np.int64)
    ids = np.full((len(sids), k_out), -1, dtype=np.int64)
    mask = np.arange(k_out)[None, :] < cnt[:, None]
    ids[mask] = flat[1]
    return flat, ids, cnt, mask


def check_results(out: str, config: str, cases: tp.Sequence[str], provider: str) -> str:
    """All ranks bit-identical; rank 0 equal to the oracle on every row of every call.  Returns a short report."""
    world, item_shards = CONFIGS[config]
    per_rank = [np.load(os.path.join(out, f"rank{r}.npz")) for r in range(world)]
    keys = [k for k in per_rank[0].files if k.startswith(config + "|")]
    for r in range(1, world):
        assert sorted(k for k in per_rank[r].files if k.startswith(config + "|")) == sorted(keys)
        for k in keys:
            a, b = per_rank[0][k], per_rank[r][k]
            assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), f"rank {r} differs from rank 0 in {k}"
    got = per_rank[0]
    n_calls = n_rows = 0
    for name in cases:
        case = CASES[name](world, item_shards, provider)
        extra = [Call("snapshot", RankerSpec(), "device_cuda", sub=case.u, csr=_big_data()[2]),
                 Call("after-close", RankerSpec("dot", True), sids=np.arange(N_BIG), csr=_big_data()[2])] if case.extra else []
        for call in case.calls + extra:
            key = f"{config}|{name}|{call.key}"
            flat, e_ids, e_cnt, mask = expected_padded(case, call)
            ids, sc, cnt = got[f"{key}|ids"], got[f"{key}|sc"], got[f"{key}|cnt"]
            assert ids.shape == e_ids.shape and ids.dtype == np.int32 and sc.dtype == np.float32, key
            euclid = call.ranker.distance == "euclidean"
            if not euclid:  # (EUCLIDEAN: near-ties of the fp32 engine may swap neighbours; held to the flat comparison below)
                np.testing.assert_array_equal(cnt, e_cnt, err_msg=key)
                np.testing.assert_array_equal(ids, e_ids, err_msg=key)
            assert (ids[~(np.arange(ids.shape[1])[None, :] < cnt[:, None])] == -1).all(), key
            assert (sc[~(np.arange(ids.shape[1])[None, :] < cnt[:, None])] == -FLT_MAX).all(), key
            if call.kind == "rank":
                f_sub, f_ids, f_sc = got[f"{key}|fsub"], got[f"{key}|fids"], got[f"{key}|fsc"]
                np.testing.assert_array_equal(f_sub, flat[0], err_msg=key)
                if euclid:  # the tolerance of test_gpu_parity.py for EUCLIDEAN
                    assert_same_ranking(f_ids, f_sc, flat[1], flat[2], tie_tol=2e-6, atol=2e-4, msg=key)
                else:
                    np.testing.assert_array_equal(f_ids, flat[1], err_msg=key)
                    np.testing.assert_allclose(f_sc, flat[2], rtol=3e-7, atol=1e-9, err_msg=key)
                if call.ranker.distance == "dot":
                    np.testing.assert_array_equal(sc[mask], f_sc, err_msg=key)
            else:
                np.testing.assert_allclose(sc[mask], flat[2], rtol=3e-7, atol=1e-9, err_msg=key)
            n_calls += 1
            n_rows += len(ids)
    return f"[{config}] {world} ranks bit-identical; {n_calls} calls, {n_rows} rows equal to the fp64 oracle"


def free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


class LaunchFailed(AssertionError):
    def __init__(self, reason: str, procs, logs: str):
        super().__init__(f"{reason}\n{logs}")
        self.reason, self.procs = reason, procs


def launch(world: int, worker_args: tp.Sequence[str], out: str, timeout: float = 900.0) -> str:
    """Start `world` ranks of this module, wait for them with a timeout, and leave none behind: on a timeout or a non-zero
    exit of any rank the remaining ranks are killed and `LaunchFailed` is raised.  Returns rank 0's output."""
    os.makedirs(out, exist_ok=True)
    port = free_port()
    procs, logs = [], []
    try:
        for r in range(world):
            env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            logs.append(open(os.path.join(out, f"rank{r}.log"), "w+", encoding="utf-8"))  # pylint: disable=consider-using-with
            procs.append(subprocess.Popen([sys.executable, "-m", "tests.sharded_cases", "--out", out, *worker_args], cwd=ROOT, env=env,
                                          stdout=logs[-1], stderr=subprocess.STDOUT))
        deadline = time.monotonic() + timeout
        reason = None
        while reason is None:
            codes = [p.poll() for p in procs]
            if any(c not in (None, 0) for c in codes):
                reason = f"rank {[r for r, c in enumerate(codes) if c not in (None, 0)][0]} exited with {[c for c in codes if c not in (None, 0)][0]}"
            elif all(c == 0 for c in codes):
                break
            elif time.monotonic() > deadline:
                reason = f"timeout after {timeout:.0f} s"
            else:
                time.sleep(0.2)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            p.wait()
        texts = []
        for f in logs:
            f.seek(0)
            texts.append(f.read())
            f.close()
    if reason is not None:
        raise LaunchFailed(reason, procs, "\n".join(f"--- rank {r}\n{t[-3000:]}" for r, t in enumerate(texts)))
    return texts[0] + "".join(line + "\n" for t in texts[1:] for line in t.splitlines() if "|snapshot rank" in line)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--backend", choices=("nccl", "gloo"), default="gloo")
    ap.add_argument("--one-device", action="store_true", help="every rank uses device 0 (gloo only)")
    ap.add_argument("--provider", choices=("engine", "oracle"), default="engine")
    ap.add_argument("--configs", default="", help="comma-separated names of CONFIGS (default: all of this world size)")
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--out", required=True)
    ap.add_argument("--check", action="store_true", help="rank 0 compares the results with the oracle itself")
    ap.add_argument("--die-on-rank", type=int, default=None, help="that rank exits with code 3 at once (tests the launcher)")
    Worker(ap.parse_args(argv)).run()


if __name__ == "__main__":
    main()

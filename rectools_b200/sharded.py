"""Sharded ranking over several GPUs (one process per GPU, `torch.distributed`).

The reference is single-device (SURVEY.md section 2b).  Default = the north-star multi-GPU scheme (section 8e): the object
catalogue is split into contiguous ranges, every rank scores ALL subjects against its range and keeps a local top-k
with GLOBAL object ids into ONE packed buffer, the ranks exchange the buffers by subject slice (all-to-all, NCCL over NVLink
on GPUs), every rank merges the `world * k` candidates of ITS slice of the subjects and one all-gather hands the merged
slices round.  Exact local lists => exact global
top-k; ties resolve by (score desc, id asc) in the merge exactly as inside a shard.

Threshold sharing (GPUs, k <= 24): a rank's K'-th best score of a subject is a lower bound of the global K'-th best, so
every rank may prune with the maximum of ALL ranks' running thresholds.  The fused kernel publishes its thresholds to a
peer-mapped array and polls the other ranks' arrays over NVLink (helper warps, `fused_topk.cuh`); a shard of N/8 objects
then sees the hit rate of the whole catalogue instead of 8 x log(N/8) warm-ups.  Local lists are no longer complete on
their own, so every rank also reports, per subject, a bound on the scores it discarded, and the merge certifies the
global top-k against the maximum bound (`b200_rank_merge_certified`); rows that fail are re-ranked without sharing.

`item_shards=I` (a divisor of the world size) selects the other partitionings of section 8e: the ranks form a grid of
I item shards x world/I subject groups; a rank scores ITS slice of the subject batch against ITS item range, the I ranks
of a subject group exchange + merge as above, and one more all-gather among the ranks holding the same item range hands
every rank the rows of the other subject groups.  `item_shards=1` is plain subject sharding (no merge at all).
"""
from __future__ import annotations

import typing as tp

import numpy as np
from scipy import sparse

from .ranker import Distance, Engine, _as_distance, _dense_f32, check_whitelist, flatten_padded, prepare_factors, strip_sentinel_tail

NEG_MAX = -3.4028234663852886e38


def shard_bounds(n_objects: int, world_size: int) -> tp.List[tp.Tuple[int, int]]:
    """Contiguous ranges of ceil(n/world) objects (the last ones may be short or empty)."""
    per = -(-n_objects // world_size) if world_size > 0 else n_objects
    return [(min(r * per, n_objects), min((r + 1) * per, n_objects)) for r in range(world_size)]


def split_whitelist(whitelist: np.ndarray, lo: int, hi: int) -> np.ndarray:
    """Part of a sorted global whitelist that falls into [lo, hi), as LOCAL positions of that shard."""
    whitelist = np.asarray(whitelist, dtype=np.int64)
    a, b = np.searchsorted(whitelist, [lo, hi], side="left")
    return (whitelist[a:b] - lo).astype(np.int32)


def merge_padded_numpy(ids: np.ndarray, scores: np.ndarray, counts: np.ndarray, k: int):
    """Host restatement of `b200_rank_merge` (used by the CPU/gloo tests of the exchange logic only)."""
    n_lists, n_rows, _ = ids.shape
    out_ids = np.full((n_rows, k), -1, dtype=np.int32)
    out_sc = np.full((n_rows, k), -np.finfo(np.float32).max, dtype=np.float32)
    out_cnt = np.zeros(n_rows, dtype=np.int32)
    for r in range(n_rows):
        ci = np.concatenate([ids[l, r, : counts[l, r]] for l in range(n_lists)])
        cs = np.concatenate([scores[l, r, : counts[l, r]] for l in range(n_lists)])
        order = np.lexsort((ci, -cs.astype(np.float64)))[:k]
        out_ids[r, : len(order)] = ci[order]
        out_sc[r, : len(order)] = cs[order]
        out_cnt[r] = len(order)
    return out_ids, out_sc, out_cnt


class Packed:
    """One rank's results of one call in ONE int32 buffer: [ids n*k | score bits n*k | counts n | bound bits n], so that the
    exchange moves one buffer per rank.  The four views alias the buffer."""

    def __init__(self, torch: tp.Any, n: int, k: int, device: tp.Any) -> None:
        self.n, self.k = n, k
        self.stride = n * (2 * k + 2)
        self.buf = torch.empty((self.stride,), dtype=torch.int32, device=device)
        self.ids = self.buf[: n * k].view(n, k)
        self.scores = self.buf[n * k : 2 * n * k].view(torch.float32).view(n, k)
        self.counts = self.buf[2 * n * k : 2 * n * k + n]
        self.bounds = self.buf[2 * n * k + n :].view(torch.float32)

    @staticmethod
    def views(torch: tp.Any, g: tp.Any, w: int, n: int, k: int):
        """(ids [w,n,k], scores [w,n,k], counts [w,n], bounds [w,n]) views of `w` gathered buffers."""
        g = g.view(w, n * (2 * k + 2))
        ids = g[:, : n * k].reshape(w, n, k)
        sc = g[:, n * k : 2 * n * k].view(torch.float32).reshape(w, n, k)
        cnt = g[:, 2 * n * k : 2 * n * k + n]
        bnd = g[:, 2 * n * k + n :].view(torch.float32)
        return ids, sc, cnt, bnd


class EngineShard:
    """Local top-k provider backed by the CUDA engine (device tensors in / out)."""

    def __init__(self, objects: np.ndarray, cosine: bool, lo: int, device: int, tc_mode: str) -> None:
        import torch

        self.torch = torch
        self.device = torch.device("cuda", device)
        self.engine = Engine(objects, cosine=cosine, device=device, tc_mode=tc_mode, id_offset=lo)
        self.sharing = False

    def set_subjects(self, subjects: np.ndarray) -> None:
        self.engine.set_subjects(subjects)

    def enable_sharing(self, dist: tp.Any, group: tp.Any, max_rows: int) -> None:
        """Exchange the CUDA IPC handles of the published-threshold arrays with the ranks of `group` (collective)."""
        world = dist.get_world_size(group)
        if world < 2 or world > 9:
            return
        handle = self.engine.peer_export(max_rows)
        handles: tp.List[tp.Any] = [None] * world
        dist.all_gather_object(handles, handle, group=group)
        self.engine.peer_import(handles, dist.get_rank(group))
        self.sharing = True
        self.max_shared_rows = int(max_rows)

    def local_topk(self, n_rows: int, k: int, out: Packed, shared_epoch: int = 0, **inputs: tp.Any) -> tp.Dict[str, tp.Any]:
        """Rank `n_rows` subjects against this shard into `out` (its first k_loc columns when the shard is short).
        `inputs`: keyword arguments of `Engine.topk_ptrs` (raw host / device pointers + flags)."""
        from . import _lib

        torch = self.torch
        flags = int(inputs.pop("flags", 0)) | _lib.Q_OUTPUTS_ON_DEVICE
        # (a whitelist that leaves this shard no position is still a whitelist: the address of an empty array says nothing)
        n_pos_local = inputs.get("n_whitelist", 0) if "whitelist" in inputs else self.engine.n_objects
        k_loc = min(k, n_pos_local)  # the engine writes rows of k_out = min(k, local candidates) columns
        if k_loc < k:  # short shard: rank into a narrow scratch, widen into the packed buffer
            out.ids.fill_(-1)
            out.scores.fill_(NEG_MAX)
            out.counts.zero_()
            out.bounds.fill_(float("-inf"))
            if k_loc == 0 or n_rows == 0:
                return {}
            ids = torch.empty((n_rows, k_loc), dtype=torch.int32, device=self.device)
            sc = torch.empty((n_rows, k_loc), dtype=torch.float32, device=self.device)
        else:
            ids, sc = out.ids, out.scores
        if shared_epoch:
            flags |= _lib.Q_SHARED_THRESHOLDS
        st = self.engine.topk_ptrs(
            n_rows, k, ids.data_ptr(), sc.data_ptr(), out.counts.data_ptr(), flags,
            stream=torch.cuda.current_stream().cuda_stream, out_bounds=out.bounds.data_ptr() if shared_epoch else 0,
            peer_epoch=shared_epoch, **inputs,
        )
        if not shared_epoch:
            out.bounds.fill_(float("-inf"))  # locally certified lists: nothing above them was discarded
        if k_loc < k:
            out.ids[:, :k_loc] = ids
            out.scores[:, :k_loc] = sc
        return st

    def merge_into(self, g: tp.Any, w: int, n: int, k: int, certified: bool, o_ids, o_sc, o_cnt, fail_rows, fail_count) -> None:
        """Merge `w` packed buffers of `n` rows each (one after the other in `g`) into the given output tensors; with
        `certified` the rows the global certificate rejects are listed in `fail_rows` / counted in `fail_count` (zeroed here)."""
        from . import _lib

        torch = self.torch
        base = g.data_ptr()
        stride = n * (2 * k + 2)
        fail_count.zero_()
        if n == 0:  # a subject group without a row (a batch smaller than the grid): empty tensors have no address to hand over
            return
        args = (self.device.index, torch.cuda.current_stream().cuda_stream, w, n, k, base, base + 4 * n * k, base + 8 * n * k)
        if certified and k <= 32:
            _lib.check(_lib.load().b200_rank_merge_certified(
                *args, base + 8 * n * k + 4 * n, stride, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), fail_rows.data_ptr(),
                fail_count.data_ptr()))
        else:
            ids, sc, cnt, _ = Packed.views(torch, g, w, n, k)
            ids, sc, cnt = ids.contiguous(), sc.contiguous(), cnt.contiguous()
            _lib.check(_lib.load().b200_rank_merge(
                self.device.index, torch.cuda.current_stream().cuda_stream, w, n, k, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr()))

    def merge(self, g: tp.Any, w: int, n: int, k: int, certified: bool):
        """Merge `w` gathered packed buffers; returns (ids, scores, counts, fail_rows, fail_count) device tensors."""
        from . import _lib

        torch = self.torch
        o_ids = torch.empty((n, k), dtype=torch.int32, device=self.device)
        o_sc = torch.empty((n, k), dtype=torch.float32, device=self.device)
        o_cnt = torch.empty((n,), dtype=torch.int32, device=self.device)
        fail_rows = torch.empty((max(n, 1),), dtype=torch.int32, device=self.device)
        fail_count = torch.zeros((1,), dtype=torch.int32, device=self.device)
        base = g.data_ptr()
        stride = n * (2 * k + 2)
        args = (self.device.index, torch.cuda.current_stream().cuda_stream, w, n, k, base, base + 4 * n * k, base + 8 * n * k)
        if certified and k <= 32:
            _lib.check(_lib.load().b200_rank_merge_certified(
                *args, base + 8 * n * k + 4 * n, stride, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(), fail_rows.data_ptr(),
                fail_count.data_ptr()))
        else:
            ids, sc, cnt, _ = Packed.views(torch, g, w, n, k)
            ids, sc, cnt = ids.contiguous(), sc.contiguous(), cnt.contiguous()
            _lib.check(_lib.load().b200_rank_merge(
                self.device.index, torch.cuda.current_stream().cuda_stream, w, n, k, ids.data_ptr(), sc.data_ptr(), cnt.data_ptr(),
                o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr()))
        return o_ids, o_sc, o_cnt, fail_rows, fail_count


class ShardedB200Ranker:
    """`Ranker`-protocol object whose catalogue is sharded over the ranks of a `torch.distributed` group.

    `objects_factors` is the FULL matrix (every rank slices its own range) unless `objects_are_local=True`, in which case
    it is this rank's range and `n_objects_total` must be given.  Every rank must call `rank()` with the same arguments
    (SPMD); every rank returns the full, identical result.
    `local_factory(objects_local, cosine, lo)` may replace the CUDA engine with another local top-k provider -- the
    CPU (gloo) tests of the exchange logic plug the oracle in here (`local_topk_host` / `merge_host` protocol).
    `share_thresholds` (GPU provider, item shards > 1): see the module docstring; `max_rows` = the largest subject batch
    of a shared call (the published-threshold arrays are sized once).
    """

    def __init__(
        self,
        distance: tp.Any,
        subjects_factors: tp.Any,
        objects_factors: tp.Any,
        group: tp.Any = None,
        device: tp.Optional[int] = None,
        tc_mode: str = "auto",
        objects_are_local: bool = False,
        n_objects_total: tp.Optional[int] = None,
        local_factory: tp.Optional[tp.Callable[..., tp.Any]] = None,
        item_shards: tp.Optional[int] = None,
        share_thresholds: bool = True,
        max_rows: tp.Optional[int] = None,
    ) -> None:
        import torch
        import torch.distributed as dist

        self.dist, self.torch, self.group = dist, torch, group
        self.rank_id, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.item_shards = self.world if item_shards is None else int(item_shards)
        if self.item_shards < 1 or self.world % self.item_shards:
            raise ValueError("`item_shards` must divide the world size")
        self.subject_groups = self.world // self.item_shards
        self.shard_idx, self.group_idx = self.rank_id % self.item_shards, self.rank_id // self.item_shards
        # communicators: `exchange` = the ranks of my subject group (one per item shard), `collect` = the ranks that hold my
        # item range (one per subject group).  new_group is collective over the parent group: every rank creates all of them.
        self.exchange_group, self.collect_group = group, None
        if self.subject_groups > 1:
            ranks = list(range(self.world)) if group is None else dist.get_process_group_ranks(group)
            for g in range(self.subject_groups):
                grp = dist.new_group([ranks[g * self.item_shards + s] for s in range(self.item_shards)])
                if g == self.group_idx:
                    self.exchange_group = grp
            for s_ in range(self.item_shards):
                grp = dist.new_group([ranks[g * self.item_shards + s_] for g in range(self.subject_groups)])
                if s_ == self.shard_idx:
                    self.collect_group = grp
        self.distance = _as_distance(distance)
        subjects = _dense_f32(subjects_factors) if subjects_factors is not None else None
        objects = _dense_f32(objects_factors)
        n_total = int(n_objects_total) if objects_are_local else objects.shape[0]
        self.bounds = shard_bounds(n_total, self.item_shards)
        self.lo, self.hi = self.bounds[self.shard_idx]
        if not objects_are_local:
            objects = objects[self.lo : self.hi]
        if objects.shape[0] != self.hi - self.lo:
            raise ValueError("local object matrix does not match this rank's shard range")
        self.n_subjects, self.n_objects = (subjects.shape[0] if subjects is not None else 0), n_total
        self.subjects_norms = self.subjects_dots = None
        if subjects is not None:
            subjects, objects, self.subjects_norms, self.subjects_dots = prepare_factors(self.distance, subjects, objects)
        elif self.distance == Distance.EUCLIDEAN:
            raise ValueError("EUCLIDEAN needs the subject factors at construction (dot augmentation)")
        cosine = self.distance == Distance.COSINE
        self.host_provider = local_factory is not None
        if local_factory is not None:
            self.local = local_factory(objects, cosine, self.lo)
        else:
            dev = torch.cuda.current_device() if device is None else device
            self.local = EngineShard(objects, cosine, self.lo, dev, tc_mode)
        if subjects is not None:
            self.local.set_subjects(subjects)
        self.epoch = 0
        self.last_stats: tp.Dict[str, tp.Any] = {}
        if not self.host_provider and share_thresholds and self.item_shards > 1:
            rows = max_rows if max_rows is not None else max(self.n_subjects, 1)
            per_group = -(-int(rows) // self.subject_groups)
            self.local.enable_sharing(dist, self.exchange_group, per_group)

    # ------------------------------------------------------------------------------------------------------------
    def _exchange(self, pk: tp.Any, n: int, k: int, shared: bool, rerank: tp.Optional[tp.Callable[..., tp.Any]]):
        """Exchange + merge of my subject group's packed local results (SURVEY 8e, the optimised collective): an ALL-TO-ALL by
        subject slice -- rank j receives every shard's lists of rows [j n/w, (j+1) n/w) and merges only those (1/w of the
        merge work, (w-1)/w x one buffer inbound instead of (w-1) buffers) -- then ONE all-gather of the merged slices (with
        the rows the global certificate rejected).  Rejected rows are re-ranked without threshold sharing on every rank."""
        torch, w = self.torch, self.item_shards
        if w == 1:
            return pk.ids, pk.scores, pk.counts
        dev = pk.buf.device
        per = -(-n // w)  # rows per slice (the last slices may be short or empty: padded with empty rows)
        sect = per * (2 * k + 2)
        # ---- by destination: [w][ids per*k | scores per*k | counts per | bounds per]
        send = torch.empty((w, sect), dtype=torch.int32, device=dev)

        def by_slice(t, width, fill):
            """[n, width] section -> [w, per * width] (rows beyond n: `fill`)."""
            if per * w == n:
                return t.reshape(w, per * width)
            out = torch.full((w * per, width), fill, dtype=t.dtype, device=dev)
            out[:n] = t.reshape(n, width)
            return out.view(w, per * width)

        send[:, : per * k] = by_slice(pk.ids, k, -1)
        send[:, per * k : 2 * per * k] = by_slice(pk.scores, k, NEG_MAX).view(torch.int32)
        send[:, 2 * per * k : 2 * per * k + per] = by_slice(pk.counts, 1, 0)
        send[:, 2 * per * k + per :] = by_slice(pk.bounds, 1, float("-inf")).view(torch.int32)
        recv = torch.empty((w * sect,), dtype=torch.int32, device=dev)
        self.dist.all_to_all_single(recv, send.view(-1), group=self.exchange_group)
        # ---- merge my slice; [ids | scores | counts | failed rows | n failed] goes round
        out_len = per * (2 * k + 2) + 2
        mine = torch.zeros((out_len,), dtype=torch.int32, device=dev)
        m_ids = mine[: per * k].view(per, k)
        m_sc = mine[per * k : 2 * per * k].view(torch.float32).view(per, k)
        m_cnt = mine[2 * per * k : 2 * per * k + per]
        m_fail = mine[2 * per * k + per : 2 * per * k + 2 * per]
        m_nfail = mine[2 * per * k + 2 * per : 2 * per * k + 2 * per + 1]
        if self.host_provider:
            ids, sc, cnt, _ = Packed.views(torch, recv, w, per, k)
            o = merge_padded_numpy(ids.numpy(), sc.numpy(), cnt.numpy(), k)
            m_ids[:], m_sc[:], m_cnt[:] = (torch.from_numpy(x) for x in o)
        else:
            self.local.merge_into(recv, w, per, k, shared, m_ids, m_sc, m_cnt, m_fail, m_nfail)
        allm = torch.empty((w, out_len), dtype=torch.int32, device=dev)
        self.dist.all_gather_into_tensor(allm.view(-1), mine, group=self.exchange_group)
        o_ids = allm[:, : per * k].reshape(w * per, k)[:n]
        o_sc = allm[:, per * k : 2 * per * k].view(torch.float32).reshape(w * per, k)[:n]
        o_cnt = allm[:, 2 * per * k : 2 * per * k + per].reshape(w * per)[:n]
        n_fail = 0
        if shared and not self.host_provider:
            counts = allm[:, 2 * per * k + 2 * per].cpu().tolist()  # (the one host read-back of the exchange)
            n_fail = int(sum(counts))
            self.last_stats["n_uncertified_rows"] = n_fail
            if n_fail:
                fails = allm[:, 2 * per * k + per : 2 * per * k + 2 * per]
                rows = torch.cat([fails[j, :c].long() + j * per for j, c in enumerate(counts) if c]).sort().values
                pk2 = rerank(rows)  # local, self-certified lists of those rows
                g2 = torch.empty((w * pk2.stride,), dtype=torch.int32, device=dev)
                self.dist.all_gather_into_tensor(g2, pk2.buf, group=self.exchange_group)
                r_ids, r_sc, r_cnt, _, _ = self.local.merge(g2, w, n_fail, k, certified=False)
                o_ids, o_sc, o_cnt = o_ids.contiguous(), o_sc.contiguous(), o_cnt.contiguous()
                o_ids[rows], o_sc[rows], o_cnt[rows] = r_ids, r_sc, r_cnt
        return o_ids, o_sc, o_cnt

    def _collect(self, o_ids: tp.Any, o_sc: tp.Any, o_cnt: tp.Any, row_bounds: tp.Sequence[tp.Tuple[int, int]], k: int):
        """Hand every rank the rows of the other subject groups (slices padded to the longest one), one all-gather."""
        torch, u = self.torch, self.subject_groups
        if u == 1:
            return o_ids, o_sc, o_cnt
        per = max(b - a for a, b in row_bounds)
        n = o_ids.shape[0]
        pk = Packed(torch, per, k, o_ids.device)
        pk.ids.fill_(-1)
        pk.scores.fill_(NEG_MAX)
        pk.counts.zero_()
        pk.bounds.fill_(float("-inf"))
        pk.ids[:n], pk.scores[:n], pk.counts[:n] = o_ids, o_sc, o_cnt
        g = torch.empty((u * pk.stride,), dtype=torch.int32, device=o_ids.device)
        self.dist.all_gather_into_tensor(g, pk.buf, group=self.collect_group)
        ids, sc, cnt, _ = Packed.views(torch, g, u, per, k)
        keep = [slice(0, b - a) for a, b in row_bounds]
        return (torch.cat([ids[i, s] for i, s in enumerate(keep)]), torch.cat([sc[i, s] for i, s in enumerate(keep)]),
                torch.cat([cnt[i, s] for i, s in enumerate(keep)]))

    def _prepare(self, n_all: int, k: tp.Optional[int], sorted_object_whitelist: tp.Optional[np.ndarray]):
        wl_local = None
        n_pos_total = self.n_objects
        if sorted_object_whitelist is not None:
            wl = np.asarray(sorted_object_whitelist, dtype=np.int64).reshape(-1)
            check_whitelist(wl, self.n_objects)
            wl_local = np.ascontiguousarray(split_whitelist(wl, self.lo, self.hi))
            n_pos_total = len(wl)
        if k is None:
            k = n_pos_total
        k = min(int(k), n_pos_total)
        if k <= 0:
            raise ValueError("`k` must be positive")
        row_bounds = shard_bounds(n_all, self.subject_groups)
        return k, wl_local, row_bounds

    def rank_padded(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None):
        """Host inputs (the `Ranker` protocol): `(subject_ids, ids [n,k], scores [n,k], counts [n])` tensors."""
        subject_ids = np.asarray(subject_ids, dtype=np.int64).reshape(-1)
        if filter_pairs_csr is not None and filter_pairs_csr.shape[0] != len(subject_ids):
            raise ValueError("Number of rows in `filter_pairs_csr` must be equal to `len(sublect_ids)`")
        if len(subject_ids) and (subject_ids.min() < 0 or subject_ids.max() >= self.n_subjects):
            raise IndexError("subject id out of range")
        k, wl_local, row_bounds = self._prepare(len(subject_ids), k, sorted_object_whitelist)
        indptr = indices = None
        if filter_pairs_csr is not None:
            csr = filter_pairs_csr if sparse.isspmatrix_csr(filter_pairs_csr) else sparse.csr_matrix(filter_pairs_csr)
            if not csr.has_sorted_indices:
                csr = csr.sorted_indices()
            indptr, indices = csr.indptr, csr.indices
        # my subject group's slice of the batch (contiguous rows; the CSR filter is sliced by its row pointer)
        r0, r1 = row_bounds[self.group_idx]
        my_ids = np.ascontiguousarray(subject_ids[r0:r1])
        my_indptr = my_indices = None
        if indptr is not None:
            my_indptr = np.ascontiguousarray(np.asarray(indptr[r0 : r1 + 1], dtype=np.int64) - int(indptr[r0]))
            my_indices = np.ascontiguousarray(indices[int(indptr[r0]) : int(indptr[r1])], dtype=np.int32)
        n = len(my_ids)
        torch = self.torch
        if self.host_provider:
            ids, sc, cnt = self.local.local_topk(my_ids, k, my_indptr, my_indices, wl_local)
            pk = Packed(torch, n, k, ids.device)
            pk.ids.fill_(-1)
            pk.scores.fill_(NEG_MAX)
            pk.bounds.fill_(float("-inf"))
            pk.ids[:, : ids.shape[1]], pk.scores[:, : sc.shape[1]], pk.counts[:] = ids, sc, cnt
            o = self._exchange(pk, n, k, False, None)
            return (subject_ids,) + tuple(self._collect(*o, row_bounds, k))

        def host_inputs(ids_np, indptr_np, indices_np):
            kw = dict(subject_ids=ids_np.ctypes.data)
            if indptr_np is not None:
                kw.update(indptr=indptr_np.ctypes.data, indices=indices_np.ctypes.data)
            if wl_local is not None:
                kw.update(whitelist=wl_local.ctypes.data, n_whitelist=len(wl_local))
            return kw

        shared = self._shared_ok(n, k)
        pk = Packed(torch, n, k, self.local.device)
        self.last_stats = {}
        if n:
            self.last_stats = dict(self.local.local_topk(n, k, pk, shared_epoch=self._next_epoch() if shared else 0,
                                                         **host_inputs(my_ids, my_indptr, my_indices)))

        def rerank(rows):
            rows_np = rows.cpu().numpy()
            ids2 = np.ascontiguousarray(my_ids[rows_np])
            ip2 = ix2 = None
            if my_indptr is not None:
                sub = sparse.csr_matrix((np.ones(len(my_indices), np.int8), my_indices, my_indptr), shape=(n, self.n_objects))[rows_np]
                ip2, ix2 = np.ascontiguousarray(sub.indptr, dtype=np.int64), np.ascontiguousarray(sub.indices, dtype=np.int32)
            pk2 = Packed(torch, len(rows_np), k, self.local.device)
            self.local.local_topk(len(rows_np), k, pk2, **host_inputs(ids2, ip2, ix2))
            return pk2

        o = self._exchange(pk, n, k, shared, rerank)
        return (subject_ids,) + tuple(self._collect(*o, row_bounds, k))

    def rank_device(self, subjects: tp.Any, k: int, indptr: tp.Any = None, indices: tp.Any = None):
        """Subject MATRIX in, device tensors out: `subjects` [n, d] fp32 = THIS subject group's rows of the batch in batch order
        (all rows with pure item sharding), `indptr` int64 [n+1] / `indices` int32 = their filter rows -- either CUDA tensors
        (resident inputs, no copies) or host arrays / pinned CPU tensors (staged by the engine's chunk pipeline: the copies
        overlap the ranking).  Returns `(ids [n_all,k], scores, counts)` CUDA tensors of the whole batch.  DOT / COSINE scores
        as the engine defines them (COSINE: not yet divided by the subject norms)."""
        from . import _lib

        torch = self.torch
        on_device = bool(getattr(subjects, "is_cuda", False))
        if not on_device:  # host: numpy views (pinned tensors stay pinned)
            to_np = lambda t, dt: None if t is None else np.ascontiguousarray(t.numpy() if hasattr(t, "numpy") else t, dtype=dt)
            subjects, indptr, indices = to_np(subjects, np.float32), to_np(indptr, np.int64), to_np(indices, np.int32)
        ptr = (lambda t: t.data_ptr()) if on_device else (lambda t: t.ctypes.data)
        n = int(subjects.shape[0])
        if self.subject_groups > 1:  # the groups' slice lengths
            t = torch.tensor([n], dtype=torch.int64, device=self.local.device)
            sizes = [torch.zeros_like(t) for _ in range(self.subject_groups)]
            self.dist.all_gather(sizes, t, group=self.collect_group)
            starts = np.concatenate([[0], np.cumsum([int(x.item()) for x in sizes])])
            row_bounds = [(int(starts[i]), int(starts[i + 1])) for i in range(self.subject_groups)]
        else:
            row_bounds = [(0, n)]
        k = min(int(k), self.n_objects)

        def inputs(sub_t, ip_t, ix_t):
            kw = dict(subjects=ptr(sub_t), flags=_lib.Q_INPUTS_ON_DEVICE if on_device else 0)
            if ip_t is not None:
                kw.update(indptr=ptr(ip_t), indices=ptr(ix_t))
            return kw

        shared = self._shared_ok(n, k)
        pk = Packed(torch, n, k, self.local.device)
        self.last_stats = dict(self.local.local_topk(n, k, pk, shared_epoch=self._next_epoch() if shared else 0,
                                                     **inputs(subjects, indptr, indices)))

        def rerank(rows):
            if on_device:
                sub2 = subjects[rows].contiguous()
                ip2 = ix2 = None
                if indptr is not None:
                    a, b = indptr[rows], indptr[rows + 1]
                    lens = b - a
                    ip2 = torch.zeros((len(rows) + 1,), dtype=torch.int64, device=indptr.device)
                    ip2[1:] = torch.cumsum(lens, 0)
                    pos = (torch.arange(int(ip2[-1].item()), device=indptr.device) - torch.repeat_interleave(ip2[:-1], lens)
                           + torch.repeat_interleave(a, lens))
                    ix2 = indices[pos].contiguous()
            else:
                rows_np = rows.cpu().numpy()
                sub2 = np.ascontiguousarray(subjects[rows_np])
                ip2 = ix2 = None
                if indptr is not None:
                    lens = indptr[rows_np + 1] - indptr[rows_np]
                    ip2 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
                    ix2 = np.ascontiguousarray(np.concatenate([indices[indptr[r] : indptr[r + 1]] for r in rows_np]) if len(rows_np) else
                                               np.empty(0, np.int32), dtype=np.int32)
            pk2 = Packed(torch, len(rows), k, self.local.device)
            self._keep = (sub2, ip2, ix2)
            self.local.local_topk(len(rows), k, pk2, **inputs(sub2, ip2, ix2))
            return pk2

        o = self._exchange(pk, n, k, shared, rerank)
        return self._collect(*o, row_bounds, k)

    def _shared_ok(self, n: int, k: int) -> bool:
        return (not self.host_provider and getattr(self.local, "sharing", False) and self.item_shards > 1 and k <= 24
                and 0 < n <= self.local.max_shared_rows)

    def _next_epoch(self) -> int:
        self.epoch += 1
        return self.epoch

    def rank(self, subject_ids, k=None, filter_pairs_csr=None, sorted_object_whitelist=None):
        subject_ids, ids, sc, cnt = self.rank_padded(subject_ids, k, filter_pairs_csr, sorted_object_whitelist)
        ids, sc, cnt = strip_sentinel_tail(*(t.cpu().numpy() if hasattr(t, "cpu") else np.array(t) for t in (ids, sc, cnt)))
        all_subjects, all_ids, all_scores = flatten_padded(subject_ids, ids, sc, cnt)
        if self.distance == Distance.COSINE:
            all_scores = all_scores / self.subjects_norms[all_subjects]
        elif self.distance == Distance.EUCLIDEAN:
            all_scores = np.sqrt(np.maximum(self.subjects_dots[all_subjects] - all_scores, 0)).astype(np.float32)
        return all_subjects, all_ids, all_scores

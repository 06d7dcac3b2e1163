"""Candidate sets (engine path 5) against the obvious alternatives, on one GPU, in one process.

    python scripts/candidate_sets_ab.py [--reps 5] [--out results.json]

Workloads:
  1. re-rank: U = 65 536 users, N = 1M items, d = 128 fp32, DOT, 1 000 random candidates per row, 100 of them viewed
     (filtered), k = 100;
  2. the config-5 catalogue: N = 5M, d = 256, bf16 kept at 16 bits, COSINE, U = 65 536, 500 candidates, k = 20;
  3. long lists: U = 1 024 rows of 100 000 candidates over workload 1's catalogue, k = None (the longest list).
Arms, alternated within every repeat: the engine (`Engine.topk_candidates`); torch on the same GPU (gather the candidate
rows, batched matmul in fp32, mask the filter, `topk`); for workload 1 also the engine's full-catalogue `topk` with the
lists as a complement filter, at U = 64 (a complement row is ~1M entries).
Reported per arm: ms_total / ms_main / ms_select (engine statistics; wall ms for torch, inputs already on the GPU), the spread
over repeats, the achieved gather bandwidth sum|C_r| * d * bytes / ms_main against H100 SXM's 3.35 TB/s data-sheet figure,
whether two engine runs return bit-identical ids, and 8 sampled rows per workload against the rounding-interval oracle.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # pylint: disable=broad-except
        power = "unknown"
    return name, power


def lists(rng, n_rows, n_obj, per_row):
    """Sorted unique random ids, `per_row` per row: (indptr, indices)."""
    draw = np.sort(rng.integers(0, n_obj, (n_rows, per_row + per_row // 8 + 16)), axis=1)
    dup = np.zeros_like(draw, dtype=bool)
    dup[:, 1:] = draw[:, 1:] == draw[:, :-1]
    order = np.argsort(dup, axis=1, kind="stable")  # unique values first, in ascending order
    ids = np.take_along_axis(draw, order, axis=1)[:, :per_row]
    assert not np.take_along_axis(dup, order, axis=1)[:, :per_row].any()
    return np.arange(n_rows + 1, dtype=np.int64) * per_row, ids.astype(np.int32).reshape(-1)


def viewed(rng, cand_indptr, cand_indices, per_row):
    n = len(cand_indptr) - 1
    width = int(cand_indptr[1] - cand_indptr[0])
    pick = np.sort(rng.random((n, width)).argsort(axis=1)[:, :per_row], axis=1)
    rows = cand_indices.reshape(n, width)
    return np.arange(n + 1, dtype=np.int64) * per_row, np.take_along_axis(rows, pick, axis=1).reshape(-1).astype(np.int32)


def torch_arm(sub_t, obj_t, norms_t, cand_indptr, cand_indices, f_indptr, f_indices, k, batch_cands=1 << 27):
    """gather + bmm in fp32 + topk, in row batches of at most `batch_cands` gathered elements."""
    import torch

    n = len(cand_indptr) - 1
    width = int(cand_indptr[1] - cand_indptr[0])
    ci = torch.from_numpy(cand_indices.reshape(n, width).astype(np.int64)).cuda()
    fmask = None
    if f_indptr is not None:
        fw = int(f_indptr[1] - f_indptr[0])
        fi = torch.from_numpy(f_indices.reshape(n, fw).astype(np.int64)).cuda()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    d = obj_t.shape[1]
    rows = max(1, batch_cands // (width * d))
    out_ids, out_sc = [], []
    for r0 in range(0, n, rows):
        r1 = min(n, r0 + rows)
        idx = ci[r0:r1]
        g = obj_t[idx].float()  # [b, width, d]
        s = torch.bmm(g, sub_t[r0:r1].unsqueeze(2)).squeeze(2)
        if norms_t is not None:
            s = s / norms_t[idx]
        if f_indptr is not None:
            fmask = (idx.unsqueeze(2) == fi[r0:r1].unsqueeze(1)).any(dim=2)
            s = s.masked_fill(fmask, float("-inf"))
        v, p = torch.topk(s, min(k, width), dim=1)
        out_ids.append(torch.gather(idx, 1, p))
        out_sc.append(v)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, torch.cat(out_ids).cpu().numpy(), torch.cat(out_sc).cpu().numpy()


def sampled_check(got, subjects, objects, k, cand_indptr, cand_indices, f_indptr, f_indices, cosine, rows):
    """Rows `rows` against the interval oracle, over the local catalogue of their candidates (ids remapped)."""
    from tests.score_interval import check_topk

    ids, sc, cnt = got
    cand = [cand_indices[cand_indptr[r] : cand_indptr[r + 1]] for r in rows]
    local = np.unique(np.concatenate(cand))
    if hasattr(objects, "detach"):  # a CPU torch tensor (bf16 has no numpy type)
        import torch

        obj = objects[torch.from_numpy(local)]
    else:
        obj = np.asarray(objects[local])
    lid = np.where(ids[rows] >= 0, np.searchsorted(local, np.maximum(ids[rows], 0)), -1).astype(np.int32)
    banned = []
    for i, r in enumerate(rows):
        b = np.setdiff1d(np.arange(len(local)), np.searchsorted(local, cand[i]))
        if f_indptr is not None:
            f = f_indices[f_indptr[r] : f_indptr[r + 1]]
            f = f[np.isin(f, local)]
            b = np.union1d(b, np.searchsorted(local, f))
        banned.append(b)
    ip = np.zeros(len(rows) + 1, np.int64)
    np.cumsum([len(b) for b in banned], out=ip[1:])
    k_loc = min(k, len(local))
    got_loc = (lid[:, :k_loc], sc[rows][:, :k_loc], np.minimum(cnt[rows], k_loc))
    assert (cnt[rows] <= k_loc).all()
    rep = check_topk(got_loc, subjects[rows], obj, k_loc, cosine=cosine, filter_csr=(ip, np.concatenate(banned)), name="sampled",
                     verbose=False)
    amb = rep.n_ambiguous
    return {"rows": len(rows), "checked": int(rep.n_checked), "ambiguous": int(amb() if callable(amb) else amb), "ok": True}


def run_workload(name, eng, sub_np, objects_host, sub_t, obj_t, norms_t, cand, filt, k, reps, cosine, complement_rows=0):
    import torch  # noqa: F401

    from scipy import sparse

    cand_indptr, cand_indices = cand
    f_indptr, f_indices = filt if filt is not None else (None, None)
    n_cand = int(cand_indptr[-1])
    elem = 2 if obj_t.dtype.itemsize == 2 else 4
    res = {"workload": name, "rows": len(cand_indptr) - 1, "candidates": n_cand, "k": k, "engine": [], "torch": [], "complement": []}
    first = None
    identical = True
    for rep in range(reps):
        t0 = time.perf_counter()
        got = eng.topk_candidates(k, cand_indptr, cand_indices, subjects=sub_np, indptr=f_indptr, indices=f_indices)
        wall = (time.perf_counter() - t0) * 1e3
        st = dict(eng.last_stats, wall_ms=wall)
        if first is None:
            first = got
        else:
            identical &= bool(np.array_equal(first[0], got[0]))
        res["engine"].append({m: st[m] for m in ("ms_total", "ms_main", "ms_select", "n_chunks", "n_launches", "wall_ms")})
        if rep < 3:  # the torch arm is the slow one: three repeats
            ms, _, _ = torch_arm(sub_t, obj_t, norms_t, cand_indptr, cand_indices, f_indptr, f_indices, k)
            res["torch"].append({"ms_total": ms})
        if complement_rows and rep < 3:
            n = complement_rows
            n_obj = eng.n_objects
            comp = []
            for r in range(n):
                banned = np.setdiff1d(np.arange(n_obj, dtype=np.int32), cand_indices[cand_indptr[r] : cand_indptr[r + 1]])
                if f_indptr is not None:
                    banned = np.union1d(banned, f_indices[f_indptr[r] : f_indptr[r + 1]])
                comp.append(banned.astype(np.int32))
            ip = np.zeros(n + 1, np.int64)
            np.cumsum([len(c) for c in comp], out=ip[1:])
            t0 = time.perf_counter()
            full = eng.topk(k, subjects=sub_np[:n], indptr=ip, indices=np.concatenate(comp))
            wall = (time.perf_counter() - t0) * 1e3
            st2 = dict(eng.last_stats)
            part = eng.topk_candidates(k, cand_indptr[: n + 1], cand_indices[: cand_indptr[n]], subjects=sub_np[:n],
                                       indptr=None if f_indptr is None else f_indptr[: n + 1],
                                       indices=None if f_indptr is None else f_indices[: f_indptr[n]])
            st3 = dict(eng.last_stats)
            res["complement"].append({"rows": n, "ms_total": st2["ms_total"], "wall_ms": wall, "path": st2["path"],
                                      "engine_same_rows_ms_total": st3["ms_total"],
                                      "same_ids": bool(np.array_equal(full[0], part[0])), "same_scores": bool(np.array_equal(full[1], part[1]))})
    ms_main = np.array([e["ms_main"] for e in res["engine"]])
    res["engine_ids_bit_identical"] = identical
    res["gather_TBps_median"] = n_cand * sub_np.shape[1] * elem / (np.median(ms_main) * 1e-3) / 1e12
    res["gather_fraction_of_3.35TBps"] = res["gather_TBps_median"] / HBM_TBS
    for arm in ("engine", "torch"):
        tot = np.array([e["ms_total"] for e in res[arm]])
        res[f"{arm}_ms_total_min_median_max"] = [float(tot.min()), float(np.median(tot)), float(tot.max())]
    for m in ("ms_main", "ms_select"):
        v = np.array([e[m] for e in res["engine"]])
        res[f"engine_{m}_min_median_max"] = [float(v.min()), float(np.median(v)), float(v.max())]
    rows = np.random.default_rng(0).choice(len(cand_indptr) - 1, 8, replace=False)
    res["sampled_oracle"] = sampled_check(first, sub_np, objects_host, k, cand_indptr, cand_indices, f_indptr, f_indices, cosine, rows)
    print(json.dumps({k_: v for k_, v in res.items() if k_ not in ("engine", "torch")}), flush=True)
    return res


def main() -> None:
    import torch

    from rectools_b200 import _lib
    from rectools_b200.ranker import Engine

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--only", default="123")
    args = ap.parse_args()
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power}), flush=True)
    out = {"card": name, "power_limit": power, "workloads": []}
    rng = np.random.default_rng(0)

    if "1" in args.only or "3" in args.only:
        n_obj, d = 1_000_000, 128
        objects = rng.standard_normal((n_obj, d), dtype=np.float32)
        eng = Engine(objects, cosine=False)
        obj_t = torch.from_numpy(objects).cuda()
        if "1" in args.only:
            U = 65_536
            sub = rng.standard_normal((U, d), dtype=np.float32)
            cand = lists(rng, U, n_obj, 1000)
            filt = viewed(rng, *cand, 100)
            out["workloads"].append(run_workload("1 re-rank", eng, sub, objects, torch.from_numpy(sub).cuda(), obj_t, None, cand, filt, 100,
                                                 args.reps, False, complement_rows=64))
        if "3" in args.only:
            U = 1024
            sub = rng.standard_normal((U, d), dtype=np.float32)
            cand = lists(rng, U, n_obj, 100_000)
            out["workloads"].append(run_workload("3 long lists", eng, sub, objects, torch.from_numpy(sub).cuda(), obj_t, None, cand, None,
                                                 100_000, args.reps, False))
        eng.close()
        del obj_t
        torch.cuda.empty_cache()

    if "2" in args.only:
        n_obj, d, U = 5_000_000, 256, 65_536
        g = torch.Generator(device="cuda").manual_seed(5)
        obj_t = torch.randn((n_obj, d), generator=g, device="cuda", dtype=torch.float32).to(torch.bfloat16)
        eng = Engine(None, cosine=True, objects_device_ptr=obj_t.data_ptr(), shape=(n_obj, d), objects_dtype=_lib.DT_BF16, keep_16bit=True)
        norms_t = torch.sqrt((obj_t.float().double() ** 2).sum(dim=1)).float()
        objects_host = obj_t.cpu()
        sub = rng.standard_normal((U, d), dtype=np.float32)
        cand = lists(rng, U, n_obj, 500)
        out["workloads"].append(run_workload("2 c5 bf16 cosine", eng, sub, objects_host, torch.from_numpy(sub).cuda(), obj_t, norms_t, cand,
                                             None, 20, args.reps, True))
        eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

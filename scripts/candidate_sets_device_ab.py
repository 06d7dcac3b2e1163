"""Candidate sets (engine path 5) from device memory against the host route and torch, on one GPU, in one process.

    python scripts/candidate_sets_device_ab.py [--reps 5] [--out results.json] [--only 123]

The three workloads of scripts/candidate_sets_ab.py (1: 65 536 rows x 1 000 candidates, 100 of them filtered, k = 100 over
1M x 128 fp32 DOT; 2: 65 536 x 500, k = 20 over 5M x 256 bf16 COSINE kept at 16 bits; 3: 1 024 x 100 000, k = None over
workload 1's catalogue).  Arms, alternated within every repeat:
  host    `Engine.topk_candidates`: host lists, subjects and outputs;
  device  `Engine.topk_candidates_device`: the same lists, subjects and filter as CUDA tensors, device outputs;
  raw     the same with each row as a first stage hands it over: its ids shuffled, m/16 of them repeated and m/16 -1
          holes added (the same set, so the same answer);
  torch   gather + bmm in fp32 + topk on the GPU, inputs already there (wall ms).
Reported per workload: ms_total / ms_main / ms_select of the engine arms (min, median, max over repeats) and the torch
arm's ms, the device route's wall ms, the preparation cost (ms_main of `device` / `raw` - host ms_main, medians), and
whether every engine arm returns bit-identical ids, score bits and counts.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from candidate_sets_ab import card, lists, torch_arm, viewed  # noqa: E402


def spread(values):
    v = np.asarray(values, dtype=np.float64)
    return [float(v.min()), float(np.median(v)), float(v.max())]


def raw_lists(rng, cand):
    """Fixed-width lists (indptr = m * r) as a first stage returns them: each row shuffled, with m/16 of its ids repeated
    and m/16 -1 holes, the same set of valid ids."""
    cand_indptr, cand_indices = cand
    n = len(cand_indptr) - 1
    m = int(cand_indptr[1] - cand_indptr[0])
    rows = cand_indices.reshape(n, m)
    e = max(1, m // 16)
    rep = np.take_along_axis(rows, rng.integers(0, m, (n, e)), axis=1)
    wide = np.concatenate([rows, rep, np.full((n, e), -1, np.int32)], axis=1)
    wide = np.take_along_axis(wide, rng.random(wide.shape, dtype=np.float32).argsort(axis=1), axis=1)
    return np.arange(n + 1, dtype=np.int64) * wide.shape[1], np.ascontiguousarray(wide, dtype=np.int32).reshape(-1)


def run_workload(name, eng, sub_np, sub_t, obj_t, norms_t, cand, filt, k, reps):
    import torch

    cand_indptr, cand_indices = cand
    f_indptr, f_indices = filt if filt is not None else (None, None)
    d_cand = (torch.from_numpy(cand_indptr).cuda(), torch.from_numpy(cand_indices).cuda())
    d_raw = tuple(torch.from_numpy(a).cuda() for a in raw_lists(np.random.default_rng(7), cand))
    d_filt = (None, None) if filt is None else (torch.from_numpy(f_indptr).cuda(), torch.from_numpy(f_indices).cuda())
    res = {"workload": name, "rows": len(cand_indptr) - 1, "candidates": int(cand_indptr[-1]), "k": k}
    arms = {"host": [], "device": [], "raw": [], "torch": []}
    same = True
    for rep in range(reps):
        host = eng.topk_candidates(k, cand_indptr, cand_indices, subjects=sub_np, indptr=f_indptr, indices=f_indices)
        arms["host"].append(dict(eng.last_stats))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dev = eng.topk_candidates_device(k, *d_cand, subjects=sub_t, indptr=d_filt[0], indices=d_filt[1])
        torch.cuda.synchronize()
        arms["device"].append(dict(eng.last_stats, wall_ms=(time.perf_counter() - t0) * 1e3))
        raw = eng.topk_candidates_device(k, *d_raw, subjects=sub_t, indptr=d_filt[0], indices=d_filt[1])
        arms["raw"].append(dict(eng.last_stats))
        for got in (dev, raw):
            got = tuple(t.cpu().numpy() for t in got)
            same &= bool(np.array_equal(host[0], got[0]) and np.array_equal(host[1].view(np.int32), got[1].view(np.int32))
                         and np.array_equal(host[2], got[2]))
        del host, dev, raw
        ms, _, _ = torch_arm(sub_t, obj_t, norms_t, cand_indptr, cand_indices, f_indptr, f_indices, k)
        arms["torch"].append({"ms_total": ms})
    for arm in ("host", "device", "raw"):
        for m in ("ms_total", "ms_main", "ms_select"):
            res[f"{arm}_{m}_min_median_max"] = spread([s[m] for s in arms[arm]])
    res["device_wall_ms_min_median_max"] = spread([s["wall_ms"] for s in arms["device"]])
    res["torch_ms_min_median_max"] = spread([s["ms_total"] for s in arms["torch"]])
    res["preparation_ms_median"] = res["device_ms_main_min_median_max"][1] - res["host_ms_main_min_median_max"][1]
    res["raw_preparation_ms_median"] = res["raw_ms_main_min_median_max"][1] - res["host_ms_main_min_median_max"][1]
    res["routes_bit_identical"] = same
    print(json.dumps(res), flush=True)
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
            out["workloads"].append(run_workload("1 re-rank", eng, sub, torch.from_numpy(sub).cuda(), obj_t, None, cand, filt, 100, args.reps))
        if "3" in args.only:
            U = 1024
            sub = rng.standard_normal((U, d), dtype=np.float32)
            cand = lists(rng, U, n_obj, 100_000)
            out["workloads"].append(run_workload("3 long lists", eng, sub, torch.from_numpy(sub).cuda(), obj_t, None, cand, None, 100_000,
                                                 args.reps))
        eng.close()
        del obj_t
        torch.cuda.empty_cache()

    if "2" in args.only:
        n_obj, d, U = 5_000_000, 256, 65_536
        g = torch.Generator(device="cuda").manual_seed(5)
        obj_t = torch.randn((n_obj, d), generator=g, device="cuda", dtype=torch.float32).to(torch.bfloat16)
        eng = Engine(None, cosine=True, objects_device_ptr=obj_t.data_ptr(), shape=(n_obj, d), objects_dtype=_lib.DT_BF16, keep_16bit=True)
        norms_t = torch.sqrt((obj_t.float().double() ** 2).sum(dim=1)).float()
        sub = rng.standard_normal((U, d), dtype=np.float32)
        cand = lists(rng, U, n_obj, 500)
        out["workloads"].append(run_workload("2 c5 bf16 cosine", eng, sub, torch.from_numpy(sub).cuda(), obj_t, norms_t, cand, None, 20,
                                             args.reps))
        eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

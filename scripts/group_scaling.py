"""Config-2 users/s through `B200Ranker.rank` on one engine and on engine groups (`device=[...]`).

    python scripts/group_scaling.py [--users 1000000] [--items 1000000] [--dim 128] [--k 10] [--steps 5]
                                    [--groups 0 0,0 0,1 0,1,2,3 0,1,2,3,4,5,6,7] [--out DIR]

Factors as bench.py's config 2 (ImplicitALS-shaped, d = 128, Distance.DOT, K = 10), resident subjects, a viewed-items
filter of 100 items per user.  Groups naming devices the host does not have are skipped.  Per group, after one warm-up
call: the median wall-clock seconds of `rank()` over --steps calls, users/s, each member's CUDA-event ms (`ms_total`
summed over its slices), kernel ms and fallback rows, and the share of the wall-clock time outside the members' kernels: 1 - max over members
of the kernel ms (fused kernel + selection) / wall-clock ms -- slicing, staging, copies back, flattening and the host work
of `rank()`.  On a one-GPU host only [0] against [0, 0] (and more members on device 0) can run: that is the group's
overhead, not scaling.  Prints one JSON line per group (with the card's name and power limit); with --out DIR also writes
them to DIR/group_scaling.jsonl."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rectools_b200 import B200Ranker  # noqa: E402


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().replace("\n", "; ")
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def viewed_csr(n_users: int, n_items: int, per_user: int, seed: int = 2):
    from scipy import sparse

    cols = np.sort(np.random.default_rng(seed).integers(0, n_items, size=(n_users, per_user), dtype=np.int32), axis=1)
    indptr = np.arange(n_users + 1, dtype=np.int64) * per_user
    return sparse.csr_matrix((np.ones(cols.size, np.float32), cols.reshape(-1), indptr), shape=(n_users, n_items))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--viewed", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--groups", nargs="+", default=["0", "0,0", "0,1", "0,1,2,3", "0,1,2,3,4,5,6,7"])
    ap.add_argument("--out", default="", help="directory for group_scaling.jsonl (default: print only)")
    a = ap.parse_args()
    import torch

    n_gpus = torch.cuda.device_count()
    if n_gpus == 0:
        raise SystemExit("no CUDA device: nothing to measure")
    card = gpu_info()
    rng = np.random.default_rng(0)
    users = (rng.standard_normal((a.users, a.dim), dtype=np.float32) / np.sqrt(a.dim)).astype(np.float32)
    items = (rng.standard_normal((a.items, a.dim), dtype=np.float32) / np.sqrt(a.dim)).astype(np.float32)
    csr = viewed_csr(a.users, a.items, a.viewed)
    sids = np.arange(a.users)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    reference = None
    with open(os.path.join(a.out, "group_scaling.jsonl") if a.out else os.devnull, "w") as fh:
        for spec in a.groups:
            devices = [int(x) for x in spec.split(",")]
            if max(devices) >= n_gpus:
                print(json.dumps({"group": devices, "skipped": f"the host has {n_gpus} GPU(s)"}), flush=True)
                continue
            device = devices[0] if len(devices) == 1 and spec == "0" else devices
            ranker = B200Ranker("dot", users, items, device=device)
            result = ranker.rank(sids, a.k, csr)  # warm-up (and the result every group must reproduce)
            if reference is None:
                reference = result
            same = all(np.array_equal(x, y) for x, y in zip(result, reference))
            times, members = [], []
            for _ in range(a.steps):
                t0 = time.perf_counter()
                ranker.rank(sids, a.k, csr)
                times.append(time.perf_counter() - t0)
                members.append(getattr(ranker.engine, "last_member_stats", None) or [ranker.engine.last_stats])
            i_med = int(np.argsort(times)[len(times) // 2])
            sec, per = times[i_med], members[i_med]
            kernel_ms = max(m["ms_main"] + m["ms_select"] for m in per)
            line = {
                "group": devices if device != 0 else 0, "users": a.users, "items": a.items, "dim": a.dim, "k": a.k,
                "seconds": sec, "users_per_s": a.users / sec, "equal_to_first": bool(same),
                "member_ms_total": [round(m["ms_total"], 3) for m in per], "member_kernel_ms": [round(m["ms_main"] + m["ms_select"], 3) for m in per],
                "member_fallback_rows": [m["n_fallback_rows"] for m in per],
                "outside_kernels_share": 1.0 - kernel_ms / (1e3 * sec), "card": card,
            }
            print(json.dumps(line), flush=True)
            fh.write(json.dumps(line) + "\n")
            ranker.engine.close()
            del ranker


if __name__ == "__main__":
    main()

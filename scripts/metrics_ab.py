"""Time RecTools' stock `calc_metrics` against the installed one (path 10, `rectools_b200.metrics.calc_metrics`), DataFrames
in and the dict out, alternated in one run, and check that every value is `==`.

    python scripts/metrics_ab.py [--users 100000 1000000] [--repeats 5] [--warmup 1] [--out results.json]

Tables (tests/metrics_cases.large_tables): every user has a reco list of k = 10 distinct items and 1-10 test rows, each a
hit with probability 0.3, users interleaved in the interactions; seeded.  Two metric sets: the nine metrics Precision,
Recall, HitRate, F1Beta, Accuracy, MCC, MAP, NDCG and MRR at 10, and NDCG@10 alone.  Each call is timed on the host
clock around the whole call (the device call synchronises before it returns); medians over `--repeats` calls after
`--warmup` untimed ones.  Per layer (installed call, medians): host extraction (column checks, int64 copies, NDCG tables),
H2D, kernels, D2H (CUDA events), host assembly (confusion tables, per-user values, means).  Prints the GPU name and power
limit read in the same run."""
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


def gpu_info() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
        if out:
            return out
    except (OSError, subprocess.SubprocessError):
        pass
    import torch

    return torch.cuda.get_device_name(0) + ", power limit not read"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, nargs="+", default=[100_000, 1_000_000])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    a = ap.parse_args()

    from tests import metrics_cases  # before the reference goes on sys.path (it has a `tests` package too)
    from oracle import stage_reference

    stage_reference.add_to_path()
    from rectools.metrics import NDCG
    from rectools.metrics import calc_metrics as stock

    import rectools_b200

    info = gpu_info()
    print(f"GPU: {info}", flush=True)
    results = {"gpu": info, "runs": []}
    for n_users in a.users:
        reco, interactions = metrics_cases.large_tables(n_users, seed=1)
        catalog = np.arange(20_001)
        sets = {"nine@10": metrics_cases.nine_metrics(10), "ndcg@10": {"ndcg@10": NDCG(k=10)}}
        for set_name, metrics in sets.items():
            t_stock, t_dev, layers = [], [], []
            for r in range(a.warmup + a.repeats):
                t0 = time.perf_counter()
                expected = stock(metrics, reco, interactions, catalog=catalog)
                t1 = time.perf_counter()
                st: dict = {}
                actual = rectools_b200.calc_metrics(metrics, reco, interactions, catalog=catalog, stats=st)
                t2 = time.perf_counter()
                if list(actual) != list(expected) or any(actual[k] != expected[k] for k in expected):
                    raise SystemExit(f"values differ at {n_users} users, {set_name}: {actual} != {expected}")
                if r >= a.warmup:
                    t_stock.append(t1 - t0)
                    t_dev.append(t2 - t1)
                    layers.append({"extract": st["ms_extract"], "h2d": st["ms_h2d"], "kernels": st["ms_main"], "d2h": st["ms_d2h"],
                                   "assemble": st["ms_assemble"]})
            med = {k: float(np.median([x[k] for x in layers])) for k in layers[0]}
            run = {"users": n_users, "test_rows": len(interactions), "reco_rows": len(reco), "metrics": set_name,
                   "stock_s": float(np.median(t_stock)), "installed_s": float(np.median(t_dev)),
                   "stock_all_s": t_stock, "installed_all_s": t_dev, "layers_ms": med, "equal": True}
            run["speedup"] = run["stock_s"] / run["installed_s"]
            results["runs"].append(run)
            print(f"{n_users:>9} users, {len(interactions)} test rows, {len(reco)} reco rows, {set_name}: stock {run['stock_s']:.3f} s, "
                  f"installed {run['installed_s']:.4f} s ({run['speedup']:.1f}x); layers ms " +
                  ", ".join(f"{k} {v:.1f}" for k, v in med.items()) + "; every value ==", flush=True)
    print(json.dumps(results, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

"""Scored pairs (path 6): the per-user top-k of `Reranker.recommend` four ways, for DESIGN section 3.9.

    python scripts/rerank_pairs_ab.py [--repeats 5] [--out results.json] [--workloads 100000x100,...]

Arms, each a median with [min, max] over the repeats:
  reference  `Reranker.recommend` (one pandas sort per user), timed on a subsample of users and extrapolated linearly to
             all users -- labelled as such;
  numpy      the stable restatement: factorize, lexsort on (position, key, code), take;
  export     `b200_rank_topk_pairs` on host arrays: its `ms_total` (copies included);
  engine     `reranker_recommend` wall time, with `pd.factorize` and `take` (+ rank column) shown separately.
Workloads: float64 scores, k = 10 and 100, over 10^5 users x 100 pairs, 10^6 x 100, 10^4 x 10 000 and 1 x 10^7; rows are
shuffled.  Every engine repeat must return the same positions as the numpy restatement, or the script fails.
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

WORKLOADS = [(100_000, 100), (1_000_000, 100), (10_000, 10_000), (1, 10_000_000)]
REF_USERS = 2000  # users the reference is timed on (all of them when fewer)


def _frame(n_users, per_user, seed):
    import pandas as pd

    rng = np.random.default_rng(seed)
    n = n_users * per_user
    perm = rng.permutation(n)
    return pd.DataFrame({
        "user_id": (np.arange(n, dtype=np.int64) // per_user)[perm] * 7 + 100,
        "item_id": rng.integers(0, 1 << 20, n),
        "score": rng.random(n),
    })


def _stat(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="", help="also write the results to this JSON file")
    ap.add_argument("--small", action="store_true", help="tiny workloads (a rehearsal of the script)")
    ap.add_argument("--workloads", default="", help="a subset, e.g. 10000x10000,1x10000000 (default: all four)")
    args = ap.parse_args()

    import pandas as pd
    import torch

    from oracle import stage_reference
    from rectools_b200 import rank_pairs, reranker_recommend
    from tests.pairs_oracle import rank_pairs_np

    stage_reference.add_to_path()
    from rectools.models.ranking.candidate_ranking import Reranker

    props = torch.cuda.get_device_properties(0)
    header = {"gpu": props.name}
    try:
        import subprocess

        header["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # pylint: disable=broad-except
        header["power_limit"] = "unknown"
    print(json.dumps(header), flush=True)
    workloads = [(200, 50), (10, 3000)] if args.small else WORKLOADS
    if args.workloads:
        workloads = [tuple(int(v) for v in w.split("x")) for w in args.workloads.split(",")]
    results = []
    for n_users, per_user in workloads:
        df = _frame(n_users, per_user, seed=n_users)
        codes, uniques = pd.factorize(df["user_id"], sort=False)
        scores = df["score"].to_numpy()
        rank_pairs(codes, scores, 10, n_groups=len(uniques))  # warm-up of this shape
        for k in (10, 100):
            row = {"n_users": n_users, "per_user": per_user, "k": k}
            # reference on a user subsample
            sub_users = uniques[: min(REF_USERS, n_users)]
            sub = df[df["user_id"].isin(sub_users)] if n_users > 1 else df.iloc[: min(len(df), 200_000)]
            t = []
            for _ in range(min(args.repeats, 3) if len(sub) <= 1_000_000 else 1):
                t0 = time.perf_counter()
                Reranker.recommend(sub, k)
                t.append(time.perf_counter() - t0)
            scale = len(df) / max(len(sub), 1)
            row["reference_subsample_rows"] = int(len(sub))
            row["reference_s_extrapolated"] = {key: v * scale for key, v in _stat(t).items()}
            # numpy restatement
            t = []
            for _ in range(args.repeats if len(df) <= 20_000_000 else 1):  # one lexsort of 10^8 rows takes about a minute
                t0 = time.perf_counter()
                c, u = pd.factorize(df["user_id"], sort=False)
                exp_pos, exp_off = rank_pairs_np(c, df["score"].to_numpy(), k, len(u))
                df.take(exp_pos)
                t.append(time.perf_counter() - t0)
            row["numpy_s"] = _stat(t)
            # the export
            ms = []
            for _ in range(args.repeats):
                st = {}
                pos, off = rank_pairs(codes, scores, k, n_groups=len(uniques), stats=st)
                if not (np.array_equal(pos, exp_pos) and np.array_equal(off, exp_off)):
                    raise SystemExit(f"positions differ from the restatement at {row}")
                ms.append(st["ms_total"])
                row.setdefault("export_stats", st)
            row["export_ms_total"] = _stat(ms)
            # reranker_recommend, end to end
            wall, fac, take = [], [], []
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                reco = reranker_recommend(df, k)
                wall.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                pd.factorize(df["user_id"], sort=False)
                fac.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                r2 = df.take(exp_pos).reset_index(drop=True)
                r2["rank"] = np.arange(len(exp_pos)) - np.repeat(exp_off[:-1], np.diff(exp_off)) + 1
                take.append(time.perf_counter() - t0)
                if not np.array_equal(reco["item_id"].to_numpy(), df["item_id"].to_numpy()[exp_pos]):
                    raise SystemExit(f"reranker_recommend differs from the restatement at {row}")
            row["engine_wall_s"] = _stat(wall)
            row["factorize_s"] = _stat(fac)
            row["take_s"] = _stat(take)
            print(json.dumps(row), flush=True)
            results.append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"header": header, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()

"""Transformer id-embedding scorers (SASRec / BERT4Rec / HSTU): stock `TorchRanker` against the ranker that
`install(transformers=True)` binds, at SASRec-like shapes, for DESIGN section 9.3.

    python scripts/transformer_ab.py [--items 1000000] [--d 256] [--targets 100000] [--users 100000] [--k 20]
                                     [--viewed 50] [--repeats 3] [--small] [--out results.json]

Each arm is one ranker construction plus its `rank()` call, with exactly the arguments the two seams pass:
  i2i  `TransformerLightningModule._recommend_i2i` (lightning.py:440-449): the item embeddings (on the device) as both
       factors, COSINE, `--targets` target items, whitelist = every item but PAD (row 0), no filter.  The installed ranker
       takes the identity route (no copy of the catalogue);
  u2i  `DistanceSimilarityModule._recommend_u2i` (similarity.py:127-138): `--users` user embeddings on the host (the
       lightning module copies them there, lightning.py:397), the item embeddings on the device, `--viewed` viewed items
       per user as the filter, the same whitelist; DOT and COSINE.
Catalogues are fp32 and bf16.  Per arm: ms per call (median [min, max] of `--repeats`, CUDA events around the call after
a device synchronise; the call ends with its results on the host), peak device memory above the baseline
(`torch.cuda.max_memory_allocated`, reset before the call; the engine's own buffers are not torch allocations and are not
in it), and whether the outputs agree (same subjects; ids equal at every position, or the fraction that is; largest
score difference).  The card's name and power limit are printed first and stored with every row.  JSON is written only
with `--out`.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def _stat(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def _time(fn, repeats):
    import torch

    times, peaks, out = [], [], None
    for _ in range(repeats):
        out = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        out = fn()
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
        peaks.append(torch.cuda.max_memory_allocated() - base)
    return out, _stat(times), int(max(peaks))


def _agree(a, b):
    sa, ia, xa = (np.asarray(v) for v in a)
    sb, ib, xb = (np.asarray(v) for v in b)
    res = {"same_subjects": bool(sa.shape == sb.shape and (sa == sb).all())}
    if ia.shape == ib.shape:
        res["ids_equal_frac"] = float((ia == ib).mean()) if len(ia) else 1.0
        res["max_score_diff"] = float(np.abs(xa.astype(np.float64) - xb.astype(np.float64)).max()) if len(xa) else 0.0
    else:
        res["ids_equal_frac"] = None
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=256)
    ap.add_argument("--targets", type=int, default=100_000)
    ap.add_argument("--users", type=int, default=100_000)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--viewed", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--routes", default="i2i,u2i", help="comma-separated subset of i2i, u2i")
    ap.add_argument("--small", action="store_true", help="a tiny run of every arm (rehearsal)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.small:
        args.items, args.d, args.targets, args.users, args.repeats = 5000, 32, 300, 300, 1

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("transformer_ab.py measures on a CUDA device; none is available")
    from oracle import stage_reference

    stage_reference.add_to_path()
    from rectools.models.rank import TorchRanker

    from rectools_b200.integration import transformer_ranker

    props = torch.cuda.get_device_properties(0)
    header = {"gpu": props.name}
    try:
        header["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # pylint: disable=broad-except
        header["power_limit"] = "unknown"
    print(json.dumps(header), flush=True)

    installed = transformer_ranker()
    arms = {"stock": TorchRanker, "installed": installed}
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    items32 = torch.randn((args.items, args.d), generator=g, device=dev) / np.sqrt(args.d)
    items32[0] = 0.0  # PAD
    whitelist = np.arange(1, args.items)
    rng = np.random.default_rng(1)
    targets = np.sort(rng.choice(np.arange(1, args.items), args.targets, replace=False))
    users = (torch.randn((args.users, args.d), generator=torch.Generator().manual_seed(2)) / np.sqrt(args.d)).contiguous()
    user_ids = np.arange(args.users)
    cols = np.sort(rng.integers(1, args.items, size=(args.users, args.viewed), dtype=np.int32), axis=1)
    from scipy import sparse

    viewed = sparse.csr_matrix((np.ones(cols.size, np.float32), cols.reshape(-1), np.arange(args.users + 1) * args.viewed),
                               shape=(args.users, args.items))
    results = []
    for dtype in ("float32", "bfloat16"):
        item_embs = items32.to(getattr(torch, dtype))
        routes = args.routes.split(",")
        cases = [("i2i", "cosine")] * ("i2i" in routes) + [("u2i", dist) for dist in ("dot", "cosine") if "u2i" in routes]
        for route, dist in cases:
            outs = {}
            row = dict(header, route=route, distance=dist, dtype=dtype, n_items=args.items, d=args.d, k=args.k)
            for arm, cls in arms.items():
                if route == "i2i":
                    row["n_targets"] = args.targets

                    def call(cls=cls):
                        r = cls(distance=dist, device=item_embs.device, subjects_factors=item_embs, objects_factors=item_embs)
                        return r.rank(subject_ids=targets, k=args.k, filter_pairs_csr=None, sorted_object_whitelist=whitelist)
                else:
                    row["n_users"], row["viewed_per_user"] = args.users, args.viewed

                    def call(cls=cls):
                        r = cls(distance=dist, device=item_embs.device, subjects_factors=users[user_ids], objects_factors=item_embs)
                        return r.rank(subject_ids=np.arange(len(user_ids)), k=args.k, filter_pairs_csr=viewed,
                                      sorted_object_whitelist=whitelist)

                print(f"# {route} {dist} {dtype}: {arm} ...", flush=True)
                out, ms, peak = _time(call, args.repeats)
                outs[arm] = tuple(np.asarray(v.cpu() if hasattr(v, "cpu") else v) for v in out)
                row[f"{arm}_ms"] = ms
                row[f"{arm}_peak_bytes"] = peak
                torch.cuda.empty_cache()
            row["agree"] = _agree(outs["installed"], outs["stock"])
            row["speedup"] = row["stock_ms"]["median"] / row["installed_ms"]["median"]
            print(json.dumps(row), flush=True)
            results.append(row)
        del item_embs
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

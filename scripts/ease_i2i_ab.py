"""EASE item-to-item on the GPU (path 4: the weight rows ranked where the engine holds them) against the reference's numpy
`EASEModel._recommend_i2i` (rectools/models/ease.py:163-188), the unmodified method of the staged reference package.

    python scripts/ease_i2i_ab.py [--items 20000,50000] [--ks 10,100] [--steps 5] [--ref-targets 200] [--out DIR]

Weights: random fp32 EASE-shaped matrices (items x items, zero diagonal) set as `EASEModel().weight`.  Targets: every
item.  Per (items, k), each GPU route runs --steps times after one warm-up call (medians reported):
  engine   `rank_object_rows_padded` on an engine created once: wall-clock ms per call (host inputs and outputs), the
           engine's ms_select (CUDA events around the selection kernel) and the row bytes the selection reads (one stored
           row per target, items x 4 B) as GB/s of that kernel time -- the first read of a row comes from HBM, the
           re-reads of the radix passes mostly from L2;
  install  `model._recommend_i2i(...)` after `rectools_b200.install()`: what `recommend_to_items` calls, including the
           `content_hash` of the whole weight by which every call finds its cached engine (timed alone as well).
The reference runs on a sample of --ref-targets targets on the host CPU; its time for every item is an extrapolation
(linear in the targets) and labelled so.  The GPU's name and power limit are printed with every line.  Needs the staged
reference package (oracle/_ref, made by `__graft_entry__.build()`).  Prints one JSON line per measurement and writes them
to DIR/ease_i2i_ab.jsonl."""
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

import rectools_b200  # noqa: E402
from oracle import stage_reference  # noqa: E402
from rectools_b200 import Engine  # noqa: E402
from rectools_b200.integration import clear_engine_cache, content_hash  # noqa: E402
from rectools_b200.ranker import rank_object_rows_padded  # noqa: E402


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pylint: disable=broad-except
        return f"unavailable: {e}"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", default="20000,50000")
    ap.add_argument("--ks", default="10,100")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--ref-targets", type=int, default=200)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    gpu = gpu_info()
    lines = []
    stage_reference.add_to_path()
    from rectools.models import EASEModel  # pylint: disable=import-outside-toplevel

    reference_i2i = EASEModel._recommend_i2i  # pylint: disable=protected-access  (the unmodified method)

    def emit(rec):
        rec["gpu"] = gpu
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    for n in (int(x) for x in args.items.split(",")):
        rng = np.random.default_rng(n)
        w = np.empty((n, n), np.float32)
        for r0 in range(0, n, 4096):  # in slices: no fp64 temporary of the whole matrix
            w[r0:r0 + 4096] = rng.standard_normal((min(4096, n - r0), n), dtype=np.float32) * np.float32(0.01)
        np.fill_diagonal(w, 0.0)
        model = EASEModel()
        model.weight = w
        targets = np.arange(n, dtype=np.int64)
        sample = np.sort(rng.choice(n, min(args.ref_targets, n), replace=False))

        def timed(fn):
            fn()  # warm-up
            walls, stats = [], []
            for _ in range(args.steps):
                t0 = time.perf_counter()
                out = fn()
                walls.append((time.perf_counter() - t0) * 1e3)
                stats.append(dict(eng_stats()))
            return float(np.median(walls)), stats, out

        eng = Engine(w, cosine=False)
        eng_stats = lambda: eng.last_stats  # noqa: E731
        engine_runs = {}
        for k in (int(x) for x in args.ks.split(",")):
            engine_runs[k] = timed(lambda k=k: rank_object_rows_padded(eng, targets, k))
        eng.close()
        t0 = time.perf_counter()
        content_hash(w)
        hash_ms = (time.perf_counter() - t0) * 1e3
        rectools_b200.install(device=0)
        try:
            from rectools_b200 import integration  # pylint: disable=import-outside-toplevel

            eng_stats = lambda: next(iter(integration._ENGINE_CACHE.values())).last_stats  # noqa: E731  pylint: disable=protected-access
            install_runs = {k: timed(lambda k=k: model._recommend_i2i(targets, None, k, None))  # pylint: disable=protected-access
                            for k in engine_runs}
        finally:
            rectools_b200.uninstall()
            clear_engine_cache()
        for k, (wall, stats, (_, ids, scores, _counts)) in engine_runs.items():
            ms_sel = float(np.median([st["ms_select"] for st in stats]))
            st = stats[-1]
            # the unmodified reference method on a sample of the targets, checked against the GPU route on those targets
            t0 = time.perf_counter()
            _, _, ref_scores = reference_i2i(model, sample, None, k, None)
            ref_ms = (time.perf_counter() - t0) * 1e3
            np.testing.assert_array_equal(np.asarray(ref_scores).reshape(len(sample), -1), scores[sample])
            inst_wall, _, (_, inst_ids, _) = install_runs[k]
            np.testing.assert_array_equal(inst_ids.reshape(n, -1), ids)
            ref_all = ref_ms * n / len(sample)
            emit({
                "items": n, "k": k, "targets": n, "path": st["path"], "n_chunks": st["n_chunks"], "n_launches": st["n_launches"],
                "engine_ms_per_call_wall": round(wall, 3), "engine_ms_total": round(float(np.median([x["ms_total"] for x in stats])), 3),
                "engine_ms_select": round(ms_sel, 3), "row_bytes_read": 4 * n * n,
                "row_read_gb_per_s_of_ms_select": round(4 * n * n / (ms_sel * 1e-3) / 1e9, 1),
                "install_ms_per_call_wall": round(inst_wall, 3), "content_hash_ms": round(hash_ms, 2),
                "ref_targets_measured": len(sample), "ref_ms_measured": round(ref_ms, 2),
                "ref_ms_all_targets_extrapolated": round(ref_all, 1),
                "speedup_engine_vs_ref_extrapolated": round(ref_all / wall, 1),
                "speedup_install_vs_ref_extrapolated": round(ref_all / inst_wall, 1),
            })
        del w, model
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ease_i2i_ab.jsonl"), "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()

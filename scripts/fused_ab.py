#!/usr/bin/env python
"""A/B of two builds of the engine library on bench.py's workloads, alternated, with output comparison.

    python scripts/fused_ab.py --base rectools_b200/libb200rank_parent.so [--new rectools_b200/libb200rank.so] --out DIR

The base library is usually the parent commit built with the same flags (`git worktree add` + `python -m
rectools_b200.build` there, copied here under an untracked name: `*.so` is git-ignored).  Each library is loaded
through B200_RANK_LIB.  Per workload the arms alternate `--reps` times; every bench.py JSON line is kept in DIR/runs.jsonl,
every arm writes `--dump-outputs`, and the dumps of the two arms are compared array for array (then deleted unless
--keep-dumps).  Config 2 is also run
under B200_TC_DEBUG=1 (no candidates: MMA + staging + threshold scan only) and =2 (the epilogue skips the staged reads)
with --debug-reps N: `ms_main` then also counts the re-rank launches of the rows those modes leave uncertified.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKLOADS = {
    "c2": ["--config", "c2"],
    "c3": ["--config", "c3"],
    "c5u": ["--config", "c5", "--users", "262144", "--parity-users", "256"],
}


def run_bench(lib: str, args: list, steps: int, warmup: int, debug: int, dump: str | None) -> dict:
    env = dict(os.environ, B200_RANK_LIB=os.path.abspath(lib))
    env.pop("B200_TC_DEBUG", None)
    if debug:
        env["B200_TC_DEBUG"] = str(debug)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--no-cpu-baseline", "--no-model", "--no-e2e", *args]
    if dump:
        cmd += ["--dump-outputs", dump]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    if res.returncode != 0 or not lines:
        sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
        raise RuntimeError(f"bench.py failed ({res.returncode}): {' '.join(cmd)}")
    return json.loads(lines[-1])


def same_outputs(a: str, b: str) -> dict:
    out = {}
    for name in ("rows", "ids", "scores", "counts"):
        pa, pb = os.path.join(a, name + ".npy"), os.path.join(b, name + ".npy")
        if os.path.exists(pa) or os.path.exists(pb):
            out[name] = bool(os.path.exists(pa) and os.path.exists(pb) and np.array_equal(np.load(pa), np.load(pb)))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True)
    ap.add_argument("--new", default=os.path.join(ROOT, "rectools_b200", "libb200rank.so"))
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--workloads", default="c2,c3,c5u")
    ap.add_argument("--debug-reps", type=int, default=0,
                    help="repetitions of the B200_TC_DEBUG decomposition of config 2 (default 0: skip; with no candidates every row "
                         "is re-ranked, about a minute per step on an H100)")
    ap.add_argument("--keep-dumps", action="store_true", help="keep the --dump-outputs arrays (tens of MB per arm)")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    arms = {"base": a.base, "new": a.new}
    runs, summary = [], {"card": card}
    log = open(os.path.join(a.out, "runs.jsonl"), "w")
    plan = [(w, 0) for w in a.workloads.split(",")]
    if a.debug_reps > 0 and "c2" in a.workloads.split(","):
        plan += [("c2", 1), ("c2", 2)]
    for wl, dbg in plan:
        key = wl if not dbg else f"{wl}_debug{dbg}"
        per = {"base": [], "new": []}
        for rep in range(a.reps if not dbg else a.debug_reps):
            for arm in (("base", "new") if rep % 2 == 0 else ("new", "base")):
                dump = os.path.join(a.out, key, f"{arm}_{rep}") if not dbg else None
                line = run_bench(arms[arm], WORKLOADS[wl], a.steps, a.warmup, dbg, dump)
                rec = {"workload": key, "arm": arm, "rep": rep, "card": card, "line": line}
                log.write(json.dumps(rec) + "\n")
                log.flush()
                eng = line["config"]["engine"]
                per[arm].append({
                    "ms_per_step": line["ms_per_step"], "steps_ms": line.get("ms_steps_rank0"),
                    "ms_main": line["roofline"].get("ms_per_launch"), "tflops": line["roofline"].get("achieved"),
                    "n_fallback_rows": eng.get("n_fallback_rows"),
                    "parity_mismatches": (line.get("parity") or {}).get("id_mismatches"),
                })
                print(key, arm, rep, json.dumps(per[arm][-1]), flush=True)
        entry = dict(per)
        if not dbg:
            entry["outputs_equal"] = [same_outputs(os.path.join(a.out, key, f"base_{r}"), os.path.join(a.out, key, f"new_{r}"))
                                      for r in range(a.reps)]
            if not a.keep_dumps:
                shutil.rmtree(os.path.join(a.out, key))
        for arm in ("base", "new"):
            entry[f"{arm}_mean_ms"] = float(np.mean([r["ms_per_step"] for r in per[arm]]))
        entry["ratio"] = entry["new_mean_ms"] / entry["base_mean_ms"]
        summary[key] = entry
        print(key, "ratio new/base = %.4f" % entry["ratio"], entry.get("outputs_equal"), flush=True)
    json.dump(summary, open(os.path.join(a.out, "summary.json"), "w"), indent=1)


if __name__ == "__main__":
    main()

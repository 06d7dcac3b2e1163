#!/usr/bin/env python
"""The fused kernel's main pass alone, two builds of the engine library alternated, on bench.py's config-2 inputs.

    python scripts/fused_pass_ab.py --base rectools_b200/libb200rank_parent.so [--new rectools_b200/libb200rank.so] --out DIR

Reports `ms_main_pass` of the call statistics -- CUDA events around the main-pass launches of the fused kernel only,
without the second-chance and re-rank launches that `ms_main` also sums -- for three arms:
  normal   the kernel as it ranks;
  debug2   B200_TC_DEBUG=2: the epilogue skips its reads of the staged accumulators;
  debug1   B200_TC_DEBUG=1: every threshold is +inf, so no score can become a candidate (with the threshold gate of the
           accumulator hand-off nothing is staged either: the MMA + TMA floor of the pass).
The debug modes leave every row uncertified, and the engine then ranks those rows again with its exhaustive kernel (about
a minute per million rows on an H100): so the debug arms rank the first --debug-users rows, and the normal arm is timed at
that size too, next to the full config-2 batch.  Each library runs in its own process (the library is chosen by
B200_RANK_LIB when the package loads); the two alternate --reps times, each arm takes the median of --calls calls after
one warm-up call.  Prints the card name, power limit and max SM clock, writes DIR/fused_pass_ab.json.

    python scripts/fused_pass_ab.py --profile rectools_b200/libb200rank_profile.so --out DIR

runs the measurement build instead (`python -m rectools_b200.build --variant profile -DB200_FUSED_PROFILE`): one call of
the normal arm at --users rows and one of debug1, each after a warm-up, and prints where the fused kernel waits, as shares
of the pass (the MMA warp group's thread 0 from start to end, per CTA): that thread on `full` (TMA / L2), on `qempty`
(the hand-off) and in `wgmma.wait_group` (the tensor pipe); the producer on `empty` / `aempty` (slots still in use);
the epilogue warps on `qfull` (mean over the eight).
Writes DIR/fused_profile.json.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("ms_main_pass", "ms_main", "ms_total", "n_tc_launches", "n_fallback_rows")
PROF_FIELDS = ("full", "handoff", "pipe", "empty", "qfull", "pass")  # the counters of fused_topk.cuh, in its order


def worker(a) -> None:
    """One library (this process's B200_RANK_LIB): every arm, --calls timed calls each, JSON on stdout."""
    sys.path.insert(0, ROOT)
    import torch

    from bench import CONFIGS, gen_factors, gen_viewed
    from rectools_b200 import Engine, _lib

    cfg = CONFIGS["c2"]
    n_users, n_items, d, k = a.users, cfg["items"], cfg["dim"], cfg["k"]
    users = gen_factors(n_users, d, 0)
    items = gen_factors(n_items, d, 1)
    indptr, indices = gen_viewed(n_users, n_items, cfg["viewed"])
    dev = torch.device("cuda", 0)
    eng = Engine(items, cosine=False, device=0, tc_mode=cfg["tc"])
    d_users = torch.from_numpy(users).to(dev)
    d_indptr = torch.from_numpy(indptr).to(dev)
    d_indices = torch.from_numpy(indices).to(dev)
    o_ids = torch.empty((n_users, k), dtype=torch.int32, device=dev)
    o_sc = torch.empty((n_users, k), dtype=torch.float32, device=dev)
    o_cnt = torch.empty((n_users,), dtype=torch.int32, device=dev)

    def call(n_rows):
        st = eng.topk_ptrs(n_rows, k, o_ids.data_ptr(), o_sc.data_ptr(), o_cnt.data_ptr(),
                           _lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE,
                           subjects=d_users.data_ptr(), indptr=d_indptr.data_ptr(), indices=d_indices.data_ptr(),
                           stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return {f: st[f] for f in FIELDS}

    out = {}
    if a.profile_worker:
        import ctypes

        lib = _lib.load()
        lib.b200_rank_fused_profile.restype = ctypes.c_int
        lib.b200_rank_fused_profile.argtypes = [ctypes.c_int32, ctypes.POINTER(ctypes.c_ulonglong)]
        cnt = (ctypes.c_ulonglong * len(PROF_FIELDS))()
        for name, dbg, n_rows in [("normal", 0, n_users), ("debug1", 1, a.debug_users)]:
            if dbg:
                os.environ["B200_TC_DEBUG"] = str(dbg)
            else:
                os.environ.pop("B200_TC_DEBUG", None)
            call(n_rows)  # warm-up
            _lib.check(lib.b200_rank_fused_profile(0, cnt))
            st = call(n_rows)
            _lib.check(lib.b200_rank_fused_profile(0, cnt))
            c = dict(zip(PROF_FIELDS, (int(v) for v in cnt)))
            pas = max(c["pass"], 1)
            out[name] = {"rows": n_rows, "ms_main_pass": st["ms_main_pass"], "cycles": c,
                         "shares": {"mma_full": c["full"] / pas, "mma_handoff": c["handoff"] / pas,
                                    "mma_wgmma_wait": c["pipe"] / pas, "producer_empty": c["empty"] / pas,
                                    "epilogue_qfull": c["qfull"] / (8 * pas)}}
        os.environ.pop("B200_TC_DEBUG", None)
        eng.close()
        print("RESULT " + json.dumps(out), flush=True)
        return
    arms = [("normal", 0, n_users), ("normal_small", 0, a.debug_users), ("debug2", 2, a.debug_users), ("debug1", 1, a.debug_users)]
    for name, dbg, n_rows in arms:
        if dbg:
            os.environ["B200_TC_DEBUG"] = str(dbg)  # hooks are read once per call
        else:
            os.environ.pop("B200_TC_DEBUG", None)
        call(n_rows)  # warm-up
        calls = [call(n_rows) for _ in range(a.calls)]
        out[name] = {"rows": n_rows, "ms_main_pass": float(np.median([c["ms_main_pass"] for c in calls])), "calls": calls}
    os.environ.pop("B200_TC_DEBUG", None)
    eng.close()
    print("RESULT " + json.dumps(out), flush=True)


def run_worker(lib: str, a, profile: bool = False) -> dict:
    env = dict(os.environ, B200_RANK_LIB=os.path.abspath(lib))
    env.pop("B200_TC_DEBUG", None)
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--users", str(a.users), "--debug-users", str(a.debug_users),
           "--calls", str(a.calls)] + (["--profile-worker"] if profile else [])
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("RESULT ")]
    if res.returncode != 0 or not lines:
        sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
        raise RuntimeError(f"worker failed ({res.returncode}) for {lib}")
    return json.loads(lines[-1][len("RESULT "):])


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="library of the parent commit (built with the same flags, an untracked *.so)")
    ap.add_argument("--new", default=os.path.join(ROOT, "rectools_b200", "libb200rank.so"))
    ap.add_argument("--only", choices=["base", "new"], help="run one library only")
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--users", type=int, default=1_000_000, help="rows of the normal arm (config 2: 1M)")
    ap.add_argument("--debug-users", type=int, default=65_536, help="rows of the debug arms and of normal_small")
    ap.add_argument("--profile", help="a B200_FUSED_PROFILE build: report the kernel's wait shares instead of the A/B")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--profile-worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a)
        return
    if a.out is None:
        ap.error("--out is required")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, flush=True)
    if a.profile:
        r = run_worker(a.profile, a, profile=True)
        print("wait shares of the pass:", json.dumps({m: {"rows": v["rows"], "ms_main_pass": round(v["ms_main_pass"], 2),
                                                          **{k: round(x, 3) for k, x in v["shares"].items()}}
                                                      for m, v in r.items()}, indent=1), flush=True)
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fused_profile.json"), "w") as f:
            json.dump({"card": card, "users": a.users, "debug_users": a.debug_users, "profile": r}, f, indent=1)
        return
    arms = {"base": a.base, "new": a.new}
    if a.only:
        arms = {a.only: arms[a.only]}
    if any(v is None for v in arms.values()):
        ap.error("--base is required unless --only new")
    per = {arm: [] for arm in arms}
    for rep in range(a.reps):
        order = list(arms) if rep % 2 == 0 else list(arms)[::-1]
        for arm in order:
            r = run_worker(arms[arm], a)
            per[arm].append(r)
            print(rep, arm, json.dumps({m: (v["rows"], round(v["ms_main_pass"], 2)) for m, v in r.items()}), flush=True)
    table = {}
    for arm, reps in per.items():
        table[arm] = {m: float(np.median([r[m]["ms_main_pass"] for r in reps])) for m in reps[0]}
    if len(arms) == 2:
        table["new/base"] = {m: table["new"][m] / table["base"][m] for m in table["base"] if table["base"][m] > 0}
    print("median ms_main_pass:", json.dumps(table, indent=1), flush=True)
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "fused_pass_ab.json"), "w") as f:
        json.dump({"card": card, "users": a.users, "debug_users": a.debug_users, "calls": a.calls, "median_ms_main_pass": table,
                   "runs": per}, f, indent=1)


if __name__ == "__main__":
    main()

"""Widened (fp32 master copy) against 16-bit (B200_F_OBJECTS_16BIT) object factors on the config-5 shape.

    python scripts/objects16_ab.py [--items 5000000] [--dim 256] [--rows 65536] [--k 20] [--rounds 5]
                                   [--large-k-rows 4000] [--out DIR]

bf16 item embeddings on the device (SASRec-shaped, bench.py config 5: d = 256, 5M items, K = 20), subjects rounded to
bf16 values, a viewed-items filter of 100 items per row, device inputs and outputs.  For Distance.DOT and COSINE, two
engines over the same bf16 tensor -- the widened one and the one that keeps the objects at 16 bits -- rank the same
--rows rows in alternating order for --rounds rounds after one warm-up call each; then path 3 (k = 1025) on
--large-k-rows rows.  Per engine: `hbm_bytes`, the median `ms_total` / `ms_select` / `ms_main` of the call statistics
(CUDA events on the engine stream) and whether the outputs of the timed calls are bit-identical between the two.
Prints one JSON line per measurement, with the card's name and power limit; with --out DIR also writes them to
DIR/objects16_ab.jsonl."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rectools_b200 import Engine, _lib  # noqa: E402


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().replace("\n", "; ")
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=5_000_000)
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--rows", type=int, default=65_536)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--viewed", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--large-k-rows", type=int, default=4000)
    ap.add_argument("--out", default="", help="directory for objects16_ab.jsonl (default: print only)")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dev = torch.device("cuda:0")
    card = gpu_info()
    g = torch.Generator(device=dev).manual_seed(0)
    items = (torch.randn((a.items, a.dim), generator=g, device=dev) / a.dim**0.5).to(torch.bfloat16)
    subjects = (torch.randn((a.rows, a.dim), generator=g, device=dev) / a.dim**0.5).to(torch.bfloat16).float()
    cols = torch.randint(0, a.items, (a.rows, a.viewed), generator=g, device=dev, dtype=torch.int32).sort(dim=1).values
    indptr = torch.arange(a.rows + 1, device=dev, dtype=torch.int64) * a.viewed
    stream = torch.cuda.current_stream(dev).cuda_stream
    lines = []

    def emit(line):
        line["card"] = card
        print(json.dumps(line), flush=True)
        lines.append(line)

    def call(eng, n, k):
        k_out = min(k, a.items)
        out = (torch.empty((n, k_out), dtype=torch.int32, device=dev), torch.empty((n, k_out), dtype=torch.float32, device=dev),
               torch.empty((n,), dtype=torch.int32, device=dev))
        st = eng.topk_ptrs(n, k, out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                           _lib.Q_INPUTS_ON_DEVICE | _lib.Q_OUTPUTS_ON_DEVICE, subjects=subjects.data_ptr(), indptr=indptr.data_ptr(),
                           indices=cols.data_ptr(), stream=stream)
        torch.cuda.synchronize(dev)
        return dict(st), out

    for distance in ("dot", "cosine"):
        kw = dict(objects_device_ptr=items.data_ptr(), shape=(a.items, a.dim), objects_dtype=_lib.DT_BF16, tc_mode="bf16")
        engines = {"widened": Engine(None, cosine=distance == "cosine", **kw),
                   "16bit": Engine(None, cosine=distance == "cosine", keep_16bit=True, **kw)}
        hbm = {name: int(e.info()["hbm_bytes"]) for name, e in engines.items()}  # before any call: the resident data only
        for label, n, k in (("config5", a.rows, a.k), ("path3_k1025", min(a.large_k_rows, a.rows), 1025)):
            stats = {name: [] for name in engines}
            last = {}
            for name, e in engines.items():  # warm-up
                call(e, n, k)
            for r in range(a.rounds):
                order = list(engines) if r % 2 == 0 else list(engines)[::-1]
                for name in order:
                    st, out = call(engines[name], n, k)
                    stats[name].append(st)
                    last[name] = out
            x, y = last["widened"], last["16bit"]
            same = bool(torch.equal(x[0], y[0]) and torch.equal(x[1].view(torch.int32), y[1].view(torch.int32)) and torch.equal(x[2], y[2]))
            for name in engines:
                med = {f: float(np.median([s[f] for s in stats[name]])) for f in ("ms_total", "ms_select", "ms_main")}
                emit({"distance": distance, "workload": label, "engine": name, "rows": n, "k": k, "items": a.items, "dim": a.dim,
                      "hbm_bytes": hbm[name], "path": stats[name][-1]["path"], "rounds": a.rounds, **med,
                      "n_fallback_rows": int(stats[name][-1]["n_fallback_rows"]), "bit_identical": same})
        for e in engines.values():
            e.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "objects16_ab.jsonl"), "w") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

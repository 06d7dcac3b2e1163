"""A/B of the selection of paths 2 and 3 at large k: the radix selection (default, B200_SELECT=1) against the ceil(k/32)
streaming passes (B200_SELECT=0), alternated in one process on the same engine and inputs, outputs compared bit for bit.

    python scripts/large_k_ab.py [--users 8192] [--items 1000000] [--dim 128] [--ks 1025,2048,4096,10000]
                                 [--passes-ks 1025,2048] [--none-users 512] [--ease-items 20000] [--ease-users 8192]
                                 [--out DIR]

Dense workload: DOT, 100 viewed items per user filtered, k in --ks; the passes arm runs only at --passes-ks (above that it
takes minutes per step: its time is extrapolated from the measured cost per pass and labelled so), and k = None over the
whole catalogue runs the radix arm only, for --none-users users.  EASE workload: sparse
subjects (~50 interactions per user) over an items x items weight matrix, k = None (all items), both arms once.
Prints one JSON line per measurement and writes them to DIR/large_k_ab.jsonl."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
from scipy import sparse

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rectools_b200 import Engine  # noqa: E402


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pylint: disable=broad-except
        return f"unavailable: {e}"


def viewed_csr(rng, n_rows, n_cols, per_row):
    idx = np.sort(rng.integers(0, n_cols, (n_rows, per_row)), axis=1)
    indptr = np.arange(n_rows + 1, dtype=np.int64) * per_row
    return indptr, idx.reshape(-1).astype(np.int32)


def step(eng, select, k, **kw):
    os.environ["B200_SELECT"] = str(select)
    try:
        t0 = time.perf_counter()
        out = eng.topk(k, **kw)  # host outputs: returns after the call's final synchronisation
        ms = (time.perf_counter() - t0) * 1e3
    finally:
        del os.environ["B200_SELECT"]
    st = eng.last_stats
    return out, dict(ms_step=round(ms, 1), ms_main=round(st["ms_main"], 1), ms_select=round(st["ms_select"], 1),
                     n_launches=st["n_launches"], path=st["path"])


def same(a, b):
    return all(np.array_equal(np.ascontiguousarray(x).view(np.int32), np.ascontiguousarray(y).view(np.int32)) for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=8192)
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--ks", default="1025,2048,4096,10000")
    ap.add_argument("--passes-ks", default="1025,2048")
    ap.add_argument("--none-users", type=int, default=512, help="users of the dense k = None step")
    ap.add_argument("--ease-items", type=int, default=20_000)
    ap.add_argument("--ease-users", type=int, default=8192)
    ap.add_argument("--out", default="bench_out")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    lines = []

    def emit(rec):
        rec["gpu"] = info
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    info = gpu_info()
    rng = np.random.default_rng(0)
    objects = (rng.standard_normal((a.items, a.dim), dtype=np.float32) / np.sqrt(a.dim)).astype(np.float32)
    subjects = rng.standard_normal((a.users, a.dim), dtype=np.float32)
    indptr, indices = viewed_csr(rng, a.users, a.items, 100)
    eng = Engine(objects, cosine=False)
    kw = dict(subjects=subjects, indptr=indptr, indices=indices)
    step(eng, 1, 1025, **kw)  # warm-up: module load, buffers
    passes_ks = {int(k) for k in a.passes_ks.split(",") if k}
    per_pass = None
    for k in (int(k) for k in a.ks.split(",")):
        rad1, r1 = step(eng, 1, k, **kw)
        rec = dict(workload="dense", users=a.users, items=a.items, dim=a.dim, k=k, radix=r1)
        if k in passes_ks:
            pas, rp = step(eng, 0, k, **kw)
            rad2, r2 = step(eng, 1, k, **kw)
            rec.update(passes=rp, radix_again=r2, equal=same(rad1, pas) and same(rad1, rad2))
            per_pass = rp["ms_select"] / ((k + 31) // 32)
        elif per_pass is not None:
            rec["passes_ms_select_extrapolated"] = round(per_pass * ((k + 31) // 32), 1)
        emit(rec)
        del rad1
    # k = None over the whole catalogue: radix only (the passes would take ceil(N / 32) passes); fewer users, since the
    # outputs alone take N x 8 B per user
    sub_none = dict(kw, subjects=subjects[: a.none_users], indptr=indptr[: a.none_users + 1])
    _, rn = step(eng, 1, a.items, **sub_none)
    rec = dict(workload="dense", users=a.none_users, items=a.items, dim=a.dim, k="None", radix=rn)
    if per_pass is not None:
        rec["passes_ms_select_extrapolated"] = round(per_pass * a.none_users / a.users * ((a.items + 31) // 32), 1)
    emit(rec)
    eng.close()
    del objects

    # EASE-shaped: items x items weights, sparse user rows, k = None
    n = a.ease_items
    weights = (rng.standard_normal((n, n), dtype=np.float32) * 0.01).astype(np.float32)
    nnz = 50
    sp = sparse.csr_matrix((np.ones(a.ease_users * nnz, np.float32), rng.integers(0, n, a.ease_users * nnz).astype(np.int32),
                            np.arange(a.ease_users + 1, dtype=np.int64) * nnz), shape=(a.ease_users, n))
    sp.sum_duplicates()
    eng = Engine(weights, cosine=False)
    fk = dict(sparse_subjects=sp, indptr=sp.indptr.astype(np.int64), indices=sp.indices.astype(np.int32))
    step(eng, 1, 1025, **fk)  # warm-up (transposed weights built here)
    rad, r1 = step(eng, 1, n, **fk)
    pas, rp = step(eng, 0, n, **fk)
    emit(dict(workload="ease", users=a.ease_users, items=n, k="None", radix=r1, passes=rp, equal=same(rad, pas)))
    eng.close()
    with open(os.path.join(a.out, "large_k_ab.jsonl"), "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()

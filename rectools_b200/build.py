"""Build libb200rank.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m rectools_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import typing as tp

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200rank.so")
SOURCES = ["engine.cu", "group.cu", "pairs.cu", "list.cu", "list_mix.cu", "knn.cu"]
HEADERS = ["cuda_call.h", "common.cuh", "sizes.h", "plan.h", "group_plan.h", "engine_internal.h", "order_key.h", "large_k_select.cuh", "row_select.cuh", "cand_select.cuh", "cand_prep.cuh", "prep.cuh", "select.cuh", "sparse.cuh", "tc_common.cuh", "fused_topk.cuh", "pairs_select.cuh", "list_plan.h", "list_select.cuh", "list_call.h", "list_mix_plan.h", "list_mix.cuh", "knn.cuh", "knn_plan.h", os.path.join("..", "..", "include", "b200_rank.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wno-format-truncation",
    "-shared",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC or add /usr/local/cuda/bin to PATH)")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(os.path.normpath(d)) > t for d in deps)


def build(force: bool = False, verbose: bool = False, variant: str = "", defines: tp.Sequence[str] = ()) -> str:
    """`variant` / `defines`: measurement builds (libb200rank_<variant>.so with extra -D flags, loaded through the
    B200_RANK_LIB environment variable); the product library is the plain build."""
    out = LIB if not variant else os.path.join(HERE, f"libb200rank_{variant}.so")
    if not variant and not force and not needs_build():
        return LIB
    cmd = [_nvcc(), *NVCC_FLAGS, *defines, "-o", out, *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas")
        cmd.insert(2, "-v")
        print(" ".join(cmd))
    env = dict(os.environ)
    # the image exports CC/CXX pointing at a gcc without a usable spec set; let nvcc pick the system g++
    env.pop("CC", None)
    env.pop("CXX", None)
    res = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libb200rank.so")
    if verbose:
        print(res.stdout + res.stderr)
    return out


if __name__ == "__main__":
    _variant = sys.argv[sys.argv.index("--variant") + 1] if "--variant" in sys.argv else ""
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, variant=_variant,
                defines=[a for a in sys.argv[1:] if a.startswith("-D")]))

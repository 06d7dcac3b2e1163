"""CPU: the fused kernel's wgmma pipeline as ptxas builds it.

ptxas reports C7514 (wgmmas serialised because other instructions read accumulator registers) and C7517 (a
warpgroup.wait injected so that such registers can be used) when accumulators are touched while their wgmma is in
flight, and C7512 when it serialises wgmmas for lack of registers.  Each drains the tensor pipe.  The test compiles the
library with the product flags into a temporary directory and checks that none of these reports names a
fused_topk_kernel instantiation, and that none of the six instantiations (plain, wide and peers, each with fp16 and bf16
operands) spills.  About half a minute of compile; skipped without nvcc."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


@pytest.fixture(scope="module")
def ptxas_log():
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    from rectools_b200 import build

    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc, "-Xptxas", "-v", *build.NVCC_FLAGS, "-o", os.path.join(tmp, "lib.so"),
               *[os.path.join(build.CSRC, s) for s in build.SOURCES]]
        res = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=tmp)
    assert res.returncode == 0, res.stdout + res.stderr
    return res.stdout + res.stderr


def _spills(log):
    """{mangled fused_topk_kernel name: spill store bytes} from the ptxas -v report."""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1) if "fused_topk_kernel" in m.group(1) else None
            continue
        m = re.search(r"(\d+) bytes spill stores", line)
        if m and cur:
            out[cur] = int(m.group(1))
            cur = None
    return out


def test_no_injected_wgmma_waits(ptxas_log):
    bad = [ln for ln in ptxas_log.splitlines() if re.search(r"C751[247]", ln) and "fused_topk_kernel" in ln]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("kind", ["plain", "wide", "peers"])
def test_fused_kernels_do_not_spill(ptxas_log, kind):
    spills = _spills(ptxas_log)
    assert len(spills) == 6, spills
    wide, peers = int(kind == "wide"), int(kind == "peers")
    names = [n for n in spills if re.search(rf"fused_topk_kernelILb{wide}ELb{peers}ELb[01]E", n)]
    assert len(names) == 2, names  # fp16 and bf16 operands
    for n in names:
        assert spills[n] == 0, (n, spills[n])

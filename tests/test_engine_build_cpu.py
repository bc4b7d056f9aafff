"""The tensor-core GEMM engine (csrc/umma.cu) compiles without register spills.

Every `umma_kernel` instantiation keeps its accumulators, operand fragments and addresses in registers at the 168-register cap of its
288-thread CTA.  A spill puts local-memory round trips into the MMA loop or the epilogue, and with the operand ring taking all of shared
memory there is little L1 left to absorb them.  The check reads ptxas's report from the build log `build()` leaves in
makani_b200/build/umma.o.log, or compiles umma.cu into a temporary directory when that log is missing or older than the sources.
Needs nvcc, not a GPU.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "makani_b200", "csrc")
LOG = os.path.join(ROOT, "makani_b200", "build", "umma.o.log")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc is not available")


def _ptxas_report():
    sources = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    if os.path.exists(LOG) and os.path.getmtime(LOG) >= max(os.path.getmtime(s) for s in sources):
        with open(LOG) as f:
            return f.read()
    from makani_b200 import build as _build

    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [nvcc] + _build.FLAGS + ["-c", os.path.join(CSRC, "umma.cu"), "-o", os.path.join(tmp, "umma.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout + r.stderr


def _kernels(report):
    """{mangled name: (spill store bytes, spill load bytes, registers)} of every umma_kernel instantiation"""
    out = {}
    pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?Function properties for \1\n\s+(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads\n.*?Used (\d+) registers")
    for m in pat.finditer(report):
        if "umma_kernel" in m.group(1):
            out[m.group(1)] = (int(m.group(3)), int(m.group(4)), int(m.group(5)))
    return out


def test_engine_kernels_do_not_spill():
    kernels = _kernels(_ptxas_report())
    # five GEMMs (analysis, synthesis, mix forward, dgrad, wgrad), each at several tile widths
    for traits in ("AnaTraits", "SynTraits", "MixFwdTraits", "MixDgradTraits", "MixWgradTraits"):
        assert any(traits in k for k in kernels), f"no umma_kernel<{traits}, ...> in the ptxas report"
    spilling = {k: v for k, v in kernels.items() if v[0] or v[1]}
    assert not spilling, "umma_kernel instantiations spill (store bytes, load bytes, registers): " + ", ".join(
        f"{k}: {v}" for k, v in sorted(spilling.items()))

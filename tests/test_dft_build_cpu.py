"""The tensor-core longitude DFT kernels (csrc/dft.cu) compile without register spills.

`dft_analysis_kernel` runs 16 warps, so each thread has 128 registers; its producer warps hold two rows x 16 samples and their radix-8
outputs, the MMA warps 32 accumulators plus 16-byte operand fragments.  A spill puts local-memory round trips into the butterflies or the
MMA loop of every tile.  `dft_synthesis_kernel` runs 12 warps at 168 registers; its MMA + epilogue warps keep 64 accumulators per thread.  The check reads ptxas's report from the build log
`build()` leaves in makani_b200/build/dft.o.log, or compiles dft.cu into a temporary directory when that log is missing or older than the
sources.  Needs nvcc, not a GPU.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "makani_b200", "csrc")
LOG = os.path.join(ROOT, "makani_b200", "build", "dft.o.log")
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
        cmd = [nvcc] + _build.FLAGS + ["-c", os.path.join(CSRC, "dft.cu"), "-o", os.path.join(tmp, "dft.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout + r.stderr


def _kernels(report):
    """{mangled name: (spill store bytes, spill load bytes, registers)} of every DFT kernel instantiation"""
    out = {}
    pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?Function properties for \1\n\s+(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads\n.*?Used (\d+) registers")
    for m in pat.finditer(report):
        if "dft_analysis_kernel" in m.group(1) or "dft_synthesis_kernel" in m.group(1):
            out[m.group(1)] = (int(m.group(3)), int(m.group(4)), int(m.group(5)))
    return out


def test_dft_kernels_do_not_spill():
    kernels = _kernels(_ptxas_report())
    # analysis: fp32 and bf16 samples x (the compile-time lengths N2 = 60, 90, 180 and the run-time one); synthesis: fp32 and bf16 output
    for name, count in (("dft_analysis_kernel", 8), ("dft_synthesis_kernel", 2)):
        assert sum(name in k for k in kernels) == count, f"expected {count} {name} instantiations in the ptxas report, found {sorted(kernels)}"
    spilling = {k: v for k, v in kernels.items() if v[0] or v[1]}
    assert not spilling, "DFT kernel instantiations spill (store bytes, load bytes, registers): " + ", ".join(
        f"{k}: {v}" for k, v in sorted(spilling.items()))

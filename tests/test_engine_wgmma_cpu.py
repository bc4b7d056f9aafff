"""The TF32 K-major GEMMs of the tensor-core engine (csrc/umma.cu) run on wgmma, and only they do.

`umma_kernel<AnaTraits, NB, false>` and `umma_kernel<MixDgradTraits, NB, false>` must hold HGMMA instructions and no HMMA; every other
instantiation (synthesis, mix forward, weight gradient, the 3 x TF32 analysis) stays on mma.sync.  ptxas must not serialize the wgmma
(warning C7510: a function call in the kernel, an accumulator touched while a wgmma is in flight), and the wrappers in
csrc/wgmma_tf32.cuh must be what scripts/gen_wgmma_tf32.py writes.  Reads makani_b200/build/umma.o and its log when `build()` left them
newer than the sources, otherwise compiles umma.cu into a temporary directory.  Needs nvcc and cuobjdump, not a GPU.
"""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "makani_b200", "csrc")
OBJ = os.path.join(ROOT, "makani_b200", "build", "umma.o")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)), reason="nvcc / cuobjdump are not available")


@pytest.fixture(scope="module")
def compiled():
    """(SASS dump, ptxas report) of umma.cu"""
    sources = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    newest = max(os.path.getmtime(s) for s in sources)
    if os.path.exists(OBJ) and os.path.exists(OBJ + ".log") and min(os.path.getmtime(OBJ), os.path.getmtime(OBJ + ".log")) >= newest:
        with open(OBJ + ".log") as f:
            report = f.read()
        sass = subprocess.run([CUOBJDUMP, "-sass", OBJ], capture_output=True, text=True, check=True).stdout
        return sass, report
    from makani_b200 import build as _build

    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "umma.o")
        r = subprocess.run([NVCC] + _build.FLAGS + ["-c", os.path.join(CSRC, "umma.cu"), "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return sass, r.stdout + r.stderr


def _mma_counts(sass):
    """{mangled umma_kernel name: (HGMMA count, HMMA count)}"""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "umma_kernel" in m.group(1) else None
            if cur:
                out[cur] = [0, 0]
        elif cur and "HGMMA." in line:
            out[cur][0] += 1
        elif cur and "HMMA." in line:
            out[cur][1] += 1
    return out


def test_wgmma_runs_exactly_the_tf32_k_major_gemms(compiled):
    counts = _mma_counts(compiled[0])
    wg = {k for k in counts if re.search(r"umma_kernelINS_\d+(AnaTraits|MixDgradTraits)ELi\d+ELb0E", k)}
    assert len([k for k in wg if "AnaTraits" in k]) == 7 and len([k for k in wg if "MixDgradTraits" in k]) == 3, sorted(wg)
    for k, (hgmma, hmma) in counts.items():
        if k in wg:
            assert hgmma > 0 and hmma == 0, f"{k}: {hgmma} HGMMA, {hmma} HMMA"
        else:
            assert hgmma == 0 and hmma > 0, f"{k}: {hgmma} HGMMA, {hmma} HMMA"


def test_wgmma_is_not_serialized(compiled):
    warnings = [line for line in compiled[1].splitlines() if "C7510" in line or "wgmma.mma_async instructions are serialized" in line]
    assert not warnings, "\n".join(warnings)


def test_wgmma_wrappers_are_generated():
    gen = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gen_wgmma_tf32.py")], capture_output=True, text=True, check=True).stdout
    with open(os.path.join(CSRC, "wgmma_tf32.cuh")) as f:
        assert f.read() == gen, "csrc/wgmma_tf32.cuh differs from scripts/gen_wgmma_tf32.py's output"

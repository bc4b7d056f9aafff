"""The longitude-DFT analysis contraction (csrc/dft.cu) runs on wgmma, and the synthesis stays on mma.sync.

Every `dft_analysis_kernel` instantiation must hold HGMMA instructions and no HMMA; every `dft_synthesis_kernel` instantiation holds HMMA
and no HGMMA.  ptxas must not serialize the wgmma (warning C7510: a function call in the kernel -- the printf of a timed-out mbarrier
wait, for one -- or an accumulator touched while a wgmma is in flight), neither in the shipped build nor in the wait-profile build
(-DB200SHT_DFT_PROFILE).  Reads makani_b200/build/dft.o and its log when `build()` left them newer than the sources, otherwise compiles
dft.cu into a temporary directory.  Needs nvcc and cuobjdump, not a GPU.
"""
import os
import re
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "makani_b200", "csrc")
OBJ = os.path.join(ROOT, "makani_b200", "build", "dft.o")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")

pytestmark = pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)), reason="nvcc / cuobjdump are not available")


def _compile(defines=()):
    """(SASS dump, ptxas report) of dft.cu built with the library's flags and `defines`"""
    from makani_b200 import build as _build

    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "dft.o")
        cmd = [NVCC] + _build.FLAGS + ["-D" + d for d in defines] + ["-c", os.path.join(CSRC, "dft.cu"), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return sass, r.stdout + r.stderr


@pytest.fixture(scope="module")
def compiled():
    sources = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    newest = max(os.path.getmtime(s) for s in sources)
    if os.path.exists(OBJ) and os.path.exists(OBJ + ".log") and min(os.path.getmtime(OBJ), os.path.getmtime(OBJ + ".log")) >= newest:
        with open(OBJ + ".log") as f:
            report = f.read()
        sass = subprocess.run([CUOBJDUMP, "-sass", OBJ], capture_output=True, text=True, check=True).stdout
        return sass, report
    return _compile()


def _mma_counts(sass):
    """{mangled DFT kernel name: [HGMMA count, HMMA count]}"""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if ("dft_analysis_kernel" in m.group(1) or "dft_synthesis_kernel" in m.group(1)) else None
            if cur:
                out[cur] = [0, 0]
        elif cur and "HGMMA." in line:
            out[cur][0] += 1
        elif cur and "HMMA." in line:
            out[cur][1] += 1
    return out


def _serialized(report):
    return [line for line in report.splitlines() if "C7510" in line or "wgmma.mma_async instructions are serialized" in line]


def test_dft_analysis_runs_on_wgmma(compiled):
    counts = _mma_counts(compiled[0])
    ana = {k: v for k, v in counts.items() if "dft_analysis_kernel" in k}
    syn = {k: v for k, v in counts.items() if "dft_synthesis_kernel" in k}
    assert len(ana) == 8 and len(syn) == 2, sorted(counts)
    for k, (hgmma, hmma) in ana.items():
        assert hgmma > 0 and hmma == 0, f"{k}: {hgmma} HGMMA, {hmma} HMMA"
    for k, (hgmma, hmma) in syn.items():
        assert hgmma == 0 and hmma > 0, f"{k}: {hgmma} HGMMA, {hmma} HMMA"


def test_dft_wgmma_is_not_serialized(compiled):
    warnings = _serialized(compiled[1])
    assert not warnings, "\n".join(warnings)


def test_dft_wgmma_is_not_serialized_in_the_profile_build():
    sass, report = _compile(["B200SHT_DFT_PROFILE"])
    warnings = _serialized(report)
    assert not warnings, "\n".join(warnings)
    for k, (hgmma, hmma) in _mma_counts(sass).items():
        if "dft_analysis_kernel" in k:
            assert hgmma > 0 and hmma == 0, f"{k}: {hgmma} HGMMA, {hmma} HMMA"

"""The worker loop of the longitude-DFT synthesis (csrc/dft.cu, `dft_synthesis_kernel`) keeps its issue per task low.

The load warp rewrites each landed latspec stage into fragment order, and A (E^T) is held in fragment order too, so a task loads its
fragments with 16-byte shared loads: 32 `LDS.128` for B and 4 for A, no scalar 32-bit shared load.  The bf16 epilogue converts the two
latitudes of a thread with one `F2FP` (never a pack against RZ), so there are half as many conversions as 2-byte stores.  64 `HMMA` per
task (2 planes x 8 classes x 4 k8 steps), no spills.  Checked in both instantiations (fp32 and bf16 output).  Reads
makani_b200/build/dft.o and its log when `build()` left them newer than the sources, otherwise compiles dft.cu into a temporary
directory.  Needs nvcc and cuobjdump, not a GPU.
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


@pytest.fixture(scope="module")
def compiled():
    """(SASS dump, ptxas report) of dft.cu as the library builds it"""
    sources = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh"))]
    newest = max(os.path.getmtime(s) for s in sources)
    if os.path.exists(OBJ) and os.path.exists(OBJ + ".log") and min(os.path.getmtime(OBJ), os.path.getmtime(OBJ + ".log")) >= newest:
        with open(OBJ + ".log") as f:
            report = f.read()
        return subprocess.run([CUOBJDUMP, "-sass", OBJ], capture_output=True, text=True, check=True).stdout, report
    from makani_b200 import build as _build

    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, "dft.o")
        r = subprocess.run([NVCC] + _build.FLAGS + ["-c", os.path.join(CSRC, "dft.cu"), "-o", obj], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return sass, r.stdout + r.stderr


def _synthesis_kernels(sass):
    """{mangled name: [instruction text]} of every dft_synthesis_kernel instantiation, without the never-executed `@!PT` padding"""
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "dft_synthesis_kernel" in m.group(1) else None
            if cur:
                out[cur] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if cur and m and not m.group(1).startswith("@!PT"):
            out[cur].append(m.group(1))
    return out


def _opcode(ins):
    return re.sub(r"^@!?U?P\w+\s+", "", ins).split()[0]


def test_synthesis_fragments_come_in_16_byte_loads(compiled):
    kernels = _synthesis_kernels(compiled[0])
    assert len(kernels) == 2, sorted(kernels)
    for name, code in kernels.items():
        ops = [_opcode(i) for i in code]
        assert ops.count("HMMA.1688.F32.TF32") == 64, f"{name}: {ops.count('HMMA.1688.F32.TF32')} HMMA"
        scalar = [i for i, o in zip(code, ops) if o == "LDS"]
        assert not scalar, f"{name}: 32-bit shared loads {scalar}"
        assert ops.count("LDS.128") >= 36, f"{name}: {ops.count('LDS.128')} LDS.128"


def test_synthesis_bf16_converts_latitude_pairs(compiled):
    kernels = {k: v for k, v in _synthesis_kernels(compiled[0]).items() if "bfloat16" in k}
    assert len(kernels) == 1, sorted(kernels)
    code = next(iter(kernels.values()))
    cvt = [i for i in code if _opcode(i).startswith("F2FP.BF16")]
    stores = [i for i in code if _opcode(i) == "STS.U16"]
    assert cvt and not [i for i in cvt if re.search(r",\s*RZ\b", i)], f"conversions packed against RZ: {cvt}"
    assert 2 * len(cvt) == len(stores), f"{len(cvt)} conversions for {len(stores)} 2-byte stores"


def test_synthesis_does_not_spill(compiled):
    pat = re.compile(r"Compiling entry function '(\S*dft_synthesis_kernel\S*)' for 'sm_90a'\n.*?Function properties for \1\n\s+\d+ bytes "
                     r"stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads")
    found = {m.group(1): (int(m.group(2)), int(m.group(3))) for m in pat.finditer(compiled[1])}
    assert len(found) == 2, sorted(found)
    assert all(v == (0, 0) for v in found.values()), found

"""Build the in-tree CUDA library makani_b200/libb200sht.so for sm_90a (H100) with nvcc (no GPU needed: cross-compiles)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200sht.so")
SOURCES = ["capi.cu", "fft.cu", "legendre.cu", "mix.cu", "act.cu", "umma.cu", "dft.cu", "norm.cu", "disco.cu", "resample.cu", "attention.cu", "attention_global.cu", "noise.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False, defines=(), out=OUT):
    """defines: extra -D macros (a separate object directory and output file per variant, e.g. the profile build
    `build(defines=["B200SHT_DFT_PROFILE"], out=.../libb200sht_prof.so)`)."""
    objdir = os.path.join(HERE, "build" + ("_" + "_".join(defines) if defines else ""))
    os.makedirs(objdir, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "b200sht.h"))
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        if force or _newer(src, obj) or any(_newer(h, obj) for h in headers):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC] + FLAGS + ["-D" + d for d in defines] + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(objdir, os.path.basename(obj) + ".log")
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=6) as ex:
        list(ex.map(compile_one, jobs))
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or not os.path.exists(out):
        cmd = [NVCC, "-shared", "-o", out] + objs + ["-lcudart", "-lcuda"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return out


if __name__ == "__main__":
    if "--define" in sys.argv:    # experiment builds: --define MACRO --out name.so
        d = sys.argv[sys.argv.index("--define") + 1]
        print(build(defines=d.split(","), out=os.path.join(HERE, sys.argv[sys.argv.index("--out") + 1])))
    elif "--profile" in sys.argv:   # wait-time counters in the DFT kernels (scripts/dft_waitprof.py); not the shipped build
        print(build(force="--force" in sys.argv, defines=["B200SHT_DFT_PROFILE"], out=os.path.join(HERE, "libb200sht_prof.so")))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

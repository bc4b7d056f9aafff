"""python -m makani_b200.build --profile; python scripts/dft_waitprof.py : where the roles of the DFT kernels wait (SM clocks per CTA, per tile)"""
import ctypes, os, sys
os.environ["B200SHT_DFT_PROF"] = "1"
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("B200SHT_LIBRARY", os.path.join(_ROOT, "makani_b200", "libb200sht_prof.so"))   # `python -m makani_b200.build --profile`
sys.path.insert(0, _ROOT)
import numpy as np, torch, makani_b200 as mb
from makani_b200 import _lib
from makani_b200.sht import _ptr, _stream, _VP
dev = torch.device("cuda", 0)
plan = mb.get_plan(721, 1440, 240, 241, "equiangular", True, dev)
B, C = 1, 73
x = torch.randn(B, C, 721, 1440, device=dev).bfloat16()
lat = torch.zeros(plan.latspec_elems(B, C), device=dev)
y = torch.empty_like(x)
st = _stream(dev)
lib = _lib.load()
cnt = np.zeros(16, dtype=np.uint64)
def read():
    lib.b200sht_debug_dft_profile(cnt.ctypes.data_as(ctypes.c_void_p)); return cnt.copy()
for _ in range(2):
    _lib.call("b200sht_fft_analysis", plan.handle, _ptr(x), 1, B, C, _ptr(lat), 0 | 2, st)
read()
_lib.call("b200sht_fft_analysis", plan.handle, _ptr(x), 1, B, C, _ptr(lat), 0 | 2, st)
a = read().astype(float)
def timed(fn, n=20):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize(); read()
    return e0.elapsed_time(e1) / n * 1e3
print("analysis us/launch (profile on):", round(timed(lambda: _lib.call("b200sht_fft_analysis", plan.handle, _ptr(x), 1, B, C, _ptr(lat), 0 | 2, st)), 1))
print("synthesis us/launch (profile on):", round(timed(lambda: _lib.call("b200sht_fft_synthesis", plan.handle, _ptr(lat), _ptr(y), 1, B, C, _VP(0), 0 | 2, st)), 1))
ctas = torch.cuda.get_device_properties(0).multi_processor_count   # one persistent CTA per SM
life = a[6] / ctas
print(f"analysis: CTA lifetime {life:.0f} clk; items {a[7]:.0f}")
names = ["producers wait samples (per warp)", "producers wait operand stage (per warp)", "loader waits raw stage", "MMA warps wait operand (per warp)"]
div = [8, 8, 1, 8]   # warps per role in dft_analysis_kernel: producers, producers, loader, MMA
for i, nme in enumerate(names):
    print(f"  {nme:45s} {a[i] / ctas / div[i]:10.0f} clk  = {100 * a[i] / ctas / div[i] / life:5.1f}% of the CTA lifetime")
for _ in range(2):
    _lib.call("b200sht_fft_synthesis", plan.handle, _ptr(lat), _ptr(y), 1, B, C, _VP(0), 0 | 2, st)
read()
_lib.call("b200sht_fft_synthesis", plan.handle, _ptr(lat), _ptr(y), 1, B, C, _VP(0), 0 | 2, st)
a = read().astype(float)
life = a[12] / ctas
print(f"synthesis: CTA lifetime {life:.0f} clk; tasks (8 columns of a tile) {a[13]:.0f}")
for i, nme, d in ((8, "load warp waits stage free", 1), (14, "load warp waits tile landed", 1),
                  (9, "MMA + epilogue warps wait stage rewritten (per warp)", 10),
                  (10, "epilogues wait output tile free (per warp)", 10), (11, "TMA store waits output tile written", 1)):
    print(f"  {nme:45s} {a[i] / ctas / d:10.0f} clk  = {100 * a[i] / ctas / d / life:5.1f}% of the CTA lifetime")

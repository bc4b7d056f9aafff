"""python -m makani_b200.build --define B200SHT_UMMA_PROFILE --out libb200sht_umma_prof.so; python scripts/umma_waitprof.py [--json FILE]

Where the roles of the tensor-core engine (csrc/umma.cu) spend a CTA's life, for the Legendre launches of the benched SFNO block
(721 x 1440 equiangular, lmax 240, mmax 241, B = 1, C = 73: its forward and backward passes run two analyses and two tiled syntheses of
this shape).  SM clocks per role, as a share of the CTA lifetime: the producer waiting for a free stage, the consumer warps waiting for
a loaded stage, in the MMA loop and in the epilogue.  B200SHT_LIBRARY selects the library (default: the profile build)."""
import ctypes, json, os, sys
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
os.environ.setdefault("B200SHT_LIBRARY", os.path.join(_ROOT, "makani_b200", "libb200sht_umma_prof.so"))
sys.path.insert(0, _ROOT)
import numpy as np, torch, makani_b200 as mb
from makani_b200 import _lib
from makani_b200.sht import _ptr, _stream

dev = torch.device("cuda", 0)
plan = mb.get_plan(721, 1440, 240, 241, "equiangular", True, dev)
B, C = 1, 73
st = _stream(dev)
lib = _lib.load()
gen = torch.Generator(device=dev).manual_seed(0)
lat = torch.randn(plan.latspec_elems(B, C), device=dev, generator=gen)
spec = torch.randn(plan.spec_elems(B, C), device=dev, generator=gen)
out_lat = torch.empty_like(lat)
out_spec = torch.empty_like(spec)
cnt = np.zeros(16, dtype=np.uint64)


def read():
    lib.b200sht_debug_umma_profile(cnt.ctypes.data_as(ctypes.c_void_p))
    return cnt.astype(float)


LAUNCHES = {
    "legendre_analysis": lambda: _lib.call("b200sht_legendre_analysis", plan.handle, _ptr(lat), _ptr(out_spec), B, C, _lib.PREC_TF32, st),
    "legendre_synthesis_tiled": lambda: _lib.call("b200sht_legendre_synthesis_tiled", plan.handle, _ptr(spec), _ptr(out_lat), B, C, st),
    "legendre_synthesis": lambda: _lib.call("b200sht_legendre_synthesis", plan.handle, _ptr(spec), _ptr(out_lat), B, C, _lib.PREC_TF32, st),
}
result = {"device": torch.cuda.get_device_name(0), "library": os.path.basename(os.environ["B200SHT_LIBRARY"])}
print(result["device"], result["library"])
for name, fn in LAUNCHES.items():
    for _ in range(3):
        fn()
    read()
    n = 20
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    a = read() / n
    ctas = a[7]
    warps = 8 * ctas
    life = a[4] / warps   # consumer-warp lifetime (clocks)
    r = {"us_per_launch_profiled": e0.elapsed_time(e1) / n * 1e3, "ctas": ctas, "tiles": a[6] / 8, "cta_lifetime_clk": life,
         "producer_waits_empty": a[0] / ctas / life, "consumers_wait_full": a[1] / warps / life,
         "consumers_mma": a[2] / warps / life, "consumers_epilogue": a[3] / warps / life}
    result[name] = r
    print(f"{name}: {r['us_per_launch_profiled']:.1f} us/launch (profile on), {ctas:.0f} CTAs, {r['tiles']:.0f} tiles, CTA lifetime {life:.0f} clk")
    for k in ("producer_waits_empty", "consumers_wait_full", "consumers_mma", "consumers_epilogue"):
        print(f"  {k:24s} {100 * r[k]:5.1f} % of the CTA lifetime")
if "--json" in sys.argv:
    with open(sys.argv[sys.argv.index("--json") + 1], "w") as f:
        json.dump(result, f, indent=1)

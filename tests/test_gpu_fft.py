"""The CUDA-core longitude FFT (csrc/fft.cu) through the C ABI, element by element, against the fp64 references of tests/fft_ref.py.

Every row of the case table names the kernel route it takes: "T" / "F" for the compile-time plan of its length (synthesis with the
truncated partner spectrum, 2 mmax <= nlon / 2, or with it), 4 / 2 / 1 for the run-time kernels at that many row pairs per CTA.
`row_kernels` expands the route into the `fft_{analysis,synthesis}_{ct,rt}_kernel<...>` instantiations, with the template arguments of
the plan as CT_PLANS lists them, and every row asserts through the profiler that exactly those ran.  tests/test_fft_coverage_cpu.py
checks without a GPU that the rows name every instantiation fft.cu builds, and that each route is the one the dispatch picks.

Each row runs the analysis in modes 0 and 1 and the synthesis in modes 0 and 1 with and without a bias, on random operands:
- outputs are written inside a NaN-sentinel buffer, and nothing outside the written region may change (the analysis leaves the orders
  [mmax, mmax8) of the latspec alone); the analysis writes exact zeros in the latitude padding;
- the synthesis input holds NaN in its latitude padding and in the orders [mmax, mmax8), which it must not read, and arbitrary values in the
  imaginary parts of the DC and Nyquist orders, which it must ignore;
- every element is within the bound of fft_ref: the compile-time kernels with the magnitude of the element's own row, the run-time kernels
  with that of its row pair.
Two exact-operand checks, bit for bit: constant rows of small integers c give order 0 = fl32(N c rs[k]) (mode 0) or N c (mode 1) --
the DC path adds integers and multiplies by the exact twiddle 1 only --, and DC-only spectra give y = fl32(c + bias) (mode 0) or
fl32(c rs[k]) (mode 1), rounded once more to bf16 for a bf16 output.  Every check prints the smallest C_FFT it would pass with (-s)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import engine_ref as E
import fft_ref as F
from makani_b200 import _lib
from makani_b200.quadrature import _grid_np
from makani_b200.sht import Plan, _dtype_code, _ptr, _stream
from test_fft_layout import ct_plans
from test_gpu_engine import SENTINEL, launched_kernels

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F32, BF16 = torch.float32, torch.bfloat16
SENT16 = 0x7FC1   # bf16 quiet NaN with a payload no kernel writes
ERR_INVALID, ERR_UNSUPPORTED = -1, -3   # B200SHT_ERR_INVALID / _UNSUPPORTED (include/b200sht.h)
TESTS = os.path.dirname(os.path.abspath(__file__))
FFT_CU = os.path.join(os.path.dirname(TESTS), "makani_b200", "csrc", "fft.cu")


# --------------------------------------------------------------------------------------------------------- the kernels
CT = {2 * p[3] * p[4] * p[5]: p for p in ct_plans()}


def variant_plan():
    """(nlon, plan) of the B200SHT_FFT_VARIANT=1 switch of dispatch_ct"""
    src = open(FFT_CU).read()
    m = re.search(r"variant == 1 && pl->nlon == (\d+)\) return launch_ct<T, ([\d, ]+)>", src)
    return int(m[1]), tuple(int(v) for v in m[2].split(","))


def rt_pairs(nlon):
    """row pairs per CTA of the run-time kernels (rt_pick_pairs): the most that fit the shared-memory budget, 0 for none"""
    smem = lambda p: 8 * (nlon + 2 * p * (nlon + 1))
    for p, limit in ((4, 110 * 1024), (2, 220 * 1024), (1, 220 * 1024)):
        if smem(p) <= limit:
            return p
    return 0


def dispatch_route(nlon, mmax, off):
    """the route fft.cu takes: the compile-time plan when the length has one and x / y are 16-byte aligned, else the run-time kernels"""
    if off == 0 and nlon in CT:
        return "T" if 2 * mmax <= nlon // 2 else "F"
    return rt_pairs(nlon)


def _tname(dt):
    return "float" if dt == F32 else "__nv_bfloat16"


def row_kernels(row, variant=False):
    """{(direction, family, T, template arguments after T)} that a row launches (a bool argument as 0 / 1)"""
    nlon, dt, route = row[2], row[6], row[8]
    T = _tname(dt)
    if route in ("T", "F"):
        vn, vp = variant_plan()
        plan = vp if variant and nlon == vn else CT[nlon]
        return {("analysis", "ct", T, plan), ("synthesis", "ct", T, plan + (int(route == "T"),))}
    return {("analysis", "rt", T, (route,)), ("synthesis", "rt", T, (route,))}


# the profiler reports b200sht::fft_synthesis_ct_kernel<float, 4, 2, 96, 8, 9, 10, 3, true>; cu++filt may print (int)4, (bool)1
FFT_KERNEL = re.compile(r"fft_(analysis|synthesis)_(ct|rt)_kernel<(?:b200sht::)?(float|__nv_bfloat16), ([^>]*)>")


def _targ(s):
    s = re.sub(r"^\((?:int|bool)\)", "", s.strip())
    return {"true": 1, "false": 0}.get(s) if s in ("true", "false") else int(s)


def fft_kernels(names):
    return {(m[1], m[2], m[3], tuple(_targ(a) for a in m[4].split(","))) for m in map(FFT_KERNEL.search, names) if m}


def assert_ran(tag, fn, want):
    """runs `fn` (idempotent) under the profiler: the FFT instantiations it launches must be exactly `want`, and no DFT kernel"""
    names = launched_kernels(fn, lambda n: fft_kernels(n) == want)
    assert fft_kernels(names) == want and not any("dft_" in n for n in names), f"{tag}: expected {sorted(want)}, launched {names}"


# -------------------------------------------------------------------------------------------------------- the case table
# id, nlat, nlon, mmax, B, C, dtype, offset of x and y in elements, route
def _ct_rows():
    """every CT_PLANS length x {fp32, bf16} x {synthesis T, F}.  1440 and 720 (4- and 8-row tiles) also at the TRUNC boundary
    2 mmax == H and the first non-TRUNC mmax, 2 mmax == H + 2.  The latitude counts cycle through a ragged last tile (13, 9, 17), fewer
    rows than a tile (3, 5) and kp % 16 == 8 (21, 5, 3)."""
    nlats = (13, 3, 21, 9, 17, 5)
    rows, i = [], 0
    for nlon in sorted(CT):
        H = nlon // 2
        mm = ((H // 2, H // 2 + 1, H + 1) if nlon in (1440, 720) else (max(1, H // 3), H + 1))
        for dt in (F32, BF16):
            for mmax in mm:
                nlat = nlats[i % len(nlats)]
                B, C = 1 + i % 2, 2 + i % 3
                i += 1
                route = dispatch_route(nlon, mmax, 0)
                rows.append((f"{nlon}-m{mmax}{route}-{'f32' if dt == F32 else 'bf16'}-nlat{nlat}", nlat, nlon, mmax, B, C, dt, 0, route))
    return rows


ROWS = _ct_rows() + [
    ("1440-headline-f32", 721, 1440, 241, 1, 2, F32, 0, "T"),
    ("1440-headline-bf16", 721, 1440, 241, 1, 2, BF16, 0, "T"),
    # run-time plans: radices 15 / 9 5 / 13 11 7 / 7 6 5 / 12 10 / 4 / 3 (4 pairs), 13 11 7 2 / 16 16 16 (2 pairs), 16 8 8 8 (1 pair)
    ("15-f32", 13, 15, 8, 1, 3, F32, 0, 4),
    ("15-bf16", 21, 15, 5, 2, 2, BF16, 0, 4),
    ("45-f32", 9, 45, 23, 1, 2, F32, 0, 4),
    ("45-bf16", 17, 45, 12, 2, 2, BF16, 0, 4),
    ("1001-f32", 5, 1001, 501, 1, 3, F32, 0, 4),
    ("1001-bf16", 11, 1001, 100, 1, 2, BF16, 0, 4),
    ("210-f32", 17, 210, 106, 1, 2, F32, 0, 4),
    ("120-bf16", 11, 120, 61, 2, 2, BF16, 0, 4),
    ("4-f32", 7, 4, 3, 1, 3, F32, 0, 4),
    ("3-bf16", 6, 3, 2, 2, 2, BF16, 0, 4),
    ("2002-f32", 3, 2002, 1002, 1, 2, F32, 0, 2),
    ("2002-bf16", 10, 2002, 300, 1, 2, BF16, 0, 2),
    ("4096-f32", 9, 4096, 2049, 1, 2, F32, 0, 2),
    ("8192-f32", 5, 8192, 4097, 1, 2, F32, 0, 1),
    ("8192-bf16", 4, 8192, 1000, 1, 2, BF16, 0, 1),
    # compile-time lengths with x and y off the 16-byte boundary: the run-time kernels serve them
    ("1440-xy+4B-f32", 13, 1440, 241, 1, 2, F32, 1, 4),
    ("360-xy+2B-bf16", 21, 360, 181, 1, 3, BF16, 1, 4),
    ("720-xy+8B-f32", 9, 720, 361, 2, 2, F32, 2, 4),
    # B*C = 65535: the gridDim.y limit of the run-time kernels
    ("BC65535-15-f32", 1, 15, 8, 1, 65535, F32, 0, 4),
]
ROW_IDS = [r[0] for r in ROWS]


# ----------------------------------------------------------------------------------------------------------- helpers
_plans = {}


def _plan(nlat, nlon, mmax):
    """an FFT-only plan on the Legendre-Gauss grid (the row scale holds its quadrature weights)"""
    key = (nlat, nlon, mmax)
    if key not in _plans:
        cost, w = _grid_np(nlat, "legendre-gauss")
        _plans[key] = (Plan.create_ex(nlat, nlon, 1, mmax, 0, _lib.PLAN_FFT_ONLY, cost, w, True, DEV), w)
    return _plans[key]


def nstages(nlon):
    """stages of the run-time plan of nlon (b200sht_debug_fft_plan), and its radices"""
    rad = np.zeros(20, dtype=np.int32)
    n = _lib.load().b200sht_debug_fft_plan(nlon, rad.ctypes.data_as(ctypes.c_void_p), 20)
    assert n > 0, nlon
    return n, [int(r) for r in rad[:n]]


def _buf(n, dt, off):
    """(buffer, view): n elements placed `off` elements past a 16-byte boundary inside a NaN sentinel of 16 bytes + off before and 16
    bytes after"""
    pad = 16 // (4 if dt == F32 else 2)
    if dt == F32:
        buf = torch.full((n + 2 * pad + off,), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    else:
        buf = torch.full((n + 2 * pad + off,), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    return buf, buf[pad + off: pad + off + n]


def _untouched_outside(buf, lo, hi):
    bits = buf.view(torch.int32 if buf.dtype == F32 else torch.int16)
    s = SENTINEL if buf.dtype == F32 else SENT16
    return bool((bits[:lo] == s).all() and (bits[hi:] == s).all())


def _place(vals, off):
    """vals [R][nlat][nlon] copied into a NaN-sentinel buffer at `off` elements: reads outside the rows would show as non-finite output"""
    buf, x = _buf(vals.numel(), vals.dtype, off)
    x.copy_(vals.reshape(-1))
    return buf, x


def analysis(plan, x, B, C, mode):
    """b200sht_fft_analysis into a sentinel buffer: the orders [mmax, mmax8) and everything around untouched, the latitude padding exact
    zeros.  Returns the [mmax][2][R][kp] view."""
    R, kp, nlat, mmax = B * C, plan.kp, plan.nlat, plan.mmax
    buf, lat = _buf(plan.latspec_elems(B, C), F32, 0)
    _lib.call("b200sht_fft_analysis", plan.handle, _ptr(x), _dtype_code(x.dtype), B, C, _ptr(lat), mode, _stream(DEV))
    torch.cuda.synchronize()
    n = mmax * 2 * R * kp
    assert _untouched_outside(buf, 4, 4 + n), "analysis: a store outside the orders [0, mmax) of the latspec"
    X = lat[:n].view(mmax, 2, R, kp)
    assert (X[..., nlat:] == 0).all(), "analysis: the latitude padding must hold exact zeros"
    return X


def synthesis(plan, Z, B, C, dt, bias, mode, off):
    """b200sht_fft_synthesis into y placed `off` elements past a 16-byte boundary inside a sentinel buffer; nothing outside y may change.
    Returns y [R][nlat][nlon]."""
    R, nlat, nlon = B * C, plan.nlat, plan.nlon
    n = R * nlat * nlon
    buf, y = _buf(n, dt, off)
    _lib.call("b200sht_fft_synthesis", plan.handle, _ptr(Z), _ptr(y), _dtype_code(dt), B, C, _ptr(bias), mode, _stream(DEV))
    torch.cuda.synchronize()
    pad = 16 // y.element_size()
    assert _untouched_outside(buf, pad + off, pad + off + n), "synthesis: a store outside y"
    return y.view(R, nlat, nlon)


def _complex(X, nlat):
    """[mmax][2][R][kp] -> complex [R][nlat][mmax]"""
    return torch.complex(X[:, 0, :, :nlat], X[:, 1, :, :nlat]).permute(1, 2, 0)


def _check(tag, got, ref, mag, K, r=0.0):
    ratio = E.bound_ratio(got, ref, mag, K, r=r, c=F.C_FFT)
    need = E.needed_c(got, ref, mag, K, r=r)
    print(f"[fft] {tag}: worst ratio {ratio:.3e}, needs c >= {need:.3e} (C_FFT = {F.C_FFT})")
    assert ratio <= 1.0, f"{tag}: outside the bound by {ratio:.3g}x"
    return need


def _latspec_input(plan, B, C, gen, scale=None):
    """random synthesis input [mmax8][2][R][kp]: NaN in the orders [mmax, mmax8) and the latitude padding; `scale` [nlat] per row"""
    R, kp, nlat, mmax = B * C, plan.kp, plan.nlat, plan.mmax
    Z = torch.randn(plan.latspec_elems(B, C), device=DEV, generator=gen).view(-1, 2, R, kp)
    if scale is not None:
        Z[..., :nlat] *= scale
    Z[mmax:] = float("nan")
    Z[..., nlat:] = float("nan")
    return Z


# ------------------------------------------------------------------------------------------------------------ the rows
def run_row(row, variant=False, leak=False):
    """all checks of one case-table row (see the module docstring).  `leak`: latitude rows alternate between scale 1 and 2^-20."""
    rid, nlat, nlon, mmax, B, C, dt, off, route = row
    plan, w = _plan(nlat, nlon, mmax)
    R, kp = B * C, plan.kp
    paired = route not in ("T", "F")
    fam = "rt" if paired else "ct"
    K = F.fft_len(nstages(nlon)[0])
    rs = F.row_scale(w, nlon, kp).to(DEV)
    want = row_kernels(row, variant)
    gen = torch.Generator(device=DEV).manual_seed(7 * nlon + nlat + mmax)
    scale = torch.where(torch.arange(nlat, device=DEV) % 2 == 0, 1.0, 2.0 ** -20)[:, None] if leak else None
    tag = f"{rid}{' variant' if variant else ''}{' leak' if leak else ''}"
    rbf = F.R_BF16 if dt == BF16 else 0.0

    # ---- analysis
    vals = torch.randn(R, nlat, nlon, device=DEV, generator=gen)
    if leak:
        vals = vals * scale
    _, x = _place(vals.to(dt), off)
    xv = x.view(R, nlat, nlon)
    assert_ran(f"{tag} analysis", lambda: analysis(plan, x, B, C, 0), {k for k in want if k[0] == "analysis"})
    for mode in (0, 1):
        got = _complex(analysis(plan, x, B, C, mode), nlat)
        ref, mag = F.analysis_ref(xv, mmax, mode, rs, paired)
        _check(f"{fam} analysis {tag} mode{mode}", got, ref, mag, K)
        if leak and paired:
            _, own = F.analysis_ref(xv, mmax, mode, rs, False)
            print(f"[fft] {fam} analysis {tag} mode{mode}: with the own-row magnitude it would need c >= {E.needed_c(got, ref, own, K):.3e}")
    # constant rows of small integers: order 0 exact
    c = torch.randint(-4, 5, (R, nlat, 1), device=DEV, generator=gen).float()
    _, x = _place(c.expand(R, nlat, nlon).to(dt), off)
    for mode in (0, 1):
        X = analysis(plan, x, B, C, mode)
        dc = (nlon * c[..., 0]) * (rs[None, :nlat] if mode == 0 else 1.0)
        assert torch.equal(X[0, 0, :, :nlat], dc), f"{tag} mode{mode}: order 0 of constant rows is not fl32(N c s)"
        assert (X[0, 1, :, :nlat] == 0).all(), f"{tag} mode{mode}: order 0 of constant rows has an imaginary part"
        ref, mag = F.analysis_ref(x.view(R, nlat, nlon), mmax, mode, rs, paired)
        _check(f"{fam} analysis {tag} constant rows mode{mode}", _complex(X, nlat), ref, mag, K)

    # ---- synthesis
    Z = _latspec_input(plan, B, C, gen, None if scale is None else scale[:, 0])
    bias = torch.randn(C, device=DEV, generator=gen)
    assert_ran(f"{tag} synthesis", lambda: synthesis(plan, Z, B, C, dt, None, 0, off), {k for k in want if k[0] == "synthesis"})
    for mode in (0, 1):
        for b in (None, bias):
            y = synthesis(plan, Z, B, C, dt, b, mode, off)
            ref, mag = F.synthesis_ref(Z[:mmax, :, :, :nlat], nlon, mode, rs, b, C, paired)
            t = f"{fam} synthesis {tag} mode{mode}{' +bias' if b is not None else ''}"
            _check(t, y, ref, mag, K, r=rbf)
            if leak and paired:
                _, own = F.synthesis_ref(Z[:mmax, :, :, :nlat], nlon, mode, rs, b, C, False)
                print(f"[fft] {t}: with the own-row magnitude it would need c >= {E.needed_c(y, ref, own, K, r=rbf):.3e}")
    # DC-only spectra: y exact
    Z = torch.zeros(plan.latspec_elems(B, C), device=DEV).view(-1, 2, R, kp)
    Z[mmax:] = float("nan")
    Z[..., nlat:] = float("nan")
    c = torch.randint(-4, 5, (R, nlat), device=DEV, generator=gen).float()
    Z[0, 0, :, :nlat] = c
    Z[0, 1, :, :nlat] = 3.0   # the imaginary part of the DC order is ignored
    y = synthesis(plan, Z, B, C, dt, bias, 0, off)
    want0 = (c + bias.repeat(B)[:, None]).to(dt)[..., None].expand(R, nlat, nlon)
    assert torch.equal(y, want0), f"{tag}: DC-only synthesis mode 0 is not fl(c + bias)"
    y = synthesis(plan, Z, B, C, dt, None, 1, off)
    want1 = (c * rs[None, :nlat]).to(dt)[..., None].expand(R, nlat, nlon)
    assert torch.equal(y, want1), f"{tag}: DC-only synthesis mode 1 is not fl(c rs[k])"


@pytest.mark.parametrize("row", ROWS, ids=ROW_IDS)
def test_fft_row(row):
    run_row(row)


LEAK_IDS = ("1440-headline-f32", "360-m181F-bf16-nlat5", "1001-f32", "2002-bf16", "1440-xy+4B-f32")


@pytest.mark.parametrize("row", [r for r in ROWS if r[0] in LEAK_IDS], ids=lambda r: r[0])
def test_fft_rows_of_scale_1_and_2e_20(row):
    """alternate rows of scale 1 and 2^-20: the compile-time kernels keep rows apart (own-row bound); the run-time kernels hold the pair
    bound, and the own-row need they print is the two-for-one algorithm's leakage"""
    run_row(row, leak=True)


def test_fft_variant_plan_in_a_child_process():
    """B200SHT_FFT_VARIANT=1 (read once per process): the 1440 rows on 8-row tiles, in a child process"""
    vn, vp = variant_plan()
    ids = [r[0] for r in ROWS if r[2] == vn and r[8] in ("T", "F")]
    assert len(ids) >= 4
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(TESTS)!r}, {TESTS!r}]; import test_gpu_fft as T\n"
            f"for r in T.ROWS:\n    if r[0] in {ids!r}: T.run_row(r, variant=True)\n")
    env = dict(os.environ, B200SHT_FFT_VARIANT="1")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-5000:]
    assert r.stdout.count(" variant") >= len(ids) * 8


# ------------------------------------------------------------------------------------------------- TF32 rounding (scale_mode | 2)
# calls the tensor-core DFT cannot take: fp32 rows with nlon % 32 != 0, mmax > 256, nlon > 1520, x off the 16-byte boundary
TF32_ROWS = [
    ("720-f32", 33, 720, 121, 1, 4, F32, 0, "T"),
    ("360-f32", 45, 360, 100, 1, 4, F32, 0, "F"),
    ("72-f32", 33, 72, 37, 2, 4, F32, 0, "F"),
    ("1440-m300-f32", 40, 1440, 300, 1, 3, F32, 0, "T"),
    ("1024-m400-bf16", 24, 1024, 400, 1, 4, BF16, 0, "F"),
    ("2880-f32", 13, 2880, 241, 1, 4, F32, 0, "T"),
    ("1440-x+4B-f32", 33, 1440, 241, 1, 3, F32, 1, 4),
    ("128-x+2B-bf16", 30, 128, 65, 1, 4, BF16, 1, 4),
]


@pytest.mark.parametrize("row", TF32_ROWS, ids=[r[0] for r in TF32_ROWS])
def test_fft_analysis_tf32(row):
    """the FFT serves these TF32 calls: the stored values are the nearest TF32 values (within 2^-11 of the bound, order 0 of constant
    rows exactly tf32_rna(fl32(N c s))), and the least-squares gain per mode is 1 within 1e-4 (a truncation moves it by about -3e-4)"""
    rid, nlat, nlon, mmax, B, C, dt, off, route = row
    plan, w = _plan(nlat, nlon, mmax)
    R = B * C
    paired = route not in ("T", "F")
    K = F.fft_len(nstages(nlon)[0])
    rs = F.row_scale(w, nlon, plan.kp).to(DEV)
    gen = torch.Generator(device=DEV).manual_seed(nlon + nlat)
    _, x = _place(torch.randn(R, nlat, nlon, device=DEV, generator=gen).to(dt), off)
    assert_ran(f"{rid} tf32", lambda: analysis(plan, x, B, C, 2), {k for k in row_kernels(row) if k[0] == "analysis"})
    for mode in (0, 1):
        X = analysis(plan, x, B, C, mode | 2)
        assert bool(((X.contiguous().view(torch.int32) & 0x1FFF) == 0).all()), f"{rid} mode{mode}: not TF32 values"
        got = _complex(X, nlat)
        ref, mag = F.analysis_ref(x.view(R, nlat, nlon), mmax, mode, rs, paired)
        _check(f"{'rt' if paired else 'ct'} analysis tf32 {rid} mode{mode}", got, ref, mag, K, r=F.R_TF32)
        g, rr = torch.view_as_real(got.to(torch.complex128)), torch.view_as_real(ref)
        gain = float((g * rr).sum() / (rr * rr).sum())
        print(f"[fft] tf32 {rid} mode{mode}: gain 1 {gain - 1:+.2e}")
        assert abs(gain - 1.0) <= 1e-4, f"{rid} mode{mode}: gain 1 {gain - 1:+.3e}"
    c = torch.randint(-4, 5, (R, nlat, 1), device=DEV, generator=gen).float()
    _, x = _place(c.expand(R, nlat, nlon).to(dt), off)
    for mode in (0, 1):
        X = analysis(plan, x, B, C, mode | 2)
        dc = E.tf32_rna((nlon * c[..., 0]) * (rs[None, :nlat] if mode == 0 else 1.0))
        assert torch.equal(X[0, 0, :, :nlat], dc), f"{rid} mode{mode}: order 0 of constant rows is not tf32_rna(fl32(N c s))"


# ---------------------------------------------------------------------------------- persistent CTAs walking many tiles
PERSIST = [(721, 1440, 241, F32), (53, 720, 121, BF16), (53, 2880, 241, F32)]


@pytest.mark.parametrize("nlat,nlon,mmax,dt", PERSIST, ids=[f"{c[1]}-{'f32' if c[3] == F32 else 'bf16'}" for c in PERSIST])
def test_fft_persistent_tiles_bit_identical(nlat, nlon, mmax, dt):
    """enough images that every persistent CTA walks at least three tiles, with a grid that the tiles per image do not divide (the walk
    crosses images mid-grid): every image is bit-identical to its run alone -- the same instantiation on a different grid"""
    rows = CT[nlon][0]
    plan, _ = _plan(nlat, nlon, mmax)
    ntx = -(-plan.kp // rows)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert all((p * sms) % ntx for p in range(1, 5)), "the grid (CTAs per SM x SMs) must not be a multiple of the tiles per image"
    R = -(-12 * sms // ntx) + 1           # >= 3 tiles for each of at most 4 x sms CTAs
    code = _dtype_code(dt)
    st = _stream(DEV)
    gen = torch.Generator(device=DEV).manual_seed(nlon)
    x = torch.randn(R, nlat, nlon, device=DEV, generator=gen).to(dt)
    n = mmax * 2 * R * plan.kp
    for mode in (0, 1):
        lat = torch.full((plan.latspec_elems(1, R),), float("nan"), device=DEV)
        _lib.call("b200sht_fft_analysis", plan.handle, _ptr(x), code, 1, R, _ptr(lat), mode, st)
        X = lat[:n].view(mmax, 2, R, plan.kp)
        one = torch.empty(plan.latspec_elems(1, 1), device=DEV)
        for r in range(R):
            _lib.call("b200sht_fft_analysis", plan.handle, _ptr(x[r]), code, 1, 1, _ptr(one), mode, st)
            if not torch.equal(one[: mmax * 2 * plan.kp].view(mmax, 2, plan.kp).view(torch.int32), X[:, :, r].view(torch.int32)):
                raise AssertionError(f"analysis mode {mode}: image {r} of {R} differs from its run alone")
    Z = torch.randn(mmax, 2, R, plan.kp, device=DEV, generator=gen)
    bias = torch.randn(R, device=DEV, generator=gen)
    for mode in (0, 1):
        y = torch.full((R, nlat, nlon), float("nan"), device=DEV, dtype=dt)
        _lib.call("b200sht_fft_synthesis", plan.handle, _ptr(Z), _ptr(y), code, 1, R, _ptr(bias), mode, st)
        y1 = torch.empty(nlat, nlon, device=DEV, dtype=dt)
        for r in range(R):
            zr = Z[:, :, r: r + 1].contiguous()
            _lib.call("b200sht_fft_synthesis", plan.handle, _ptr(zr), _ptr(y1), code, 1, 1, _ptr(bias[r: r + 1]), mode, st)
            if not torch.equal(y1.view(torch.int16 if dt == BF16 else torch.int32), y[r].view(torch.int16 if dt == BF16 else torch.int32)):
                raise AssertionError(f"synthesis mode {mode}: image {r} of {R} differs from its run alone")


# ------------------------------------------------------------------------------------------------------------- refusals
def test_fft_refusals_launch_nothing():
    """nlon > 9386 (a plan, but no run-time kernel fits shared memory), B*C = 65536 (gridDim.y) and a latspec off the 8-byte boundary
    are refused with an error code, and nothing is launched"""
    lib = _lib.load()
    st = _stream(DEV)
    big, _ = _plan(3, 9600, 8)
    x_big, lat_big = torch.zeros(3 * 9600, device=DEV), torch.zeros(big.latspec_elems(1, 1), device=DEV)
    p15, _ = _plan(1, 15, 8)
    x15, lat15 = torch.zeros(65536 * 15, device=DEV), torch.zeros(p15.latspec_elems(1, 65536), device=DEV)
    odd = []
    for nlon in (1440, 1001):   # a compile-time and a run-time length
        plan, _ = _plan(13, nlon, 100)
        odd.append((nlon, plan, torch.zeros(plan.latspec_elems(1, 2) + 1, device=DEV)[1:], torch.zeros(2 * 13 * nlon, device=DEV)))
    torch.cuda.synchronize()
    rcs = []

    def calls():
        rcs.clear()
        for mode in (0, 1):
            rcs.append(("9600 analysis", lib.b200sht_fft_analysis(big.handle, _ptr(x_big), 0, 1, 1, _ptr(lat_big), mode, st), ERR_UNSUPPORTED))
            rcs.append(("9600 synthesis", lib.b200sht_fft_synthesis(big.handle, _ptr(lat_big), _ptr(x_big), 0, 1, 1, _ptr(None), mode, st), ERR_UNSUPPORTED))
        rcs.append(("B*C=65536 analysis", lib.b200sht_fft_analysis(p15.handle, _ptr(x15), 0, 2, 32768, _ptr(lat15), 0, st), ERR_INVALID))
        rcs.append(("B*C=65536 synthesis", lib.b200sht_fft_synthesis(p15.handle, _ptr(lat15), _ptr(x15), 0, 2, 32768, _ptr(None), 0, st), ERR_INVALID))
        for nlon, plan, lat, y in odd:
            for mode in (0, 1):
                rcs.append((f"{nlon} latspec+4B mode{mode}", lib.b200sht_fft_synthesis(plan.handle, _ptr(lat), _ptr(y), 0, 1, 2, _ptr(None), mode, st),
                            ERR_INVALID))
        torch.cuda.synchronize()

    names = launched_kernels(calls, done=lambda n: True)
    for what, rc, want in rcs:
        assert rc == want, f"{what}: status {rc}, expected {want}"
    assert not names, f"a refused call launched {names}"

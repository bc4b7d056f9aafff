"""GPU tests of the tensor-core longitude DFT (csrc/dft.cu) through the C ABI: b200sht_fft_analysis / _synthesis with the TF32
precision bit (scale_mode | 2) against torch.fft in fp64 -- the semantics of torch_harmonics.RealSHT / InverseRealSHT along
longitude (2 pi rfft(norm="forward")[..., :mmax], irfft(norm="forward"); SURVEY App. A).  Tolerance: TF32 contraction, rtol 1e-3
(BASELINE north_star "1e-3 bf16"); rel-L2 printed and asserted as well."""
import math

import pytest
import torch

import makani_b200 as mb
from makani_b200 import _lib
from oracle import makani_oracle as O
from engine_ref import to_tiled
from test_gpu_parity import close

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (nlat, nlon, mmax, C, dtype): N2/2+1 <= 32 (4 replicas), <= 64 (2 replicas), <= 96; odd N2; Nyquist order present; ragged nlat.
# The tensor-core DFT takes fp32 rows only when nlon % 32 == 0: the other grids run with bf16 rows (test_dft_routing asserts the kernel).
CASES = [
    (64, 128, 65, 8, torch.float32),       # BASELINE cfg 1 grid, all orders incl. Nyquist
    (33, 72, 30, 5, torch.bfloat16),       # N2 = 9 (odd)
    (721, 1440, 241, 3, torch.bfloat16),   # headline grid
    (721, 1440, 241, 2, torch.float32),
    (240, 480, 241, 6, torch.float32),     # interior SFNO grid, all orders
    (240, 480, 241, 5, torch.bfloat16),
    (45, 360, 100, 2, torch.bfloat16),     # N2 = 45 (odd)
    (181, 720, 121, 3, torch.bfloat16),    # N2 = 90: two lane quadrants
    (7, 1512, 256, 2, torch.bfloat16),     # largest supported length class (N2 = 189, odd)
    (19, 16, 9, 3, torch.bfloat16),        # smallest
]


def _latview(lat, plan, B, C, mmax):
    return lat[: mmax * 2 * B * C * plan.kp].view(mmax, 2, B * C, plan.kp)


@pytest.mark.parametrize("nlat,nlon,mmax,C,dtype", CASES)
def test_dft_analysis_gpu(nlat, nlon, mmax, C, dtype):
    torch.manual_seed(333)
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    assert plan.query(8) == 1, "tensor-core DFT not available for this grid"
    B = 2
    x = torch.randn(B, C, nlat, nlon, device=DEV).to(dtype)
    st = mb.sht._stream(x.device)
    for mode in (0, 1):
        lat = torch.full((plan.latspec_elems(B, C),), float("nan"), device=DEV)
        _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(x), mb.sht._dtype_code(dtype), B, C, mb.sht._ptr(lat), mode | 2, st)
        X = _latview(lat, plan, B, C, mmax)
        got = torch.complex(X[:, 0, :, :nlat], X[:, 1, :, :nlat]).permute(1, 2, 0).reshape(B, C, nlat, mmax)
        assert (X[..., nlat:] == 0).all(), "latitude padding must hold exact zeros"
        ref = torch.fft.rfft(x.double().cpu(), dim=-1)[..., :mmax]
        if mode == 0:
            _, w = O.precompute_latitudes(nlat, "equiangular")
            ref = ref * (torch.from_numpy(w) * 2 * math.pi / nlon)[:, None]
        else:
            ms = torch.full((mmax,), 2.0, dtype=torch.float64)
            ms[0] = 1
            if mmax - 1 == nlon // 2:
                ms[-1] = 1
            ref = ref * ms
        rel = close(got, ref, 1e-3, f"dft_analysis mode{mode} {nlat}x{nlon} mmax={mmax} {dtype}")
        assert rel < 6e-4, rel


@pytest.mark.parametrize("nlat,nlon,mmax,C,dtype", CASES)
def test_dft_synthesis_gpu(nlat, nlon, mmax, C, dtype):
    torch.manual_seed(334)
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    assert plan.query(8) == 1
    B = 2
    st = mb.sht._stream(torch.device(DEV))
    Z = torch.randn(mmax, 2, B * C, plan.kp, device=DEV)
    # operands of the kind::tf32 GEMM are TF32 values in the product path (the Legendre epilogue rounds): do the same here
    Z = (Z.view(torch.int32) + 0x1000).bitwise_and(~0x1FFF).view(torch.float32)
    lat = to_tiled(Z)
    assert lat.numel() == plan.latspec_elems(B, C)
    bias = torch.randn(C, device=DEV)
    Zc = torch.complex(Z[:, 0, :, :nlat], Z[:, 1, :, :nlat]).permute(1, 2, 0).reshape(B, C, nlat, mmax).to(torch.complex128).cpu()
    y = torch.full((B, C, nlat, nlon), float("nan"), device=DEV, dtype=dtype)
    _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(lat), mb.sht._ptr(y), mb.sht._dtype_code(dtype), B, C, mb.sht._ptr(bias), 0 | 2, st)
    ref = torch.fft.irfft(Zc, n=nlon, dim=-1, norm="forward") + bias.double().cpu()[None, :, None, None]
    rel = close(y, ref, 1e-3 if dtype == torch.float32 else 4e-3, f"dft_synthesis mode0 {nlat}x{nlon} mmax={mmax} {dtype}")
    assert rel < (6e-4 if dtype == torch.float32 else 3e-3), rel
    # mode 1 = adjoint of the mode-0 analysis: y = rowscale[k] * sum_m Re(Z[m] exp(i m phi))
    y1 = torch.full((B, C, nlat, nlon), float("nan"), device=DEV, dtype=dtype)
    _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(lat), mb.sht._ptr(y1), mb.sht._dtype_code(dtype), B, C, mb.sht._VP(0), 1 | 2, st)
    _, w = O.precompute_latitudes(nlat, "equiangular")
    half = Zc.clone()
    half[..., 1:] *= 0.5
    if mmax - 1 == nlon // 2:
        half[..., -1] *= 2.0
    ref1 = torch.fft.irfft(half, n=nlon, dim=-1, norm="forward") * (torch.from_numpy(w) * 2 * math.pi / nlon)[:, None]
    rel = close(y1, ref1, 1e-3 if dtype == torch.float32 else 4e-3, f"dft_synthesis mode1 {nlat}x{nlon} mmax={mmax} {dtype}")
    assert rel < (6e-4 if dtype == torch.float32 else 3e-3), rel


def test_dft_adjoint_pair_full_size():
    """<A x, Z> = <x, A^T Z> at the headline size (size-independent property): mode-0 analysis against mode-1 synthesis."""
    torch.manual_seed(5)
    nlat, nlon, mmax, B, C = 721, 1440, 241, 1, 4
    plan = mb.get_plan(nlat, nlon, 16, mmax, "equiangular", True, torch.device(DEV))
    st = mb.sht._stream(torch.device(DEV))
    x = torch.randn(B, C, nlat, nlon, device=DEV)
    lat = torch.zeros(plan.latspec_elems(B, C), device=DEV)
    _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(x), 0, B, C, mb.sht._ptr(lat), 0 | 2, st)
    Ax = _latview(lat, plan, B, C, mmax).clone()
    Z = torch.randn(mmax, 2, B * C, plan.kp, device=DEV)
    lat2 = to_tiled(Z)
    y = torch.empty(B, C, nlat, nlon, device=DEV)
    _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(lat2), mb.sht._ptr(y), 0, B, C, mb.sht._VP(0), 1 | 2, st)
    lhs = (Ax[..., :nlat].double() * Z[..., :nlat].double()).sum().item()
    rhs = (x.double() * y.double()).sum().item()
    assert abs(lhs - rhs) <= 2e-3 * max(abs(lhs), abs(rhs), 1.0), (lhs, rhs)


@pytest.mark.parametrize("grid,nlat,nlon,lmax,mmax,B,C", [("equiangular", 64, 128, 64, 65, 1, 8), ("legendre-gauss", 48, 96, 32, 33, 2, 5), ("equiangular", 721, 1440, 240, 241, 1, 3)])
def test_legendre_synthesis_tiled_is_a_relayout(grid, nlat, nlon, lmax, mmax, B, C):
    """b200sht_legendre_synthesis_tiled writes exactly the values of b200sht_legendre_synthesis(TF32) in the tiled layout, with exact
    zeros in the padding orders -- bit-identical (same kernel, different epilogue addressing)."""
    torch.manual_seed(7)
    plan = mb.get_plan(nlat, nlon, lmax, mmax, grid, True, torch.device(DEV))
    assert plan.query(8) == 1
    st = mb.sht._stream(torch.device(DEV))
    sp = torch.randn(plan.spec_elems(B, C), device=DEV)
    std = torch.full((plan.latspec_elems(B, C),), float("nan"), device=DEV)
    til = torch.full((plan.latspec_elems(B, C),), float("nan"), device=DEV)
    _lib.call("b200sht_legendre_synthesis", plan.handle, mb.sht._ptr(sp), mb.sht._ptr(std), B, C, _lib.PREC_TF32, st)
    _lib.call("b200sht_legendre_synthesis_tiled", plan.handle, mb.sht._ptr(sp), mb.sht._ptr(til), B, C, st)
    ref = to_tiled(_latview(std, plan, B, C, mmax))
    assert torch.isfinite(til).all()
    assert torch.equal(til, ref)


# ================================================================================ fp64 references of the factorisation (dft_ref.py)
# Every analysis call asserts the kernel that served it (torch.profiler, CUDA activities); the outputs start as NaN sentinels.
import dft_ref as D
import engine_ref as E
from makani_b200.quadrature import _grid_np
from test_gpu_engine import SENTINEL, launched_kernels, sentinel, untouched

F32, BF16 = torch.float32, torch.bfloat16
SENT16 = 0x7FC1   # bf16 quiet NaN with a payload no kernel writes


def _want_ana_kernel(nlon, dtype):
    N2 = nlon // 8
    return f"dft_analysis_kernel<{'float' if dtype == F32 else '__nv_bfloat16'}, {N2 if N2 in (180, 90, 60) else 0}>"


def _rowscale(nlat, nlon, grid="equiangular"):
    _, w = _grid_np(nlat, grid)
    return torch.from_numpy(w * 2.0 * math.pi / nlon).float()


def _analysis(plan, x, B, C, mode, expect):
    """b200sht_fft_analysis(scale_mode | 2) into a sentinel buffer; asserts the kernel (`expect`), the untouched padding orders
    [mmax, mmax8) and exact zeros in the latitude padding.  Returns the [mmax][2][R][kp] view."""
    mmax, kp, nlat = plan.mmax, plan.kp, plan.nlat
    lat = sentinel(plan.latspec_elems(B, C))
    st = mb.sht._stream(x.device)
    names = launched_kernels(lambda: _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(x), mb.sht._dtype_code(x.dtype), B, C, mb.sht._ptr(lat), mode | 2, st))
    assert any(expect in n for n in names), f"expected {expect}, ran {names}"
    n = mmax * 2 * B * C * kp
    assert untouched(lat[n:]), "the padding orders [mmax, mmax8) must not be written"
    X = lat[:n].view(mmax, 2, B * C, kp)
    assert (X[..., nlat:] == 0).all(), "latitude padding must hold exact zeros"
    return X


def _as_complex(X, nlat):
    """[mmax][2][R][kp] -> complex128 [R][nlat][mmax] on the CPU"""
    return torch.complex(X[:, 0, :, :nlat].double(), X[:, 1, :, :nlat].double()).permute(1, 2, 0).cpu()


def _is_tf32(X):
    return bool(((X.contiguous().view(torch.int32) & 0x1FFF) == 0).all())


# nlat, nlon, mmax, B, C, dtype of the rows: length classes N2 = 180 / 90 / 60 (compile-time kernels) and the run-time kernel with
# fp32 rows (N2 = 16, 32, 156) and bf16 rows in box groups gs = 1 (16), 2 (12), 4 (2, 182), 8 (9, 45, 189); K-blocks 1..3; partner
# boxes (N2 < 31); Nyquist; mmax % 8 != 0; mmax < 8; kp % 16 == 8; nlat < 8
ANA_CASES = [
    (721, 1440, 241, 1, 3, F32), (721, 1440, 241, 1, 3, BF16), (181, 720, 121, 1, 3, BF16), (240, 480, 241, 1, 4, F32),
    (240, 480, 241, 1, 4, BF16), (64, 128, 65, 2, 4, F32), (16, 256, 100, 2, 3, F32), (40, 1248, 189, 1, 3, F32),
    (30, 128, 65, 2, 3, BF16), (24, 96, 5, 2, 5, BF16), (20, 96, 49, 2, 3, BF16), (19, 16, 9, 2, 6, BF16), (12, 1456, 256, 2, 2, BF16),
    (33, 72, 37, 2, 4, BF16), (45, 360, 100, 2, 3, BF16), (7, 1512, 256, 2, 3, BF16),
]
ANA_IDS = [f"{c[0]}x{c[1]}-m{c[2]}-{'f32' if c[5] == F32 else 'bf16'}" for c in ANA_CASES]


def _ana_check(tag, plan, x, X, mode, rs, periodic=False):
    """(a) the per-element bound (rounding model of dft_ref), (d) the rel-L2 of every 16-row tile and of the whole; the stored values
    are TF32.  `periodic`: rows of period N2 with small integers -- exact GEMM operands: no truncation term, and every order
    m != 0 mod 8 an exact zero.  Returns (got, ref)."""
    B_C, nlat, nlon = x.shape
    mmax = plan.mmax
    assert _is_tf32(X), f"{tag}: the stored values must be TF32 values"
    got = _as_complex(X, nlat)
    ref, mag, tmag = D.analysis_ref(x.cpu(), mmax, mode, rs)
    floor = 0.0 if periodic else D.analysis_floor(ref, tmag)
    if periodic:
        nz = torch.arange(mmax) % 8 != 0
        assert (got[..., nz] == 0).all(), f"{tag}: orders m != 0 mod 8 of N2-periodic rows must be exact zeros"
    ratio = E.bound_ratio(got, ref, mag, D.gemm_len(mmax), r=D.R_OUT, c=D.C_DFT, floor=floor)
    need = E.needed_c(got, ref, mag, D.gemm_len(mmax), r=D.R_OUT, floor=floor)
    tiles = [D.rel_l2(got[:, k:k + 16], ref[:, k:k + 16]) for k in range(0, nlat, 16)]
    rel = D.rel_l2(got, ref)
    print(f"[dft] {tag}: worst ratio {ratio:.3e}, needs c >= {need:.3e} (c = {D.C_DFT}); rel-L2 {rel:.3e}, worst 16-row tile {max(tiles):.3e}")
    assert ratio <= 1.0, f"{tag}: outside the bound by {ratio:.3g}x"
    if not periodic:
        assert max(tiles) <= ANA_TILE_REL, f"{tag}: a 16-row tile has rel-L2 {max(tiles):.3e}"
        assert rel <= ANA_REL, f"{tag}: rel-L2 {rel:.3e}"
    return got, ref


ANA_TILE_REL, ANA_REL = 7e-4, 6.5e-4   # about 2x the largest measured (3.2e-4) on an H100 80GB HBM3 at 400 W (DESIGN.md section 5)


@pytest.mark.parametrize("nlat,nlon,mmax,B,C,dtype", ANA_CASES, ids=ANA_IDS)
def test_dft_analysis_bound(nlat, nlon, mmax, B, C, dtype):
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    assert plan.dft_ok
    gen = torch.Generator(device=DEV).manual_seed(nlon + nlat)
    x = torch.randn(B, C, nlat, nlon, device=DEV, generator=gen).to(dtype)
    rs = _rowscale(nlat, nlon)
    for mode in (0, 1):
        X = _analysis(plan, x, B, C, mode, _want_ana_kernel(nlon, dtype))
        _ana_check(f"{nlat}x{nlon} m{mmax} {dtype} mode{mode}", plan, x.view(B * C, nlat, nlon), X, mode, rs)


@pytest.mark.parametrize("nlat,nlon,mmax,B,C,dtype", ANA_CASES, ids=ANA_IDS)
def test_dft_analysis_exact_operands_class0(nlat, nlon, mmax, B, C, dtype):
    """rows of period N2 with small integer values: the radix-8 outputs are exact (8 g for class 0, zeros otherwise), so are the
    compensated-and-truncated GEMM operands, and only fp32 accumulation separates the orders m = 0 mod 8 from the rounded-table
    reference -- every K-block, the halved column N2 / 2, the column-0 patch, the row scale and the mode scales"""
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    N2 = nlon // 8
    gen = torch.Generator(device=DEV).manual_seed(7 * nlon + nlat)
    g = torch.randint(-4, 5, (B, C, nlat, N2), device=DEV, generator=gen).float()
    x = g.repeat(1, 1, 1, 8).to(dtype)
    rs = _rowscale(nlat, nlon)
    for mode in (0, 1):
        X = _analysis(plan, x, B, C, mode, _want_ana_kernel(nlon, dtype))
        _ana_check(f"periodic {nlat}x{nlon} m{mmax} {dtype} mode{mode}", plan, x.view(B * C, nlat, nlon), X, mode, rs, periodic=True)


GAIN_CASES = [(721, 1440, 241, 4, F32), (181, 720, 121, 8, BF16), (240, 480, 241, 8, F32), (64, 128, 65, 32, BF16), (33, 72, 37, 64, BF16),
              (16, 1512, 256, 16, BF16), (40, 1248, 189, 16, F32)]


@pytest.mark.parametrize("nlat,nlon,mmax,C,dtype", GAIN_CASES, ids=[f"{c[1]}-{'f32' if c[4] == F32 else 'bf16'}" for c in GAIN_CASES])
def test_dft_analysis_gain_per_class(nlat, nlon, mmax, C, dtype):
    """(c) the least-squares slope of the stored value against the reference, per class c = m % 8 and mode: 1 within 1e-4.  A
    missing truncation compensation on one class path moves it by about 3.5e-4, storing the scaled value unrounded by +3.3e-4"""
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    gen = torch.Generator(device=DEV).manual_seed(nlon)
    x = torch.randn(1, C, nlat, nlon, device=DEV, generator=gen).to(dtype)
    rs = _rowscale(nlat, nlon)
    for mode in (0, 1):
        X = _analysis(plan, x, 1, C, mode, _want_ana_kernel(nlon, dtype))
        got = _as_complex(X, nlat)
        ref, _, _ = D.analysis_ref(x.view(C, nlat, nlon).cpu(), mmax, mode, rs)
        gains = [D.gain(got[..., c::8], ref[..., c::8]) for c in range(8)]
        print(f"[dft] gain {nlat}x{nlon} {dtype} mode{mode}: " + " ".join(f"{g - 1:+.2e}" for g in gains))
        for c, gn in enumerate(gains):
            assert abs(gn - 1.0) <= 1e-4, f"class {c} mode {mode}: gain 1 {gn - 1:+.3e}"


def test_dft_analysis_routes_to_the_cuda_core_fft():
    """fp32 rows with nlon % 32 != 0 and unaligned rows go to the Stockham FFT, which rounds to nearest TF32"""
    plan = mb.get_plan(33, 72, 16, 37, "equiangular", True, torch.device(DEV))
    st = mb.sht._stream(torch.device(DEV))
    x = torch.randn(2 * 33 * 72 + 1, device=DEV)
    for xv in (x[: 2 * 33 * 72], x[1:]):
        lat = sentinel(plan.latspec_elems(1, 2))
        names = launched_kernels(lambda: _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(xv), 0, 1, 2, mb.sht._ptr(lat), 1 | 2, st))
        assert any("fft_analysis_" in n for n in names) and not any("dft_analysis" in n for n in names), names
        X = lat[: 37 * 2 * 2 * plan.kp].view(37, 2, 2, plan.kp)
        assert _is_tf32(X)
        ref, mag, _ = D.analysis_ref(xv.view(2, 33, 72).cpu(), 37, 1, None, rounded=False)
        assert E.bound_ratio(_as_complex(X, 33), ref, mag, 16, r=E.R_TF32, c=D.C_DFT) <= 1.0


# ------------------------------------------------------------------------------------------------------------ synthesis
# nlat, nlon, mmax, B, C, output dtype: 8-column blocks nblk = 1 .. 12 (worker warps 2 .. 10), output boxes 16 (N2 = 2), 104
# (N2 = 39), 120 (N2 = 45), 256 (N2 = 32, 96), odd N2 (9, 39, 45, 189), Nyquist, mmax % 8 != 0, mmax < 8, nlat < 8.  (The 8-wide box of
# a prime N2 > 32 has no plan: nlon must be 13-smooth.)
SYN_CASES = [
    (19, 16, 9, 2, 3, F32), (33, 72, 37, 2, 3, BF16), (24, 96, 5, 1, 5, F32), (64, 128, 65, 2, 4, BF16), (16, 256, 100, 2, 3, F32),
    (30, 312, 149, 1, 3, BF16), (45, 360, 100, 2, 3, F32), (240, 480, 241, 1, 4, BF16), (181, 720, 121, 1, 3, F32),
    (36, 768, 256, 1, 3, BF16), (721, 1440, 241, 1, 2, F32), (721, 1440, 241, 1, 2, BF16), (7, 1512, 256, 2, 3, F32),
    (12, 1456, 256, 2, 2, BF16),
]


def _synthesis(plan, Z, B, C, dtype, bias, mode):
    """b200sht_fft_synthesis(scale_mode | 2) of the standard latspec Z (tiled here) into y placed 16 bytes inside a sentinel buffer;
    asserts that nothing outside y was written.  Returns y [R][nlat][nlon]."""
    nlat, nlon = plan.nlat, plan.nlon
    n = B * C * nlat * nlon
    pad = 16 // (4 if dtype == F32 else 2)
    if dtype == F32:
        buf = sentinel(n + 2 * pad)
    else:
        buf = torch.full((n + 2 * pad,), SENT16, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    y = buf[pad : pad + n]
    lat = E.to_tiled(Z)
    st = mb.sht._stream(torch.device(DEV))
    # scale_mode | 2 has no other route than dft_synthesis_kernel (an error where the plan has no DFT)
    _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(lat), mb.sht._ptr(y), mb.sht._dtype_code(dtype), B, C, mb.sht._ptr(bias), mode | 2, st)
    torch.cuda.synchronize()
    bits = buf.view(torch.int32 if dtype == F32 else torch.int16)
    s = SENTINEL if dtype == F32 else SENT16
    assert (bits[:pad] == s).all() and (bits[pad + n :] == s).all(), "a store outside y"
    return y.view(B * C, nlat, nlon)


@pytest.mark.parametrize("nlat,nlon,mmax,B,C,dtype", SYN_CASES, ids=[f"{c[0]}x{c[1]}-m{c[2]}-{'f32' if c[5] == F32 else 'bf16'}" for c in SYN_CASES])
def test_dft_synthesis_exact_operands(nlat, nlon, mmax, B, C, dtype):
    """TF32 latspec values (as the Legendre epilogue writes them): every GEMM product is exact, so the kernel may differ from the
    rounded-table reference only by fp32 accumulation and butterflies, + one bf16 rounding (r = 2^-8):  |got - ref| <= r |ref| + c K 2^-24 mag.
    The latitude padding rows of the input hold NaN: they are computed but must not be stored."""
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    assert plan.dft_ok
    R, kp = B * C, plan.kp
    gen = torch.Generator(device=DEV).manual_seed(3 * nlon + nlat)
    Z = E.rand_tf32(mmax, 2, R, kp, device=DEV, generator=gen)
    Z[..., nlat:] = float("nan")
    bias = torch.randn(C, device=DEV, generator=gen)
    rs = _rowscale(nlat, nlon)
    r = 0.0 if dtype == F32 else D.R_BF16
    for mode in (0, 1):
        for b in (None, bias):
            tag = f"{nlat}x{nlon} m{mmax} {dtype} mode{mode}{' +bias' if b is not None else ''}"
            y = _synthesis(plan, Z, B, C, dtype, b, mode)
            ref, mag = D.synthesis_ref(Z[..., :nlat].cpu(), nlon, mode, rs, None if b is None else b.cpu(), C)
            y = y.cpu()
            ratio = E.bound_ratio(y, ref, mag, D.gemm_len(mmax), r=r, c=D.C_DFT)
            need = E.needed_c(y, ref, mag, D.gemm_len(mmax), r=r)
            print(f"[dft] synthesis {tag}: worst ratio {ratio:.3e}, needs c >= {need:.3e} (c = {D.C_DFT})")
            assert ratio <= 1.0, f"{tag}: outside the bound by {ratio:.3g}x"


# --------------------------------------------------------------------------------------- pipeline depth, bit-exact invariance
# Enough images for >= 16 tiles per CTA (analysis: 16-row tiles, synthesis: 8-row tiles) so that every ring wraps many times; a tile's
# arithmetic depends only on its own rows, so the output of each image must be bit-identical to a run of that image alone.
DEEP = [(16, 1440, 121, BF16), (16, 720, 121, BF16), (16, 480, 129, F32), (16, 16, 9, F32), (16, 1512, 128, BF16), (8, 96, 49, BF16),
        (8, 312, 149, BF16)]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("nlat,nlon,mmax,dtype", DEEP, ids=[f"{c[1]}-{'f32' if c[3] == F32 else 'bf16'}" for c in DEEP])
def test_dft_deep_pipeline_bit_exact(nlat, nlon, mmax, dtype):
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    kp = plan.kp
    st = mb.sht._stream(torch.device(DEV))
    code = mb.sht._dtype_code(dtype)
    gen = torch.Generator(device=DEV).manual_seed(nlon)
    # analysis: (kp + 15) // 16 tiles per image
    R = 16 * _sms() // ((kp + 15) // 16) + 3
    x = torch.randn(R, nlat, nlon, device=DEV, generator=gen).to(dtype)
    assert x.numel() * x.element_size() + plan.latspec_elems(R, 1) * 4 < 150e6
    for mode in (0, 1):
        outs = []
        for _ in range(2):
            lat = torch.full((plan.latspec_elems(R, 1),), float("nan"), device=DEV)
            _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(x), code, 1, R, mb.sht._ptr(lat), mode | 2, st)
            outs.append(lat[: mmax * 2 * R * kp].view(mmax, 2, R, kp))
        assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32)), f"mode {mode}: two identical calls differ"
        one = torch.empty(plan.latspec_elems(1, 1), device=DEV)
        for r in range(R):
            _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(x[r]), code, 1, 1, mb.sht._ptr(one), mode | 2, st)
            if not torch.equal(one[: mmax * 2 * kp].view(mmax, 2, kp).view(torch.int32), outs[0][:, :, r].view(torch.int32)):
                raise AssertionError(f"analysis mode {mode}: image {r} of {R} differs from its run alone")
    # synthesis: kp / 8 tiles per image
    R = 16 * _sms() // (kp // 8) + 5
    Z = E.rand_tf32(mmax, 2, R, kp, device=DEV, generator=gen)
    lat = E.to_tiled(Z)
    bias = torch.randn(R, device=DEV, generator=gen)
    assert lat.numel() * 4 + R * nlat * nlon * x.element_size() < 150e6
    ys = []
    for _ in range(2):
        y = torch.full((R, nlat, nlon), float("nan"), device=DEV, dtype=dtype)
        _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(lat), mb.sht._ptr(y), code, 1, R, mb.sht._ptr(bias), 0 | 2, st)
        ys.append(y)
    assert torch.equal(ys[0], ys[1]), "synthesis: two identical calls differ"
    y1 = torch.empty(nlat, nlon, device=DEV, dtype=dtype)
    for r in range(R):
        zr = E.to_tiled(Z[:, :, r : r + 1].contiguous())
        _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(zr), mb.sht._ptr(y1), code, 1, 1, mb.sht._ptr(bias[r : r + 1]), 0 | 2, st)
        if not torch.equal(y1, ys[0][r]):
            raise AssertionError(f"synthesis: image {r} of {R} differs from its run alone")


# ------------------------------------------------------------------------------------------------------ TF32 bias gradient
@pytest.mark.parametrize("one_call", [True, False], ids=["one-call", "autograd"])
def test_spectral_conv_tf32_dbias_gain(one_call):
    """dbias[c] = sum of gy over (b, k, j), read by b200sht_bias_grad from the m = 0 plane of the mode-1 analysis: unbiased at TF32.
    gy rows span binades (log-uniform row scales) so that the truncation averages over them; the gain across channels against the
    fp64 oracle must be 1 within 1e-4 (a stored value scaled by 1 + 2^-10 / 3 gives +3.3e-4)"""
    from oracle import makani_oracle as O

    nlat, nlon, L, M, B, C = 64, 128, 32, 33, 2, 16
    torch.manual_seed(21)
    f = mb.RealSHT(nlat, nlon, L, M, "equiangular", precision="tf32")
    i = mb.InverseRealSHT(nlat, nlon, L, M, "equiangular", precision="tf32")
    conv = mb.SpectralConv(f, i, C, C, operator_type="dhconv", bias=True, precision="tf32").to(DEV)
    conv.one_call = one_call
    x = torch.randn(B, C, nlat, nlon)
    xd = x.to(DEV).requires_grad_(True)
    y, _ = conv(xd)
    gy = torch.exp2(4.0 * torch.rand(B, C, nlat, 1, dtype=torch.float64)) * (1.0 + 0.5 * torch.randn(B, C, nlat, nlon, dtype=torch.float64))
    gy = gy * torch.linspace(0.5, 2.0, C, dtype=torch.float64)[None, :, None, None]
    gy = gy.float()
    plan = f.plan(torch.device(DEV))
    _analysis(plan, gy.to(DEV), B, C, 1, "dft_analysis_kernel<float, 0>")   # the longitude analysis the backward runs on gy
    y.backward(gy.to(DEV))
    of = O.RealSHT(nlat, nlon, L, M, "equiangular", dtype=torch.float64)
    oi = O.InverseRealSHT(nlat, nlon, L, M, "equiangular", dtype=torch.float64)
    w = conv.weight.detach().cpu().to(torch.complex128)
    b64 = conv.bias.detach().cpu().double().requires_grad_(True)
    yr, _ = O.spectral_conv_forward(x.double(), w, of, oi, operator_type="dhconv", bias=b64)
    yr.backward(gy.double())
    got, ref = conv.bias.grad.detach().cpu().double().reshape(-1), b64.grad.reshape(-1)
    gn = D.gain(got, ref)
    print(f"[dft] dbias gain ({'one call' if one_call else 'autograd'}): 1 {gn - 1:+.3e}")
    assert abs(gn - 1.0) <= 1e-4, f"dbias gain 1 {gn - 1:+.3e}"

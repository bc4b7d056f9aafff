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

# (nlat, nlon, mmax, C, dtype): N2/2+1 <= 32 (4 replicas), <= 64 (2 replicas), <= 96; odd N2; Nyquist order present; ragged nlat
CASES = [
    (64, 128, 65, 8, torch.float32),       # BASELINE cfg 1 grid, all orders incl. Nyquist
    (33, 72, 30, 5, torch.float32),        # N2 = 9 (odd)
    (721, 1440, 241, 3, torch.bfloat16),   # headline grid
    (721, 1440, 241, 2, torch.float32),
    (240, 480, 241, 6, torch.float32),     # interior SFNO grid, all orders
    (240, 480, 241, 5, torch.bfloat16),
    (45, 360, 100, 2, torch.bfloat16),     # N2 = 45 (odd)
    (181, 720, 121, 3, torch.float32),     # N2 = 90: two lane quadrants
    (7, 1512, 256, 2, torch.float32),      # largest supported length class (N2 = 189, odd)
    (19, 16, 9, 3, torch.float32),         # smallest
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

"""The vector SHT on the GPU (RealVectorSHT / InverseRealVectorSHT, the b200sht_vector_* / b200sht_vsht_* entry points) against the fp64
oracle (oracle/makani_vector_oracle.py), whose tables and identities are pinned on the CPU in tests/test_vector_sht_cpu.py:

* the modules, forward and both gradients, on the grids makani's vector losses use, at default and truncated (lmax, mmax), fp32 and TF32,
  bf16 input and the 6-D leading shape of VortDivCRPSLoss;
* the stage entry points through ctypes with NaN sentinels: every output entry written, no unwritten stage entry read, l < m inputs ignored;
* 721 x 1440 with the losses' defaults: round trip and the adjoint identity through the modules' backward;
* the cores of GradientCRPSLoss and VortDivCRPSLoss restated in a few lines, value and gradient;
* the refusals: 3 x TF32, a scalar plan in a vector entry and a vector plan in a scalar entry.

TF32 bound: relative L2 against the fp64 oracle.  Measured on an H100 80GB HBM3 at a 700 W power limit, the largest value over the TF32
cases below is 8.5e-4 (the gradient of the forward transform at 32 x 64); the bound leaves a factor of about 2.4."""
import ctypes

import numpy as np
import pytest
import torch

import makani_b200 as mb
from makani_b200 import _lib
from oracle import makani_oracle as O
from oracle import makani_vector_oracle as V
from test_gpu_parity import close

pytestmark = pytest.mark.gpu
DEV = "cuda"
VP = ctypes.c_void_p
TF32_REL_L2 = 2e-3


def _p(t):
    return VP(t.data_ptr())


def _stream():
    return VP(torch.cuda.current_stream(torch.device(DEV)).cuda_stream)


def rel_l2(a, b):
    a = a.detach().to(torch.complex128 if a.is_complex() else torch.float64).cpu()
    b = b.detach().to(a.dtype).cpu()
    assert torch.isfinite(torch.view_as_real(a) if a.is_complex() else a).all()
    return ((a - b).abs().pow(2).sum().sqrt() / b.abs().pow(2).sum().sqrt()).item()


def check(a, b, precision, name):
    if precision == "fp32":
        close(a, b, 1e-5, name)
    else:
        r = rel_l2(a, b)
        print(f"TF32 rel-L2 {name}: {r:.3e}")
        assert r < TF32_REL_L2, (name, r)


def _coeffs(lead, L, M, gen=None):
    c = torch.randn(*lead, 2, L, M, dtype=torch.complex64, generator=gen) * torch.tril(torch.ones(L, M))
    return c


MODULE_CASES = [("equiangular", 32, 64, None, None), ("equiangular", 91, 180, None, None), ("legendre-gauss", 90, 180, None, None),
                ("equiangular", 181, 360, None, None), ("equiangular", 91, 180, 40, 35), ("legendre-gauss", 90, 180, 70, 20)]


@pytest.mark.parametrize("grid,nlat,nlon,lmax,mmax", MODULE_CASES)
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
def test_modules_against_oracle(grid, nlat, nlon, lmax, mmax, precision):
    torch.manual_seed(333)
    vsht = mb.RealVectorSHT(nlat, nlon, lmax, mmax, grid, precision=precision)
    ivsht = mb.InverseRealVectorSHT(nlat, nlon, lmax, mmax, grid, precision=precision)
    L, M = vsht.lmax, vsht.mmax
    ov = V.RealVectorSHT(nlat, nlon, lmax, mmax, grid, dtype=torch.float64)
    oiv = V.InverseRealVectorSHT(nlat, nlon, lmax, mmax, grid, dtype=torch.float64)
    tag = f"{grid} {nlat}x{nlon} L={L} M={M} {precision}"

    x = torch.randn(2, 3, 2, nlat, nlon)
    xd = x.to(DEV).requires_grad_(True)
    xr = x.double().requires_grad_(True)
    c, cr = vsht(xd), ov(xr)
    assert c.shape == (2, 3, 2, L, M) and c.dtype == torch.complex64
    check(c, cr, precision, f"vsht {tag}")
    g = _coeffs((2, 3), L, M)
    c.backward(g.to(DEV))
    cr.backward(g.to(torch.complex128))
    check(xd.grad, xr.grad, precision, f"vsht grad {tag}")

    ci = _coeffs((2, 3), L, M)
    cd = ci.to(DEV).requires_grad_(True)
    cir = ci.to(torch.complex128).requires_grad_(True)
    y, yr = ivsht(cd), oiv(cir)
    assert y.shape == (2, 3, 2, nlat, nlon) and y.dtype == torch.float32
    check(y, yr, precision, f"ivsht {tag}")
    gy = torch.randn(2, 3, 2, nlat, nlon)
    y.backward(gy.to(DEV))
    yr.backward(gy.double())
    check(cd.grad, cir.grad, precision, f"ivsht grad {tag}")


def test_bf16_input_and_6d_shape():
    """VortDivCRPSLoss passes (B, E, Cw / 2, 2, H, W); a bf16 input is transformed as its fp32 value and gets a bf16 gradient"""
    torch.manual_seed(333)
    nlat, nlon = 32, 64
    vsht = mb.RealVectorSHT(nlat, nlon, precision="fp32")
    ivsht = mb.InverseRealVectorSHT(nlat, nlon, precision="fp32")
    ov = V.RealVectorSHT(nlat, nlon, dtype=torch.float64)
    oiv = V.InverseRealVectorSHT(nlat, nlon, dtype=torch.float64)
    x = torch.randn(2, 3, 4, 2, nlat, nlon).to(torch.bfloat16)
    xd = x.to(DEV).requires_grad_(True)
    xr = x.double().requires_grad_(True)
    y, yr = ivsht(vsht(xd)), oiv(ov(xr))
    assert y.shape == x.shape
    close(y, yr, 1e-5, "6-D bf16 round trip")
    gy = torch.randn(x.shape)
    y.backward(gy.to(DEV))
    yr.backward(gy.double())
    assert xd.grad.dtype == torch.bfloat16
    close(xd.grad.float(), xr.grad, 1e-2, "6-D bf16 gradient")


@pytest.mark.parametrize("precision", [_lib.PREC_FP32, _lib.PREC_TF32])
def test_stage_entry_points_with_sentinels(precision):
    """b200sht_vector_legendre_analysis / _synthesis / _synthesis_tiled and the spec converters through ctypes on a plan whose stacked table
    puts a 128-row tile across the D / Q split (lmax 91), with ragged K (91 rows), ragged columns (C = 3) and orders past 32; nlon = 192 is
    on the tensor-core DFT's grid list, so the TF32 case also runs the tiled synthesis"""
    torch.manual_seed(333)
    lib = _lib.load()
    grid, nlat, nlon, L, M, B, C = "equiangular", 91, 192, 91, 91, 2, 3
    plan = mb.get_plan(nlat, nlon, L, M, grid, True, torch.device(DEV), vector=True)
    assert plan.vector and plan.query(9) == 1 and plan.lmax == L and plan.query(2) == L
    st = _stream()
    ov = V.RealVectorSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    oiv = V.InverseRealVectorSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    nspec = int(lib.b200sht_spec_elems(plan.handle, B, 2 * C))
    assert nspec == 2 * L * M * 2 * B * 8
    tol = 1e-5 if precision == _lib.PREC_FP32 else None
    cmp = (lambda a, b, n: close(a, b, tol, n)) if tol else (lambda a, b, n: check(a, b, "tf32", n))

    # analysis: fft_analysis of the 2C component rows in place, Legendre analysis into a NaN-filled stacked spec, unpack into NaN-filled coeffs
    x = torch.randn(B, C, 2, nlat, nlon)
    lat = torch.empty(int(lib.b200sht_latspec_elems(plan.handle, B, 2 * C)), device=DEV)
    spec = torch.full((nspec,), float("nan"), device=DEV)
    coeffs = torch.full((B, C, 2, L, M), float("nan"), dtype=torch.complex64, device=DEV)
    _lib.check(lib.b200sht_fft_analysis(plan.handle, _p(x.to(DEV)), _lib.F32, B, 2 * C, _p(lat), 2 if precision == _lib.PREC_TF32 else 0, st), "fft")
    _lib.check(lib.b200sht_vector_legendre_analysis(plan.handle, _p(lat), _p(spec), B, C, precision, st), "vector_legendre_analysis")
    _lib.check(lib.b200sht_vector_spec_unpack(plan.handle, _p(spec), _p(coeffs), B, C, 1, st), "vector_spec_unpack")
    cmp(coeffs, ov(x.double()), "stage analysis")

    # synthesis: coefficients with NaN in every l < m entry (never read), packed into a NaN-filled spec (every entry the kernels read is written)
    cin = _coeffs((B, C), L, M)
    cin_nan = cin + torch.triu(torch.full((L, M), float("nan")), 1).to(torch.complex64)
    spec.fill_(float("nan"))
    _lib.check(lib.b200sht_vector_spec_pack(plan.handle, _p(cin_nan.to(DEV)), _p(spec), B, C, 0, st), "vector_spec_pack")
    yref = oiv(cin.to(torch.complex128))
    lat.fill_(float("nan"))
    y = torch.full((B, C, 2, nlat, nlon), float("nan"), device=DEV)
    _lib.check(lib.b200sht_vector_legendre_synthesis(plan.handle, _p(spec), _p(lat), B, C, precision, st), "vector_legendre_synthesis")
    _lib.check(lib.b200sht_fft_synthesis(plan.handle, _p(lat), _p(y), _lib.F32, B, 2 * C, VP(0), 0, st), "fft_synthesis")
    cmp(y, yref, "stage synthesis")
    if precision == _lib.PREC_TF32:
        assert plan.dft_ok
        lat.fill_(float("nan"))
        y.fill_(float("nan"))
        _lib.check(lib.b200sht_vector_legendre_synthesis_tiled(plan.handle, _p(spec), _p(lat), B, C, st), "vector_legendre_synthesis_tiled")
        _lib.check(lib.b200sht_fft_synthesis(plan.handle, _p(lat), _p(y), _lib.F32, B, 2 * C, VP(0), 2, st), "fft_synthesis tiled")
        cmp(y, yref, "stage synthesis tiled")


def test_plan_tables_and_sharing():
    nlat, nlon, L, M = 46, 90, 40, 30
    v = mb.RealVectorSHT(nlat, nlon, L, M, precision="fp32")
    iv = mb.InverseRealVectorSHT(nlat, nlon, L, M, precision="fp32")
    p = v.plan(torch.device(DEV))
    assert p is iv.plan(torch.device(DEV)) and p is not mb.get_plan(nlat, nlon, L, M, "equiangular", True, DEV)
    assert p.query(5) == 2 * M * L * p.kp * 4
    t = p.table().cpu().double()
    theta, _ = O.precompute_latitudes(nlat, "equiangular")
    D, Q = V.vector_legpoly(M, L, theta)
    for got, ref in ((t[0, ..., :nlat], D), (t[1, ..., :nlat], Q)):
        ref = torch.from_numpy(ref)
        assert ((got - ref).abs() <= 2 ** -23 * ref.abs() + 1e-6 * ref.abs().max()).all()
    assert not t[..., nlat:].any()


def test_every_c_entry_point_through_ctypes():
    """b200sht_vsht_workspace_bytes / _forward / _inverse / _forward_adjoint / _inverse_adjoint with plain pointers against the oracle"""
    torch.manual_seed(333)
    lib = _lib.load()
    grid, nlat, nlon, L, M, B, C = "legendre-gauss", 48, 96, 40, 41, 2, 5
    plan = mb.get_plan(nlat, nlon, L, M, grid, True, torch.device(DEV), vector=True)
    ws = torch.empty(int(lib.b200sht_vsht_workspace_bytes(plan.handle, B, C)), dtype=torch.uint8, device=DEV)
    assert lib.b200sht_vsht_workspace_bytes(mb.get_plan(nlat, nlon, L, M, grid, True, DEV).handle, B, C) == -1
    ov = V.RealVectorSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    oiv = V.InverseRealVectorSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    st, P = _stream(), _lib.PREC_FP32

    x = torch.randn(B, C, 2, nlat, nlon)
    xr = x.double().requires_grad_(True)
    cref = ov(xr)
    coeffs = torch.full((B, C, 2, L, M), float("nan"), dtype=torch.complex64, device=DEV)
    _lib.check(lib.b200sht_vsht_forward(plan.handle, _p(x.to(DEV)), _lib.F32, B, C, _p(coeffs), _p(ws), P, st), "vsht_forward")
    close(coeffs, cref, 1e-5, "b200sht_vsht_forward")
    gc = _coeffs((B, C), L, M)
    cref.backward(gc.to(torch.complex128))
    gx = torch.full((B, C, 2, nlat, nlon), float("nan"), device=DEV)
    _lib.check(lib.b200sht_vsht_forward_adjoint(plan.handle, _p(gc.to(DEV)), _p(gx), _lib.F32, B, C, _p(ws), P, st), "vsht_forward_adjoint")
    close(gx, xr.grad, 1e-5, "b200sht_vsht_forward_adjoint")

    cin = _coeffs((B, C), L, M)
    cr = cin.to(torch.complex128).requires_grad_(True)
    yref = oiv(cr)
    y = torch.full((B, C, 2, nlat, nlon), float("nan"), device=DEV)
    _lib.check(lib.b200sht_vsht_inverse(plan.handle, _p(cin.to(DEV)), _p(y), _lib.F32, B, C, _p(ws), P, st), "vsht_inverse")
    close(y, yref, 1e-5, "b200sht_vsht_inverse")
    gy = torch.randn(B, C, 2, nlat, nlon)
    yref.backward(gy.double())
    gcoef = torch.full((B, C, 2, L, M), float("nan"), dtype=torch.complex64, device=DEV)
    _lib.check(lib.b200sht_vsht_inverse_adjoint(plan.handle, _p(gy.to(DEV)), _lib.F32, B, C, _p(gcoef), _p(ws), P, st), "vsht_inverse_adjoint")
    close(gcoef, cr.grad, 1e-5, "b200sht_vsht_inverse_adjoint")


def test_refusals():
    lib = _lib.load()
    nlat, nlon, B, C = 32, 64, 1, 2
    vplan = mb.get_plan(nlat, nlon, 32, 33, "equiangular", True, torch.device(DEV), vector=True)
    splan = mb.get_plan(nlat, nlon, 32, 33, "equiangular", True, torch.device(DEV))
    x = torch.zeros(B, C, 2, nlat, nlon, device=DEV)
    coeffs = torch.zeros(B, C, 2, 32, 33, dtype=torch.complex64, device=DEV)
    ws = torch.empty(int(lib.b200sht_vsht_workspace_bytes(vplan.handle, B, C)), dtype=torch.uint8, device=DEV)
    st = _stream()
    assert lib.b200sht_vsht_forward(vplan.handle, _p(x), _lib.F32, B, C, _p(coeffs), _p(ws), _lib.PREC_FP32X3, st) == -3
    assert lib.b200sht_vsht_inverse(vplan.handle, _p(coeffs), _p(x), _lib.F32, B, C, _p(ws), _lib.PREC_FP32X3, st) == -3
    assert lib.b200sht_vsht_forward(splan.handle, _p(x), _lib.F32, B, C, _p(coeffs), _p(ws), _lib.PREC_FP32, st) == -1
    assert lib.b200sht_vector_legendre_analysis(splan.handle, _p(ws), _p(ws), B, C, _lib.PREC_FP32, st) == -1
    assert lib.b200sht_sht_forward(vplan.handle, _p(x), _lib.F32, B, C, _p(coeffs), _p(ws), _lib.PREC_FP32, st) == -1
    assert lib.b200sht_legendre_analysis(vplan.handle, _p(ws), _p(ws), B, C, _lib.PREC_FP32, st) == -1
    assert lib.b200sht_legendre_synthesis(vplan.handle, _p(ws), _p(ws), B, C, _lib.PREC_FP32, st) == -1
    assert lib.b200sht_legendre_synthesis_tiled(vplan.handle, _p(ws), _p(ws), B, C, st) == -1
    with pytest.raises(_lib.B200ShtError):
        mb.RealVectorSHT(nlat, nlon, precision="fp32x3")(x)
    with pytest.raises(_lib.B200ShtError):
        mb.InverseRealVectorSHT(nlat, nlon, precision="fp32x3")(coeffs)
    torch.cuda.synchronize()


def test_full_resolution_round_trip_and_adjoint():
    """721 x 1440 with the losses' defaults (lmax = 721, mmax = 721): band-limited round trip, and <A x, y> = <x, A^T y> for both modules"""
    torch.manual_seed(333)
    nlat, nlon = 721, 1440
    vsht = mb.RealVectorSHT(nlat, nlon, precision="fp32")
    ivsht = mb.InverseRealVectorSHT(nlat, nlon, precision="fp32")
    L, M = vsht.lmax, vsht.mmax
    c = _coeffs((1, 2), L, M)
    c[..., 300:, :] = 0      # band limit well inside what the equiangular quadrature integrates exactly
    c[..., 0, :] = 0
    c[..., 0] = c[..., 0].real
    cd = c.to(DEV)
    back = vsht(ivsht(cd))
    assert rel_l2(back, cd) < 1e-4

    x = torch.randn(1, 2, 2, nlat, nlon, device=DEV, requires_grad=True)
    y = _coeffs((1, 2), L, M).to(DEV)
    lhs = (vsht(x) * y.conj()).real.sum()
    lhs.backward()
    rhs = (x.detach().double() * x.grad.double()).sum()
    assert abs(lhs.item() - rhs.item()) < 1e-4 * abs(rhs.item()), (lhs.item(), rhs.item())

    cx = _coeffs((1, 2), L, M).to(DEV).requires_grad_(True)
    yy = torch.randn(1, 2, 2, nlat, nlon, device=DEV)
    lhs = (ivsht(cx) * yy).sum()
    lhs.backward()
    rhs = (cx.detach().to(torch.complex128).conj() * cx.grad.to(torch.complex128)).real.sum()
    assert abs(lhs.item() - rhs.item()) < 1e-4 * abs(rhs.item()), (lhs.item(), rhs.item())


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5)])
def test_gradient_loss_core(precision, tol):
    """GradientCRPSLoss (base_loss.py:518-565): |ivsht([sht(f), 0])|, the magnitude of the surface gradient of every channel"""
    torch.manual_seed(333)
    nlat, nlon = 32, 64
    sht = mb.RealSHT(nlat, nlon, precision=precision)
    ivsht = mb.InverseRealVectorSHT(nlat, nlon, precision=precision)
    osht = O.RealSHT(nlat, nlon, dtype=torch.float64)
    oivsht = V.InverseRealVectorSHT(nlat, nlon, dtype=torch.float64)

    def core(s, iv, f):
        c = s(f)
        g = iv(torch.stack([c, torch.zeros_like(c)], dim=-3))
        return torch.sqrt(g[..., 0, :, :].square() + g[..., 1, :, :].square() + 1e-12)

    f = torch.randn(2, 4, 3, nlat, nlon)
    fd = f.to(DEV).requires_grad_(True)
    fr = f.double().requires_grad_(True)
    v, vr = core(sht, ivsht, fd), core(osht, oivsht, fr)
    close(v, vr, tol, "gradient magnitude")
    w = torch.randn(v.shape)
    (v * w.to(DEV)).sum().backward()
    (vr * w.double()).sum().backward()
    close(fd.grad, fr.grad, 10 * tol, "gradient magnitude, d/df")


def test_vort_div_loss_core():
    """VortDivCRPSLoss (base_loss.py:427-469): the u / v channels go through isht(vsht(.)) as (B, E, Cw / 2, 2, H, W) and are written back
    with index_copy"""
    torch.manual_seed(333)
    nlat, nlon, B, E, C = 32, 64, 2, 3, 7
    wind = torch.tensor([1, 2, 4, 5])            # two u / v pairs
    vsht, ivsht = mb.RealVectorSHT(nlat, nlon, precision="fp32"), mb.InverseRealVectorSHT(nlat, nlon, precision="fp32")
    ov, oiv = V.RealVectorSHT(nlat, nlon, dtype=torch.float64), V.InverseRealVectorSHT(nlat, nlon, dtype=torch.float64)

    def core(vs, iv, x):
        u = x.index_select(2, wind.to(x.device)).reshape(B, E, len(wind) // 2, 2, nlat, nlon)
        y = iv(vs(u)).reshape(B, E, len(wind), nlat, nlon).to(x.dtype)
        return x.index_copy(2, wind.to(x.device), y)

    x = torch.randn(B, E, C, nlat, nlon)
    xd = x.to(DEV).requires_grad_(True)
    xr = x.double().requires_grad_(True)
    y, yr = core(vsht, ivsht, xd), core(ov, oiv, xr)
    close(y, yr, 1e-5, "vort/div round trip")
    w = torch.randn(y.shape)
    (y * w.to(DEV)).square().sum().backward()
    (yr * w.double()).square().sum().backward()
    close(xd.grad, xr.grad, 1e-5, "vort/div gradient")

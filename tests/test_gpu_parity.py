"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Tolerances (BASELINE.json north_star): fp32 path rtol 1e-5, TF32 / bf16 path rtol 1e-3.  `close()` below is
`torch.allclose`-style: |a - b| <= atol + rtol * |b| with atol = rtol * max|b| (sums over ~1e3 quadrature points cancel,
so a purely relative element-wise bound is not meaningful; the reference's own compare_tensors uses atol = rtol too).
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

import makani_b200 as mb
from makani_b200 import _lib
from makani_b200.sht import _SpecPack, _SpecUnpack
from oracle import makani_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden", "contractions_golden.npz")
DEV = "cuda"


def close(a, b, rtol, name=""):
    a = a.detach().double().cpu() if not a.is_complex() else a.detach().to(torch.complex128).cpu()
    b = b.detach().double().cpu() if not b.is_complex() else b.detach().to(torch.complex128).cpu()
    assert a.shape == b.shape, (name, a.shape, b.shape)
    assert torch.isfinite(torch.view_as_real(a) if a.is_complex() else a).all(), f"{name}: non-finite values"
    scale = b.abs().max().item()
    err = (a - b).abs()
    bound = rtol * scale + rtol * b.abs()
    rel_l2 = ((a - b).abs().pow(2).sum().sqrt() / b.abs().pow(2).sum().sqrt().clamp_min(1e-300)).item()
    worst = (err / bound.clamp_min(1e-300)).max().item()
    print(f"[parity] {name}: rel_l2={rel_l2:.3e} max_err/bound={worst:.3f} (rtol={rtol:g}, scale={scale:.3e})")
    assert worst <= 1.0, f"{name}: max err/bound {worst:.3f}, rel_l2 {rel_l2:.3e}"
    return rel_l2


def oracle_pair(nlat_i, nlon_i, nlat_o, nlon_o, lmax, mmax, grid_i, grid_o, dtype=torch.float64):
    return (O.RealSHT(nlat_i, nlon_i, lmax, mmax, grid_i, dtype=dtype), O.InverseRealSHT(nlat_o, nlon_o, lmax, mmax, grid_o, dtype=dtype))


# ------------------------------------------------------------------------------------------------ stages
@pytest.mark.parametrize("grid,nlat,nlon,lmax,mmax", [("equiangular", 33, 64, 20, 21), ("legendre-gauss", 48, 96, 48, 49), ("equiangular", 721, 1440, 240, 241)])
def test_device_table_matches_oracle(grid, nlat, nlon, lmax, mmax):
    plan = mb.get_plan(nlat, nlon, lmax, mmax, grid, True, torch.device(DEV))
    tab = plan.table().cpu().numpy()
    th, _ = O.precompute_latitudes(nlat, grid)
    ref = O.legpoly(mmax, lmax, np.cos(th))
    assert np.abs(tab[:, :, :nlat] - ref).max() < 5e-6
    assert (tab[:, :, nlat:] == 0).all()


@pytest.mark.parametrize("nlat,nlon,mmax,C,dtype", [(64, 128, 65, 8, torch.float32), (33, 72, 30, 5, torch.float32), (721, 1440, 241, 3, torch.bfloat16),
                                                    (240, 480, 241, 6, torch.float32), (45, 360, 100, 2, torch.bfloat16), (19, 2 * 7 * 11 * 13, 50, 2, torch.float32)])
def test_fft_stages(nlat, nlon, mmax, C, dtype):
    torch.manual_seed(333)
    lib = _lib.load()
    plan = mb.get_plan(nlat, nlon, min(nlat, 16), mmax, "equiangular", True, torch.device(DEV))
    B = 2
    x = torch.randn(B, C, nlat, nlon, device=DEV).to(dtype)
    lat = torch.full((plan.latspec_elems(B, C),), float("nan"), device=DEV)
    st = mb.sht._stream(x.device)
    for mode in (0, 1):
        _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(x), mb.sht._dtype_code(dtype), B, C, mb.sht._ptr(lat), mode, st)
        X = lat[: mmax * 2 * B * C * plan.kp].view(mmax, 2, B * C, plan.kp)
        got = torch.complex(X[:, 0, :, :nlat], X[:, 1, :, :nlat]).permute(1, 2, 0).reshape(B, C, nlat, mmax)
        assert (X[..., nlat:] == 0).all()
        ref = torch.fft.rfft(x.double().cpu(), dim=-1)[..., :mmax]
        if mode == 0:
            _, w = O.precompute_latitudes(nlat, "equiangular")
            ref = ref * (torch.from_numpy(w) * 2 * math.pi / nlon)[:, None]
        else:
            ms = torch.full((mmax,), 2.0, dtype=torch.float64)
            ms[0] = 1
            if mmax - 1 == nlon // 2 and nlon % 2 == 0:
                ms[-1] = 1
            ref = ref * ms
        close(got, ref, 2e-6, f"fft_analysis mode{mode} {nlat}x{nlon} {dtype}")
    # synthesis: irfft semantics (mode 0) and the adjoint of the mode-0 analysis (mode 1, checked through <Ax,y> = <x,A^T y>)
    Z = torch.randn(mmax, 2, B * C, plan.kp, device=DEV)
    y = torch.empty(B, C, nlat, nlon, device=DEV, dtype=dtype)
    bias = torch.randn(C, device=DEV)
    _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(Z), mb.sht._ptr(y), mb.sht._dtype_code(dtype), B, C, mb.sht._ptr(bias), 0, st)
    Zc = torch.complex(Z[:, 0, :, :nlat], Z[:, 1, :, :nlat]).permute(1, 2, 0).reshape(B, C, nlat, mmax).to(torch.complex128).cpu()
    ref = torch.fft.irfft(Zc, n=nlon, dim=-1, norm="forward") + bias.double().cpu()[None, :, None, None]
    close(y, ref, 2e-6 if dtype == torch.float32 else 4e-3, f"fft_synthesis mode0 {nlat}x{nlon} {dtype}")
    if dtype == torch.float32:
        _lib.call("b200sht_fft_synthesis", plan.handle, mb.sht._ptr(Z), mb.sht._ptr(y), 0, B, C, mb.sht._VP(0), 1, st)
        _lib.call("b200sht_fft_analysis", plan.handle, mb.sht._ptr(x), 0, B, C, mb.sht._ptr(lat), 0, st)
        lhs = (lat[: mmax * 2 * B * C * plan.kp].view(mmax, 2, B * C, plan.kp)[..., :nlat].double() * Z[..., :nlat].double()).sum().item()
        rhs = (x.double() * y.double()).sum().item()
        assert abs(lhs - rhs) <= 1e-5 * max(abs(lhs), abs(rhs), 1.0), (lhs, rhs)


# --------------------------------------------------------------------------------- RealSHT / InverseRealSHT
SHT_CASES = [
    ("equiangular", 64, 128, None, None, 1, 8),       # BASELINE configs[0]
    ("legendre-gauss", 48, 96, 32, 33, 2, 5),
    ("equiangular", 91, 180, 91, 91, 1, 3),           # odd nlat, reference distributed-test shape
    ("legendre-gauss", 240, 480, 240, 241, 1, 4),     # SFNO inner grid
    ("equiangular", 721, 1440, 240, 241, 1, 2),       # SFNO outer grid
]


@pytest.mark.parametrize("grid,nlat,nlon,lmax,mmax,B,C", SHT_CASES)
def test_real_sht_forward_inverse_fp32(grid, nlat, nlon, lmax, mmax, B, C):
    torch.manual_seed(333)
    sht = mb.RealSHT(nlat, nlon, lmax, mmax, grid, precision="fp32").to(DEV)
    isht = mb.InverseRealSHT(nlat, nlon, sht.lmax, sht.mmax, grid, precision="fp32").to(DEV)
    osht, oisht = oracle_pair(nlat, nlon, nlat, nlon, sht.lmax, sht.mmax, grid, grid)
    x = torch.randn(B, C, nlat, nlon)
    c = sht(x.to(DEV))
    assert c.dtype == torch.complex64 and c.shape == (B, C, sht.lmax, sht.mmax)
    cref = osht(x.double())
    close(c, cref, 1e-5, f"RealSHT {grid} {nlat}x{nlon}")
    L, M = sht.lmax, sht.mmax
    mask = torch.triu(torch.ones(L, M, dtype=torch.bool), diagonal=1)
    assert (c.cpu()[..., mask] == 0).all(), "entries with l < m must be exactly zero"
    cin = torch.randn(B, C, L, M, dtype=torch.complex64)
    y = isht(cin.to(DEV))
    close(y, oisht(cin.to(torch.complex128)), 1e-5, f"InverseRealSHT {grid} {nlat}x{nlon}")


def test_real_sht_leading_dims_and_bf16():
    torch.manual_seed(333)
    sht = mb.RealSHT(32, 64, 20, 21, "legendre-gauss", precision="fp32")
    osht = O.RealSHT(32, 64, 20, 21, "legendre-gauss", dtype=torch.float64)
    x = torch.randn(3, 32, 64)
    close(sht(x.to(DEV)), osht(x.double()), 1e-5, "3-d input")
    x5 = torch.randn(2, 2, 3, 32, 64)
    close(sht(x5.to(DEV)), osht(x5.double()), 1e-5, "5-d input")
    xb = torch.randn(1, 4, 32, 64).bfloat16()
    close(sht(xb.to(DEV)), osht(xb.double()), 1e-5, "bf16 input (exact bf16 values, fp32 arithmetic)")


@pytest.mark.parametrize("grid,nlat,nlon,lmax,mmax,B,C", SHT_CASES[:3])
def test_sht_gradients_fp32(grid, nlat, nlon, lmax, mmax, B, C):
    """Backward of both transforms against CPU autograd through the oracle (PyTorch complex-gradient convention)."""
    torch.manual_seed(333)
    sht = mb.RealSHT(nlat, nlon, lmax, mmax, grid, precision="fp32")
    isht = mb.InverseRealSHT(nlat, nlon, sht.lmax, sht.mmax, grid, precision="fp32")
    osht, oisht = oracle_pair(nlat, nlon, nlat, nlon, sht.lmax, sht.mmax, grid, grid)
    x = torch.randn(B, C, nlat, nlon)
    gc = torch.randn(B, C, sht.lmax, sht.mmax, dtype=torch.complex64)
    xd = x.to(DEV).requires_grad_(True)
    sht(xd).backward(gc.to(DEV))
    xr = x.double().requires_grad_(True)
    osht(xr).backward(gc.to(torch.complex128))
    close(xd.grad, xr.grad, 1e-5, f"dRealSHT/dx {grid} {nlat}x{nlon}")
    cin = torch.randn(B, C, sht.lmax, sht.mmax, dtype=torch.complex64)
    gy = torch.randn(B, C, nlat, nlon)
    cd = cin.to(DEV).requires_grad_(True)
    isht(cd).backward(gy.to(DEV))
    cr = cin.to(torch.complex128).requires_grad_(True)
    oisht(cr).backward(gy.double())
    L, M = sht.lmax, sht.mmax
    keep = torch.tril(torch.ones(L, M)).bool()  # the oracle's gradient for l < m is P = 0 -> exactly zero as well
    close(cd.grad * keep.to(DEV), cr.grad * keep, 1e-5, f"dInverseRealSHT/dc {grid} {nlat}x{nlon}")


# ----------------------------------------------------------------------------------------- SpectralConv
CONV_CASES = [
    # nlat_i nlon_i grid_i        nlat_o nlon_o grid_o          lmax mmax B Cin Cout G  op         sep   bias
    (48, 96, "legendre-gauss", 48, 96, "legendre-gauss", 32, 33, 2, 8, 8, 1, "dhconv", False, True),
    (65, 128, "equiangular", 48, 96, "legendre-gauss", 32, 33, 1, 6, 10, 2, "dhconv", False, True),     # scale_residual, groups
    (48, 96, "legendre-gauss", 65, 128, "equiangular", 40, 41, 1, 73, 73, 1, "dhconv", False, False),   # odd channel count
    (32, 64, "legendre-gauss", 32, 64, "legendre-gauss", 20, 21, 2, 6, 6, 1, "diagonal", False, False),
    (32, 64, "legendre-gauss", 32, 64, "legendre-gauss", 20, 21, 2, 6, 6, 2, "dhconv", True, False),
    (32, 64, "legendre-gauss", 32, 64, "legendre-gauss", 20, 21, 1, 5, 5, 1, "diagonal", True, True),
]


def _run_conv_case(case, precision, rtol, act_dtype=torch.float32):
    (nlat_i, nlon_i, grid_i, nlat_o, nlon_o, grid_o, lmax, mmax, B, Cin, Cout, G, op, sep, bias) = case
    torch.manual_seed(333)
    f = mb.RealSHT(nlat_i, nlon_i, lmax, mmax, grid_i, precision=precision)
    i = mb.InverseRealSHT(nlat_o, nlon_o, lmax, mmax, grid_o, precision=precision)
    conv = mb.SpectralConv(f, i, Cin, Cout, num_groups=G, operator_type=op, separable=sep, bias=bias, precision=precision).to(DEV)
    if bias:
        with torch.no_grad():
            conv.bias.copy_(torch.randn_like(conv.bias))
    of, oi = oracle_pair(nlat_i, nlon_i, nlat_o, nlon_o, lmax, mmax, grid_i, grid_o)
    x = torch.randn(B, Cin, nlat_i, nlon_i).to(act_dtype)
    xd = x.to(DEV).requires_grad_(True)
    y, res = conv(xd)
    assert y.dtype == act_dtype and y.shape == (B, Cout, nlat_o, nlon_o)
    w64 = conv.weight.detach().cpu().to(torch.complex128).requires_grad_(True)
    b64 = conv.bias.detach().cpu().double().requires_grad_(True) if bias else None
    xr = x.double().requires_grad_(True)
    yr, rr = O.spectral_conv_forward(xr, w64, of, oi, num_groups=G, operator_type=op, separable=sep, bias=b64)
    tag = f"SpectralConv[{op}{'/sep' if sep else ''} G={G} {nlat_i}x{nlon_i}->{nlat_o}x{nlon_o} {precision} {act_dtype}]"
    out_tol = max(rtol, 4e-3) if act_dtype == torch.bfloat16 else rtol  # + one bf16 rounding of the output
    rel = {}
    rel["y"] = close(y, yr, out_tol, tag + " y")
    if conv.scale_residual:
        rel["residual"] = close(res, rr, out_tol, tag + " residual")
    else:
        assert res is xd
    gy = torch.randn(B, Cout, nlat_o, nlon_o).to(act_dtype)
    gres = torch.randn_like(rr).to(act_dtype) if conv.scale_residual else None
    if gres is not None:
        torch.autograd.backward([y, res], [gy.to(DEV), gres.to(DEV)])
        torch.autograd.backward([yr, rr], [gy.double(), gres.double()])
    else:
        y.backward(gy.to(DEV))
        yr.backward(gy.double())
    rel["dx"] = close(xd.grad, xr.grad, out_tol, tag + " dx")
    rel["dweight"] = close(conv.weight.grad, w64.grad, rtol, tag + " dweight")
    if bias:
        rel["dbias"] = close(conv.bias.grad, b64.grad, rtol, tag + " dbias")
    return rel


@pytest.mark.parametrize("case", CONV_CASES)
def test_spectral_conv_fwd_bwd_fp32(case):
    _run_conv_case(case, "fp32", 1e-5)


def test_spectral_conv_bf16_activations_fp32_math():
    _run_conv_case(CONV_CASES[1], "fp32", 1e-5, act_dtype=torch.bfloat16)


def test_weight_cache_tracks_parameter_updates():
    torch.manual_seed(333)
    f = mb.RealSHT(32, 64, 16, 17, "legendre-gauss", precision="fp32")
    i = mb.InverseRealSHT(32, 64, 16, 17, "legendre-gauss", precision="fp32")
    conv = mb.SpectralConv(f, i, 4, 4).to(DEV)
    x = torch.randn(1, 4, 32, 64, device=DEV)
    y0, _ = conv(x)
    with torch.no_grad():
        conv.weight.mul_(2.0)
    y1, _ = conv(x)
    close(y1, 2 * y0, 1e-6, "cached packed weight follows in-place parameter updates")
    packed = conv._wcache._packed
    conv(x)
    assert conv._wcache._packed is packed, "an unchanged parameter must reuse the packed copy"
    conv.weight.data.mul_(0.5)            # bypasses the version counter: needs an explicit invalidation
    conv.invalidate_weight_cache()
    y2, _ = conv(x)
    close(y2, y0, 1e-6, "invalidate_weight_cache after a .data write")
    sd = {k: v.clone() for k, v in conv.state_dict().items()}
    sd["weight"] = sd["weight"] * 3.0
    conv.load_state_dict(sd)
    y3, _ = conv(x)
    close(y3, 3 * y0, 1e-6, "load_state_dict invalidates the packed copy")


# ------------------------------------------------------------------- contractions / activations vs reference golden
def _mix_via_kernels(x, w, op, G=1, cbias=None):
    """x complex (B, C, L, M) -> packed -> mix kernel -> complex (B, Co, L, M)"""
    B, Ci, L, M = x.shape
    if op in (_lib.OP_DHCONV, _lib.OP_DIAGONAL):
        Co = w.shape[2] * G
    elif op in (_lib.OP_SEP_DHCONV, _lib.OP_SEP_DIAGONAL):
        Co = Ci
    else:
        Co = w.shape[-1]
    spec = _SpecPack.apply(x.to(DEV))
    y = mb.mix_packed(spec, w.to(DEV), op, L, M, B, G, Ci, Co, "fp32", cbias=None if cbias is None else cbias.to(DEV))
    return _SpecUnpack.apply(y, L, M, B, Co).cpu()


def test_contractions_match_reference_golden():
    g = np.load(GOLD)
    x = torch.from_numpy(g["x"])
    B, G, Ci, L, M = x.shape
    tri = torch.tril(torch.ones(L, M)).bool()  # the kernels only define l >= m (everything else is zero by construction)
    xf = x.reshape(B, G * Ci, L, M) * tri
    for name, op in (("dhconv", _lib.OP_DHCONV), ("diagonal", _lib.OP_DIAGONAL), ("sep_dhconv", _lib.OP_SEP_DHCONV), ("sep_diagonal", _lib.OP_SEP_DIAGONAL)):
        y = _mix_via_kernels(xf, torch.from_numpy(g[f"w_{name}"]), op, G=G)
        ref = torch.from_numpy(g[f"y_{name}"])
        ref = ref.reshape(B, -1, L, M) * tri
        assert torch.allclose(y, ref, atol=1e-5, rtol=1e-4), name  # tolerance of /root/reference/tests/test_contractions.py
    xa = torch.from_numpy(g["xa"]) * tri
    cb = torch.from_numpy(g["cbias"])
    for name, op in (("shared", _lib.OP_SHARED), ("ldep", _lib.OP_LDEP)):
        y = _mix_via_kernels(xa, torch.from_numpy(g[f"w_{name}"]), op)
        assert torch.allclose(y, torch.from_numpy(g[f"y_{name}"]) * tri, atol=1e-5, rtol=1e-4), name
        y = _mix_via_kernels(xa, torch.from_numpy(g[f"w_{name}"]), op, cbias=cb)
        ref = (torch.einsum("bixy,io->boxy" if name == "shared" else "bixy,xio->boxy", xa, torch.from_numpy(g[f"w_{name}"])) + cb) * tri
        assert torch.allclose(y, ref, atol=1e-5, rtol=1e-4), name + "+bias"


CONV_GOLD = os.path.join(os.path.dirname(__file__), "golden", "spectral_conv_golden.npz")
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_golden import CONV_GOLDEN_CASES  # noqa: E402


@pytest.mark.parametrize("name", sorted(CONV_GOLDEN_CASES))
def test_spectral_conv_matches_reference_class_golden(name):
    """The CUDA SpectralConv against the output / gradients of the REFERENCE's SpectralConv class (tests/golden/make_golden.py runs
    /root/reference/makani/models/common/spectral_convolution.py on the oracle transforms): fp32 path, rtol 1e-5."""
    g = np.load(CONV_GOLD)
    nlat_i, nlon_i, grid_i, nlat_o, nlon_o, grid_o, lmax, mmax, B, Cin, Cout, G, op, sep, bias = CONV_GOLDEN_CASES[name]
    f = mb.RealSHT(nlat_i, nlon_i, lmax, mmax, grid_i, precision="fp32")
    i = mb.InverseRealSHT(nlat_o, nlon_o, lmax, mmax, grid_o, precision="fp32")
    conv = mb.SpectralConv(f, i, Cin, Cout, num_groups=G, operator_type=op, separable=sep, bias=bias, precision="fp32").to(DEV)
    assert list(conv.weight.shape) == list(g[f"{name}/weight_shape"])
    with torch.no_grad():
        conv.weight.copy_(torch.from_numpy(g[f"{name}/weight"]))
        if bias:
            conv.bias.copy_(torch.from_numpy(g[f"{name}/bias"]))
    x = torch.from_numpy(g[f"{name}/x"]).to(DEV).requires_grad_(True)
    y, res = conv(x)
    rt = 2e-5
    close(y, torch.from_numpy(g[f"{name}/y"]), rt, f"golden {name} y")
    loss = (y * torch.from_numpy(g[f"{name}/gy"]).to(DEV)).sum()
    if f"{name}/residual" in g:
        close(res, torch.from_numpy(g[f"{name}/residual"]), rt, f"golden {name} residual")
        loss = loss + (res * torch.from_numpy(g[f"{name}/gres"]).to(DEV)).sum()
    loss.backward()
    close(x.grad, torch.from_numpy(g[f"{name}/dx"]), rt, f"golden {name} dx")
    close(conv.weight.grad, torch.from_numpy(g[f"{name}/dweight"]), rt, f"golden {name} dweight")
    if bias:
        close(conv.bias.grad, torch.from_numpy(g[f"{name}/dbias"]), 1e-4, f"golden {name} dbias")


def test_complex_relu_matches_reference_golden():
    g = np.load(GOLD)
    z = torch.from_numpy(g["z"])
    L, M = z.shape[-2:]
    tri = torch.tril(torch.ones(L, M)).bool()
    for mode in ("real", "cartesian", "modulus", "halfplane"):
        act = mb.ComplexReLU(negative_slope=0.1, mode=mode, bias_shape=(z.shape[1], 1, 1), scale=0.3).to(DEV)
        if isinstance(act.bias, torch.Tensor):
            with torch.no_grad():
                act.bias.copy_(torch.from_numpy(g[f"relu_bias_{mode}"]))
        y = act((z * tri).to(DEV)).cpu()
        assert torch.allclose(y, torch.from_numpy(g[f"relu_{mode}"]) * tri, atol=1e-6, rtol=1e-5), mode


@pytest.mark.parametrize("op,act", [("diagonal", "real"), ("l-dependant", "cartesian"), ("diagonal", "modulus"), ("diagonal", "halfplane")])
def test_spectral_attention_intended_semantics(op, act):
    torch.manual_seed(333)
    f = mb.RealSHT(32, 64, 16, 17, "legendre-gauss", precision="fp32")
    i = mb.InverseRealSHT(32, 64, 16, 17, "legendre-gauss", precision="fp32")
    att = mb.SpectralAttention(f, i, 6, 5, operator_type=op, hidden_size_factor=2, complex_activation=act, bias=True, spectral_layers=2, precision="fp32").to(DEV)
    of, oi = oracle_pair(32, 64, 32, 64, 16, 17, "legendre-gauss", "legendre-gauss")
    x = torch.randn(2, 6, 32, 64)
    xd = x.to(DEV).requires_grad_(True)
    y, _ = att(xd)
    ws = [w.detach().cpu().to(torch.complex128).requires_grad_(True) for w in att.w]
    wo = att.wout.detach().cpu().to(torch.complex128).requires_grad_(True)
    bs = [b.detach().cpu().to(torch.complex128).requires_grad_(True) for b in att.b]
    ab = [a.bias.detach().cpu().double().requires_grad_(True) if isinstance(a.bias, torch.Tensor) else 0.0 for a in att.activations]
    xr = x.double().requires_grad_(True)
    yr, _ = O.spectral_attention_forward(xr, ws, wo, of, oi, b_list=bs, act_mode=act, act_bias=ab, operator_type=op)
    close(y, yr, 1e-5, f"SpectralAttention[{op},{act}] y")
    gy = torch.randn_like(yr)
    y.backward(gy.float().to(DEV))
    yr.backward(gy)
    close(xd.grad, xr.grad, 2e-5, f"SpectralAttention[{op},{act}] dx")
    close(att.wout.grad, wo.grad, 2e-5, "dwout")
    close(att.w[0].grad, ws[0].grad, 2e-5, "dw0")
    close(att.b[1].grad, bs[1].grad, 2e-5, "db1")
    for k, (a, r) in enumerate(zip(att.activations, ab)):
        if isinstance(a.bias, torch.Tensor):
            close(a.bias.grad, r.grad if r.grad is not None else torch.zeros_like(r), 2e-5, f"activation {k} bias grad")


# ----------------------------------------------------------------- size-independent properties at BASELINE sizes
def test_full_size_properties_721x1440():
    """BASELINE configs[1] geometry (721x1440 equiangular, lmax 240, mmax 241): band-limited round trip, linearity,
    Parseval and <Ax, y> = <x, A^T y> -- no oracle run needed at this size."""
    torch.manual_seed(333)
    C = 4
    sht = mb.RealSHT(721, 1440, 240, 241, "equiangular", precision="fp32")
    isht = mb.InverseRealSHT(721, 1440, 240, 241, "equiangular", precision="fp32")
    c = torch.tril(torch.randn(1, C, 240, 241, dtype=torch.complex64)).to(DEV)
    c[..., 0] = c[..., 0].real.to(torch.complex64)
    x = isht(c)
    close(sht(x), c, 2e-5, "721x1440 isht->sht round trip (Clenshaw-Curtis exact to degree 720 > 2*239)")
    x2 = torch.randn(1, C, 721, 1440, device=DEV)
    close(sht(2.5 * x - 0.5 * x2), 2.5 * sht(x) - 0.5 * sht(x2), 2e-5, "linearity")
    _, w = O.precompute_latitudes(721, "equiangular")
    q = (torch.from_numpy(w).float() * 2 * math.pi / 1440).to(DEV)[:, None]
    mw = torch.full((241,), 2.0, device=DEV)
    mw[0] = 1.0
    lhs = (x.double() ** 2 * q.double()).sum(dim=(-1, -2))
    rhs = ((c.abs().double() ** 2) * mw.double()).sum(dim=(-1, -2))
    close(lhs, rhs, 1e-5, "Parseval")
    xg = x2.clone().requires_grad_(True)
    gc = torch.randn(1, C, 240, 241, dtype=torch.complex64, device=DEV)
    sht(xg).backward(gc)
    lhs = (torch.view_as_real(sht(x2)).double() * torch.view_as_real(gc).double()).sum()
    rhs = (x2.double() * xg.grad.double()).sum()
    assert abs(lhs.item() - rhs.item()) <= 2e-5 * max(abs(lhs.item()), 1.0), (lhs.item(), rhs.item())


# ------------------------------------------------------------------------------- distributed modules on one GPU
def test_distributed_modules_world1_and_dense_conv():
    """world size 1: Distributed* transforms (sub-plans + dense packed spectra + dense mix) == local transforms == oracle."""
    import makani_b200.distributed as mbd

    torch.manual_seed(333)
    nlat, nlon, lmax, mmax, B, C = 48, 96, 30, 33, 2, 6
    f = mbd.DistributedRealSHT(nlat, nlon, lmax, mmax, "legendre-gauss", precision="fp32")
    i = mbd.DistributedInverseRealSHT(nlat, nlon, lmax, mmax, "legendre-gauss", precision="fp32")
    conv = mb.SpectralConv(f, i, C, C, operator_type="dhconv", bias=True, precision="fp32").to(DEV)
    assert conv.modes_lat_local == lmax and conv.modes_lon_local == mmax
    of, oi = oracle_pair(nlat, nlon, nlat, nlon, lmax, mmax, "legendre-gauss", "legendre-gauss")
    x = torch.randn(B, C, nlat, nlon)
    xd = x.to(DEV).requires_grad_(True)
    y, _ = conv(xd)
    w64 = conv.weight.detach().cpu().to(torch.complex128).requires_grad_(True)
    xr = x.double().requires_grad_(True)
    yr, _ = O.spectral_conv_forward(xr, w64, of, oi, operator_type="dhconv", bias=conv.bias.detach().cpu().double())
    close(y, yr, 1e-5, "dist(world=1) SpectralConv y")
    gy = torch.randn(B, C, nlat, nlon)
    y.backward(gy.to(DEV))
    yr.backward(gy.double())
    close(xd.grad, xr.grad, 1e-5, "dist(world=1) SpectralConv dx")
    close(conv.weight.grad, w64.grad, 1e-5, "dist(world=1) SpectralConv dweight")

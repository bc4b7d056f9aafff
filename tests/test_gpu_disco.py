"""DISCO convolution on an H100: both kernels of csrc/disco.cu through ctypes against an fp64 contraction of the exact fp32 psi_hat the plan
stores, determinism, the module against the fp64 oracle (fp32 and TF32 GEMMs), and the adjoint identity at FCN3's sizes.

Kernel bound: |out - ref| <= C_SUM n 2^-24 sum |psi| |in| per element, n = the number of terms of that element's sum (fp32 accumulation of n
products; the classical bound of recursive summation has C = 1).  C_SUM = 0.25 was calibrated on an H100 80GB HBM3: the largest need over
every case below was 0.033 (forward, bf16 input) and 0.015 (adjoint).  bf16 outputs add the bf16 unit roundoff, 2^-8 |ref|.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

from makani_b200 import _lib  # noqa: E402
from makani_b200 import disco as D  # noqa: E402
from makani_b200.sht import _ptr, _stream  # noqa: E402
from oracle import makani_disco_oracle as O  # noqa: E402

C_SUM = 0.25
DEV = torch.device("cuda", 0)

# (in_shape, out_shape, grid_in, grid_out, cutoff in input spacings): pscale 1 and 2, poles on equiangular output grids, nlon_out 45 (not a multiple
# of any thread tile), nlon_in 90 (no 16-byte staging), a 13-row band over 11-row stages with > 256 points per pole latitude, and nlon 1040 (two
# longitude tiles per CTA row, two adjoint passes over K = 20)
GEOMS = {
    "eq33x64": ((33, 64), (33, 64), "equiangular", "equiangular", 3.0),
    "eq33x96_lg17x48": ((33, 96), (17, 48), "equiangular", "legendre-gauss", 3.0),
    "eq21x90_eq21x45": ((21, 90), (21, 45), "equiangular", "equiangular", 2.5),
    "eq91x180_lg46x90": ((91, 180), (46, 90), "equiangular", "legendre-gauss", 6.0),
    "eq9x1040": ((9, 1040), (9, 1040), "equiangular", "equiangular", 1.5),
}
CASES = [("eq33x64", (1, 1)), ("eq33x64", (3, 3)), ("eq33x96_lg17x48", (5, 4)), ("eq21x90_eq21x45", (3, 3)), ("eq91x180_lg46x90", (3, 3)),
         ("eq91x180_lg46x90", (5, 4)), ("eq9x1040", (5, 4)), ("eq21x90_eq21x45", (6, 6))]


def _psi(name, kernel_shape, norm="mean"):
    ish, osh, gi, go, u = GEOMS[name]
    return D.get_psi(tuple(kernel_shape), "morlet", norm, ish, osh, gi, go, u * math.pi / (ish[0] - 1))


def _dense32(psi):
    """the plan's fp32 values as an fp64 (K * nlat_out, nlat_in * nlon_in) matrix on the GPU"""
    d = D.psi_dense(psi).astype(np.float32).astype(np.float64)
    return torch.from_numpy(d.reshape(psi.kernel_size * psi.nlat_out, -1)).to(DEV)


def _sentinel(shape, dtype, pad=4096):
    buf = torch.full((pad + int(np.prod(shape)) + pad,), float("nan"), dtype=dtype, device=DEV)
    return buf, buf[pad : pad + int(np.prod(shape))].view(shape)


def _untouched(buf, pad=4096):
    return bool(torch.isnan(buf[:pad]).all() and torch.isnan(buf[-pad:]).all())


def _forward_raw(plan, x, B, C):
    buf, X = _sentinel((B, C, plan.K, plan.nlat_out, plan.nlon_out), torch.float32)
    _lib.call("b200sht_disco_forward", plan.handle, _ptr(x), 0 if x.dtype == torch.float32 else 1, B, C, _ptr(X), _stream(DEV))
    return buf, X


def _adjoint_raw(plan, dX, B, C, dtype):
    buf, dx = _sentinel((B, C, plan.nlat_in, plan.nlon_in), dtype)
    _lib.call("b200sht_disco_adjoint", plan.handle, _ptr(dX), _ptr(dx), 0 if dtype == torch.float32 else 1, B, C, _stream(DEV))
    return buf, dx


NEEDS = {}


@pytest.mark.parametrize("name,kernel_shape", CASES)
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_kernels_against_fp64(name, kernel_shape, dtype):
    psi = _psi(name, kernel_shape)
    plan = D.DiscoPlan(psi, DEV)
    K, (hi, wi), (ho, wo) = psi.kernel_size, GEOMS[name][0], GEOMS[name][1]
    assert plan.query(4) == K and plan.query(8) == wi // wo and plan.query(5) == len(psi.val)
    B, C = 3, 5                                                   # 15 rows: not a multiple of any row chunk
    g = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(B, C, hi, wi, generator=g, device=DEV).to(dtype)
    P = _dense32(psi)
    # forward
    buf, X = _forward_raw(plan, x, B, C)
    torch.cuda.synchronize()
    assert _untouched(buf) and not torch.isnan(X).any()
    ref = O.contraction(x.double(), P, K, ho, wo)
    mag = O.contraction(x.double().abs(), P.abs(), K, ho, wo)
    n_f = int(np.diff(psi.row_ptr).max()) // K
    need_f = ((X.double() - ref).abs() / (n_f * 2.0**-24 * mag + 1e-300)).max().item()
    assert need_f <= C_SUM, f"forward needs C = {need_f:.3g}"
    # adjoint
    dX = torch.randn(B, C, K, ho, wo, generator=g, device=DEV)
    buf, dx = _adjoint_raw(plan, dX, B, C, dtype)
    torch.cuda.synchronize()
    assert _untouched(buf) and not torch.isnan(dx.float()).any()
    ref = O.adjoint(dX.double(), P, hi, wi)
    mag = O.adjoint(dX.double().abs(), P.abs(), hi, wi)
    per_i = np.bincount(psi.col // wi, minlength=hi)               # entries (k, t, j) reaching input row i
    n_a = int(per_i.max())
    extra = 2.0**-8 * ref.abs() if dtype == torch.bfloat16 else 0.0
    need_a = ((dx.double() - ref).abs() - extra).clamp(min=0).div(n_a * 2.0**-24 * mag + 1e-300).max().item()
    assert need_a <= C_SUM, f"adjoint needs C = {need_a:.3g}"
    NEEDS[(name, kernel_shape, str(dtype))] = (need_f, need_a)
    print(f"\nC needed: {name} {kernel_shape} {dtype}: forward {need_f:.3g} adjoint {need_a:.3g}")


@pytest.mark.parametrize("name,kernel_shape", [("eq91x180_lg46x90", (3, 3)), ("eq33x96_lg17x48", (5, 4))])
def test_kernels_deterministic(name, kernel_shape):
    psi = _psi(name, kernel_shape)
    plan = D.DiscoPlan(psi, DEV)
    (hi, wi), (ho, wo) = GEOMS[name][0], GEOMS[name][1]
    x = torch.randn(2, 7, hi, wi, device=DEV)
    dX = torch.randn(2, 7, psi.kernel_size, ho, wo, device=DEV)
    a, b = plan.forward(x), plan.forward(x)
    assert torch.equal(a, b)
    a, b = plan.adjoint(dX), plan.adjoint(dX)
    assert torch.equal(a, b)


def _module_pair(cin, cout, ish, osh, ks, groups, bias, gi, go, norm="mean"):
    cutoff = 2.5 * math.pi / (ish[0] - 1)
    kw = dict(basis_type="morlet", basis_norm_mode=norm, groups=groups, grid_in=gi, grid_out=go, bias=bias, theta_cutoff=cutoff)
    ref = O.DiscreteContinuousConvS2(cin, cout, ish, osh, ks, **kw).double()
    mod = D.DiscreteContinuousConvS2(cin, cout, ish, osh, ks, **kw).to(DEV)
    with torch.no_grad():
        mod.weight.copy_(ref.weight.float())
        if bias:
            ref.bias.normal_()
            mod.bias.copy_(ref.bias.float())
    return mod, ref


MODULE_CASES = [
    (6, 8, (33, 64), (17, 32), (3, 3), 2, True, "equiangular", "legendre-gauss", "mean"),
    (5, 7, (33, 64), (33, 64), (3, 3), 1, False, "equiangular", "equiangular", "individual"),
    (12, 9, (21, 40), (21, 40), (5, 4), 3, True, "legendre-gauss", "legendre-gauss", "support"),
]


def _rel_l2(a, b):
    return ((a.double().cpu() - b).norm() / b.norm()).item()


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("case", MODULE_CASES)
def test_module_against_oracle(case, tf32):
    cin, cout, ish, osh, ks, G, bias, gi, go, norm = case
    torch.manual_seed(11)
    mod, ref = _module_pair(cin, cout, ish, osh, ks, G, bias, gi, go, norm)
    x = torch.randn(2, cin, *ish, dtype=torch.float64)
    gy = torch.randn(2, cout, *osh, dtype=torch.float64)
    xr = x.clone().requires_grad_(True)
    yr = ref(xr)
    yr.backward(gy)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        xd = x.float().to(DEV).requires_grad_(True)
        y = mod(xd)
        y.backward(gy.float().to(DEV))
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    pairs = [("y", y, yr), ("dx", xd.grad, xr.grad), ("dw", mod.weight.grad, ref.weight.grad)]
    if bias:
        pairs.append(("db", mod.bias.grad, ref.bias.grad))
    for what, a, b in pairs:
        a, b = a.detach(), b.detach()
        if tf32:
            rel = _rel_l2(a, b)
            assert rel < TF32_REL_L2, f"{what}: TF32 rel L2 {rel:.3g}"
            print(f"\nTF32 rel L2 {case[2]}->{case[3]} {what}: {rel:.3g}")
        else:
            err = (a.double().cpu() - b).abs().max().item()
            assert err <= 1e-5 * b.abs().max().item(), f"{what}: {err:.3g} vs max {b.abs().max().item():.3g}"


TF32_REL_L2 = 5e-3     # largest measured on an H100 80GB HBM3: 3.2e-4 (dW; y, dx and db stay below 1e-5)


def test_module_bf16_input_and_weight_read_afresh():
    torch.manual_seed(3)
    mod, ref = _module_pair(4, 6, (33, 64), (17, 32), (3, 3), 2, True, "equiangular", "equiangular")
    x = torch.randn(1, 4, 33, 64).to(torch.bfloat16)
    xd = x.to(DEV).requires_grad_(True)
    y = mod(xd)
    y.sum().backward()
    assert xd.grad.dtype == torch.bfloat16
    yr = ref(x.double())
    assert (y.double().cpu() - yr.detach()).abs().max() <= 1e-5 * yr.abs().max()
    # makani rescales the weight in place; forward must see it
    with torch.no_grad():
        mod.weight *= 2.0
    y2 = mod(xd)
    b = mod.bias.detach().view(1, -1, 1, 1)
    assert torch.allclose(y2.detach() - b, 2 * (y.detach() - b), rtol=1e-5, atol=1e-6)


def _dot(a, b, rows=32):
    """sum(a * b) in fp64, a few channels at a time (the processor's X is 6.3 GB in fp32)"""
    return sum((a[:, c : c + rows].double() * b[:, c : c + rows].double()).sum().item() for c in range(0, a.shape[1], rows))


@pytest.mark.parametrize("what", ["encoder", "processor"])
def test_adjoint_identity_at_fcn3_sizes(what):
    """<forward(x), y> = <x, adjoint(y)> with the library's two kernels at FCN3's encoder and processor geometries (B = 1)"""
    if what == "encoder":
        ish, osh, gi, go, C = (721, 1440), (360, 720), "equiangular", "legendre-gauss", 72
        cutoff = (3 + 1) * 0.5 * math.pi / 720
    else:
        ish, osh, gi, go, C = (360, 720), (360, 720), "legendre-gauss", "legendre-gauss", 677
        cutoff = 2 * (3 + 1) * 0.5 * math.pi / 359
    key = ((3, 3), "morlet", "mean", ish, osh, gi, go, cutoff)
    plan = D.get_plan(key, DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    x = torch.randn(1, C, *ish, generator=g, device=DEV)
    X = plan.forward(x)
    y = torch.randn(X.shape, generator=g, device=DEV)
    lhs, mag = _dot(X, y), _dot(X.abs(), y.abs())
    del X
    dx = plan.adjoint(y)
    rhs = _dot(x, dx)
    assert abs(lhs - rhs) <= 1e-6 * mag, (lhs, rhs, mag)
    print(f"\n{what}: <Fx, y> {lhs:.9e}  <x, F'y> {rhs:.9e}  diff / sum|Fx||y| {abs(lhs - rhs) / mag:.3g}")

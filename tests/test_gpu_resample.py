"""Bilinear resampling on an H100: both kernels of csrc/resample.cu through ctypes against an fp64 evaluation of the plan's exact fp32 tables,
the adjoint identity, determinism, the module against the fp64 oracle (forward and input gradient, 3-D and 5-D inputs), the skip path, FCN3's
full decoder shape, and makani's own decoder through the golden vectors of tests/golden/make_fcn3_decoder_golden.py.

Kernel bound: |out - ref| <= C_SUM n 2^-24 sum |w x| per element, where sum |w x| is the same evaluation on |x| and n counts the roundings of
that element: forward 6 (three lerps) plus nlon_in where a pole pseudo-row enters; adjoint (rows + 1)(columns + 1) from the two CSR lists, plus
nlon_out times the rows referencing a pole pseudo-row.  C_SUM = 1 is the worst case of that count; the largest need measured on an H100 is
printed per case and recorded in DESIGN.md section 4.8.
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
from makani_b200 import resample as R  # noqa: E402
from makani_b200.sht import _ptr, _stream  # noqa: E402
from oracle import makani_resample_oracle as O  # noqa: E402

C_SUM = 1.0
DEV = torch.device("cuda", 0)

# the grid pairs of tests/test_resample_cpu.py, plus odd sizes on both sides and a 16x latitude upsampling (many rows per input row)
PAIRS = {
    "lg24x48-eq49x96": (24, 48, 49, 96, "legendre-gauss", "equiangular"),
    "eq25x48-eq49x96": (25, 48, 49, 96, "equiangular", "equiangular"),
    "eq49x96-lg24x48": (49, 96, 24, 48, "equiangular", "legendre-gauss"),
    "eq17x35-eq33x70": (17, 35, 33, 70, "equiangular", "equiangular"),
    "lg11x21-eq37x75": (11, 21, 37, 75, "legendre-gauss", "equiangular"),
    "lg8x16-eq121x240": (8, 16, 121, 240, "legendre-gauss", "equiangular"),
}


def _tab64(pair):
    """the plan's fp32 tables in the oracle's layout, for an fp64 evaluation on the GPU"""
    t = R.precompute_tables(*pair)
    return dict(lat_idx=torch.from_numpy(t.lat_idx), lat_w=torch.from_numpy(t.lat_w), lon_left=torch.from_numpy(t.lon_left),
                lon_right=torch.from_numpy(t.lon_right), lon_w=torch.from_numpy(t.lon_w), expand_poles=t.expand_poles), t


def _sentinel(shape, pad=4096):
    buf = torch.full((pad + int(np.prod(shape)) + pad,), float("nan"), dtype=torch.float32, device=DEV)
    return buf, buf[pad : pad + int(np.prod(shape))].view(shape)


def _untouched(buf, pad=4096):
    return bool(torch.isnan(buf[:pad]).all() and torch.isnan(buf[-pad:]).all())


def _rounding_counts(pair, t):
    nlat_in, nlon_in, nlat_out, nlon_out = pair[:4]
    nexp = nlat_in + 2 * t.expand_poles
    pole_f = np.zeros(nlat_out)
    if t.expand_poles:
        pole_f = ((t.lat_idx == 0) | (t.lat_idx + 1 == nexp - 1)) * nlon_in
    n_f = torch.from_numpy(6 + pole_f).to(DEV)[:, None]                                         # per output row
    rows = np.bincount(np.concatenate([t.lat_idx, t.lat_idx + 1]), minlength=nexp)            # per expanded input row
    cols = np.bincount(np.concatenate([t.lon_left, t.lon_right]), minlength=nlon_in)
    off = 1 if t.expand_poles else 0
    n_a = (rows[off : off + nlat_in, None] + 1.0) * (cols[None, :] + 1.0)
    if t.expand_poles:
        n_a[0] += rows[0] * nlon_out + 1
        n_a[-1] += rows[-1] * nlon_out + 1
    return n_f, torch.from_numpy(n_a).to(DEV)


def _adjoint64(dy, tab, nlat_in, nlon_in):
    x = torch.zeros(*dy.shape[:-2], nlat_in, nlon_in, dtype=torch.float64, device=DEV, requires_grad=True)
    O.resample(x, tab).backward(dy)
    return x.grad


@pytest.mark.parametrize("name", list(PAIRS))
def test_kernels_against_fp64(name):
    pair = PAIRS[name]
    nlat_in, nlon_in, nlat_out, nlon_out = pair[:4]
    tab, t = _tab64(pair)
    plan = R.ResamplePlan(*pair[:4], t, DEV)
    assert [plan.query(k) for k in range(5)] == [nlat_in, nlon_in, nlat_out, nlon_out, int(t.expand_poles)]
    P = 19                                                           # not a multiple of the planes per CTA
    g = torch.Generator(device=DEV).manual_seed(7)
    x = torch.randn(P, nlat_in, nlon_in, generator=g, device=DEV)
    n_f, n_a = _rounding_counts(pair, t)
    # forward
    buf, y = _sentinel((P, nlat_out, nlon_out))
    _lib.call("b200sht_resample_forward", plan.handle, _ptr(x), _ptr(y), P, _stream(DEV))
    torch.cuda.synchronize()
    assert _untouched(buf) and not torch.isnan(y).any()
    ref, mag = O.resample(x.double(), tab), O.resample(x.double().abs(), tab)
    need_f = ((y.double() - ref).abs() / (n_f * 2.0**-24 * mag + 1e-300)).max().item()
    assert need_f <= C_SUM, f"forward needs C = {need_f:.3g}"
    # adjoint
    dy = torch.randn(P, nlat_out, nlon_out, generator=g, device=DEV)
    buf, dx = _sentinel((P, nlat_in, nlon_in))
    _lib.call("b200sht_resample_adjoint", plan.handle, _ptr(dy), _ptr(dx), P, _stream(DEV))
    torch.cuda.synchronize()
    assert _untouched(buf) and not torch.isnan(dx).any()
    ref, mag = _adjoint64(dy.double(), tab, nlat_in, nlon_in), _adjoint64(dy.double().abs(), tab, nlat_in, nlon_in)
    need_a = ((dx.double() - ref).abs() / (n_a * 2.0**-24 * mag + 1e-300)).max().item()
    assert need_a <= C_SUM, f"adjoint needs C = {need_a:.3g}"
    print(f"\nC needed: {name}: forward {need_f:.3g} adjoint {need_a:.3g}")


@pytest.mark.parametrize("name", ["lg24x48-eq49x96", "eq17x35-eq33x70", "lg8x16-eq121x240"])
def test_adjoint_identity_and_determinism(name):
    pair = PAIRS[name]
    plan = R.get_plan(pair, DEV)
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(37, *pair[:2], generator=g, device=DEV)
    y = torch.randn(37, *pair[2:4], generator=g, device=DEV)
    Rx, Rty = plan.forward(x), plan.adjoint(y)
    lhs, rhs = (Rx.double() * y.double()).sum().item(), (x.double() * Rty.double()).sum().item()
    mag = (Rx.double().abs() * y.double().abs()).sum().item()
    assert abs(lhs - rhs) <= 1e-6 * mag, (lhs, rhs, mag)
    assert torch.equal(plan.adjoint(y), Rty) and torch.equal(plan.forward(x), Rx)


@pytest.mark.parametrize("lead", [(2, 3, 4), (2, 3)], ids=["5d", "3d"])
@pytest.mark.parametrize("name", ["lg24x48-eq49x96", "eq25x48-eq49x96", "eq49x96-lg24x48", "eq17x35-eq33x70"])
def test_module_against_oracle(name, lead):
    pair = PAIRS[name]
    mod, ref = R.ResampleS2(*pair[:4], grid_in=pair[4], grid_out=pair[5]).to(DEV), O.ResampleS2(*pair[:4], grid_in=pair[4], grid_out=pair[5])
    torch.manual_seed(5)
    x = torch.randn(*lead, *pair[:2], dtype=torch.float64)
    gy = torch.randn(*lead, *pair[2:4], dtype=torch.float64)
    xd = x.float().to(DEV).requires_grad_(True)
    y = mod(xd)
    y.backward(gy.float().to(DEV))
    xr = x.float().double().requires_grad_(True)
    yr = ref(xr)
    yr.backward(gy.float().double())
    assert y.shape == yr.shape and y.dtype == torch.float32 and xd.grad.shape == xd.shape
    for what, a, b in (("y", y, yr), ("dx", xd.grad, xr.grad)):
        err = (a.detach().double().cpu() - b.detach()).abs().max().item()
        assert err <= 2e-6 * b.abs().max().item(), f"{what}: {err:.3g}"


def test_module_refusals_on_the_device():
    mod = R.ResampleS2(24, 48, 49, 96, grid_in="legendre-gauss", grid_out="equiangular").to(DEV)
    with pytest.raises(R.B200ShtError):
        mod(torch.randn(2, 24, 48, device=DEV, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        mod(torch.randn(2, 48, 24, device=DEV))
    # a non-contiguous input is resampled as its contiguous copy
    x = torch.randn(2, 48, 24, device=DEV).transpose(-1, -2)
    assert torch.equal(mod(x), mod(x.contiguous()))


def test_skip_path_returns_its_input():
    mod = R.ResampleS2(49, 96, 49, 96).to(DEV)
    x = torch.randn(3, 49, 96, device=DEV)
    assert mod.skip_resampling and mod(x) is x


def test_fcn3_decoder_shape():
    """FCN3's atmospheric decoder at B = 1: 585 planes, 360 x 720 Legendre-Gauss -> 721 x 1440 equiangular, against the oracle in fp64 on the GPU"""
    pair = (360, 720, 721, 1440, "legendre-gauss", "equiangular")
    mod = R.ResampleS2(*pair[:4], grid_in=pair[4], grid_out=pair[5]).to(DEV)
    tab, _ = _tab64(pair)
    g = torch.Generator(device=DEV).manual_seed(11)
    x = torch.randn(1, 585, 360, 720, generator=g, device=DEV).requires_grad_(True)
    y = mod(x)
    gy = torch.randn(y.shape, generator=g, device=DEV)
    y.backward(gy)
    torch.cuda.synchronize()
    worst_y = worst_dx = 0.0
    for c in range(0, 585, 65):
        xs = x.detach()[:, c : c + 65].double().requires_grad_(True)
        yr = O.resample(xs, tab)
        yr.backward(gy[:, c : c + 65].double())
        worst_y = max(worst_y, ((y[:, c : c + 65].double() - yr.detach()).abs().max() / yr.detach().abs().max()).item())
        worst_dx = max(worst_dx, ((x.grad[:, c : c + 65].double() - xs.grad).abs().max() / xs.grad.abs().max()).item())
        del xs, yr
    print(f"\nFCN3 decoder shape: max |y - ref| / max |ref| {worst_y:.3g}, dx {worst_dx:.3g}")
    assert worst_y <= 1e-6 and worst_dx <= 1e-6


GOLDEN = os.path.join(ROOT, "tests", "golden", "fcn3_decoder_golden.npz")
GOLDEN_CASES = {"lg24x48_eq49x96": ((24, 48), "legendre-gauss"), "eq25x48_eq49x96": ((25, 48), "equiangular")}


@pytest.mark.parametrize("case", list(GOLDEN_CASES))
def test_makani_decoder_golden(case):
    """makani's DiscreteContinuousDecoder(upsample_sht=False) = ResampleS2 then DiscreteContinuousConvS2 (fp32, autocast off)"""
    z = np.load(GOLDEN)
    get = lambda k: torch.from_numpy(z[f"{case}/{k}"])   # noqa: E731
    x, w, y_ref, g, dx_ref, dw_ref = get("x"), get("weight"), get("y"), get("g"), get("dx"), get("dW")
    ish, gi = GOLDEN_CASES[case]
    osh = tuple(y_ref.shape[-2:])
    cin, cout = x.shape[1], y_ref.shape[1]
    res = R.ResampleS2(*ish, *osh, grid_in=gi, grid_out="equiangular", mode="bilinear").to(DEV)
    conv = D.DiscreteContinuousConvS2(cin, cout, in_shape=osh, out_shape=osh, kernel_shape=(3, 3), basis_type="morlet", basis_norm_mode="mean",
                                      grid_in="equiangular", grid_out="equiangular", groups=math.gcd(cin, cout), bias=False,
                                      theta_cutoff=float(z[f"{case}/theta_cutoff"])).to(DEV)
    with torch.no_grad():
        conv.weight.copy_(w)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        xd = x.to(DEV).requires_grad_(True)
        y = conv(res(xd))
        (y * g.to(DEV)).sum().backward()
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    for what, a, b in (("y", y, y_ref), ("dx", xd.grad, dx_ref), ("dW", conv.weight.grad, dw_ref)):
        err = (a.detach().cpu().double() - b.double()).abs().max().item()
        assert err <= 1e-5 * b.abs().max().item(), f"{what}: {err:.3g} vs max {b.abs().max().item():.3g}"

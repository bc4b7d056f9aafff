"""DiscreteContinuousConvTransposeS2 on an H100:

* the module against the fp64 oracle (tests/disco_transpose_oracle.py): y, dx, dW and dbias at fp32 and bf16 input, groups > 1, bias on and
  off, s = 1 and s = 2, and FCN3's decoder geometry (360 x 720 Legendre-Gauss -> 721 x 1440 equiangular) at few channels, with the oracle's
  psi_T sparse on the device; fp32 GEMMs, tolerances as in tests/test_gpu_disco.py;
* the adjoint identity <y, z>_out = sum_k <Y_k, X_k>_in between the transposed plan's adjoint kernel and the forward convolution's plan (out
  grid -> in grid) at the decoder geometry, mode "none";
* two calls give bit-identical y and gradients;
* virtual ranks: each rank's window contraction (the backward) is bit-identical to the slice of the single-GPU contraction, and y of the
  module's per-rank arithmetic (window adjoints added in rank order, as the halo's adjoint adds them) is within 2e-6 relative of the module."""
import math
from types import SimpleNamespace

import pytest
import torch

import disco_transpose_oracle as TO
import makani_b200.distributed as mbd
from makani_b200 import disco as D
from makani_b200.distributed import disco as DD
from makani_b200.quadrature import precompute_latitudes

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

DECODER = ((360, 720), (721, 1440), "legendre-gauss", "equiangular", (3 + 1) * 0.5 * math.pi / 720)

# (C_in, C_out, in_shape, out_shape, kernel_shape, groups, bias, grid_in, grid_out, norm, input dtype)
MODULE_CASES = [
    (6, 8, (17, 32), (33, 64), (3, 3), 2, True, "equiangular", "equiangular", "mean", torch.float32),
    (5, 7, (33, 64), (33, 64), (3, 3), 1, False, "equiangular", "equiangular", "individual", torch.float32),
    (12, 9, (21, 40), (21, 40), (5, 4), 3, True, "legendre-gauss", "legendre-gauss", "support", torch.float32),
    (6, 4, (24, 48), (47, 96), (3, 3), 2, True, "legendre-gauss", "equiangular", "none", torch.float32),
    (4, 6, (17, 32), (33, 64), (3, 3), 2, True, "equiangular", "equiangular", "mean", torch.bfloat16),
    (2, 3, DECODER[0], DECODER[1], (3, 3), 1, True, DECODER[2], DECODER[3], "mean", torch.float32),
]


def _pair(cin, cout, ish, osh, ks, G, bias, gi, go, norm, cutoff=None):
    big = ish[0] * ish[1] > 1e5
    cutoff = cutoff if cutoff is not None else (DECODER[4] if big else 2.5 * math.pi / (osh[0] - 1))
    kw = dict(basis_type="morlet", basis_norm_mode=norm, groups=G, grid_in=gi, grid_out=go, bias=bias, theta_cutoff=cutoff)
    ref = TO.DiscreteContinuousConvTransposeS2(cin, cout, ish, osh, ks, **kw, sparse=big, device=DEV if big else "cpu").double()
    mod = D.DiscreteContinuousConvTransposeS2(cin, cout, ish, osh, ks, **kw).to(DEV)
    with torch.no_grad():
        mod.weight.copy_(ref.weight.float())
        if bias:
            ref.bias.normal_()
            mod.bias.copy_(ref.bias.float())
    return mod, ref, (DEV if big else torch.device("cpu"))


@pytest.mark.parametrize("case", MODULE_CASES)
def test_module_against_oracle(case):
    cin, cout, ish, osh, ks, G, bias, gi, go, norm, dtype = case
    torch.manual_seed(11)
    mod, ref, rdev = _pair(cin, cout, ish, osh, ks, G, bias, gi, go, norm)
    ref = ref.to(rdev)
    x = torch.randn(2, cin, *ish).to(dtype)
    gy = torch.randn(2, cout, *osh, dtype=torch.float64)
    xr = x.double().to(rdev).requires_grad_(True)
    yr = ref(xr)
    yr.backward(gy.to(rdev))
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        xd = x.to(DEV).requires_grad_(True)
        y = mod(xd)
        y.backward(gy.float().to(DEV))
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    assert y.dtype == torch.float32 and y.shape == (2, cout, *osh) and xd.grad.dtype == dtype
    pairs = [("y", y, yr), ("dx", xd.grad, xr.grad), ("dw", mod.weight.grad, ref.weight.grad)]
    if bias:
        pairs.append(("db", mod.bias.grad, ref.bias.grad))
    for what, a, b in pairs:
        a, b = a.detach().double().cpu(), b.detach().cpu()
        extra = 2.0**-8 * b.abs() if (what == "dx" and dtype == torch.bfloat16) else 0.0
        err = ((a - b).abs() - extra).max().item()
        assert err <= 1e-5 * b.abs().max().item(), f"{what}: {err:.3g} vs max {b.abs().max().item():.3g}"


def _q(nlat, nlon, grid):
    _, w = precompute_latitudes(nlat, grid)
    return torch.as_tensor(w, dtype=torch.float64, device=DEV).view(-1, 1) * (2 * math.pi / nlon)


def test_adjoint_identity_at_decoder_shape():
    (ish, osh, gi, go, cutoff), C = DECODER, 8
    tplan = D.get_plan(D._psi_key((3, 3), "morlet", "none", osh, ish, go, gi, cutoff, True), DEV)
    fplan = D.get_plan(D._psi_key((3, 3), "morlet", "none", osh, ish, go, gi, cutoff), DEV)
    g = torch.Generator(device=DEV).manual_seed(5)
    Y = torch.randn(1, C, 9, *ish, generator=g, device=DEV)
    z = torch.randn(1, C, *osh, generator=g, device=DEV)
    y, X = tplan.adjoint(Y), fplan.forward(z)
    qo, qi = _q(*osh, go), _q(*ish, gi)
    lhs = (y.double() * z.double() * qo).sum().item()
    rhs = (Y.double() * X.double() * qi).sum().item()
    mag = (Y.double().abs() * X.double().abs() * qi).sum().item()
    print(f"\n<y, z>_out {lhs:.9e}  sum_k <Y_k, X_k>_in {rhs:.9e}  diff / mag {abs(lhs - rhs) / mag:.3g}")
    assert abs(lhs - rhs) <= 1e-6 * mag, (lhs, rhs, mag)


def test_two_calls_bit_identical():
    torch.manual_seed(2)
    mod, _, _ = _pair(6, 8, (24, 48), (47, 96), (3, 3), 2, True, "legendre-gauss", "equiangular", "mean")
    x = torch.randn(2, 6, 24, 48, device=DEV)
    gy = torch.randn(2, 8, 47, 96, device=DEV)
    outs = []
    for _ in range(2):
        mod.zero_grad()
        xd = x.clone().requires_grad_(True)
        y = mod(xd)
        y.backward(gy)
        outs.append([y.detach(), xd.grad, mod.weight.grad.clone(), mod.bias.grad.clone()])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _ops(key, window):
    return DD.CudaDiscoLocalOps(SimpleNamespace(_key=key, window=window))


@torch.no_grad()
@pytest.mark.parametrize("h", [2, 3, 4])
@pytest.mark.parametrize("geom", [DECODER, ((91, 180), (181, 360), "equiangular", "equiangular", 4 * math.pi / 180)])
def test_virtual_ranks_match_single_gpu_module(geom, h):
    ish, osh, gi, go, cutoff = geom
    torch.manual_seed(3)
    mod = D.DiscreteContinuousConvTransposeS2(4, 6, ish, osh, (3, 3), basis_type="morlet", groups=2, grid_in=gi, grid_out=go,
                                              theta_cutoff=cutoff).to(DEV)
    with torch.no_grad():
        mod.bias.normal_()
    plan, psi = mod.plan(DEV), D.get_psi(*mod._key)
    wins = DD.disco_windows(psi, mbd.compute_split_shapes(mod.nlat_in, h))
    x = torch.randn(2, 4, *ish, device=DEV)
    gy = torch.randn(2 * 6, *osh, device=DEV)
    # backward: each rank's window contraction of the rows of gy it gathers is the slice of the single-GPU contraction, bit for bit
    gY = plan.forward(gy.view(12, 1, *osh)).view(12, 9, *ish)
    for win in wins:
        part = _ops(mod._key, win).contract(gy[:, win.lo : win.hi])
        assert torch.equal(part.view(torch.int32), gY[:, :, win.t0 : win.t1].contiguous().view(torch.int32)), (h, win.t0)
    # forward: the module's GEMM, the window adjoints added into the owners' rows in rank order, bias
    Y = torch.matmul(D._transposed_mix(mod.weight, 2), x.view(2, 2, 2, -1)).view(12, 9, *ish)
    y = torch.zeros(12, *osh, device=DEV)
    for win in wins:
        y[:, win.lo : win.hi] += _ops(mod._key, win).adjoint(Y[:, :, win.t0 : win.t1].contiguous())
    y = y.view(2, 6, *osh) + mod.bias.view(1, -1, 1, 1)
    ys = mod(x)
    rel = ((y - ys).abs().max() / ys.abs().max()).item()
    print(f"\nvirtual ranks h = {h} {ish}->{osh}: y rel {rel:.3g}")
    assert rel <= 2e-6, rel

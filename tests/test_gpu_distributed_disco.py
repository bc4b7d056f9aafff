"""The CUDA per-rank stages of DistributedDiscreteContinuousConvS2 and DistributedResampleS2 on one GPU, h x w virtual ranks in one process:

* X of every rank's window plan is bit-identical to the corresponding slice of the single-GPU X, at fp32 and bf16 input, at FCN3's encoder
  (721 x 1440 -> 360 x 720) and processor (360 x 720 Legendre-Gauss) geometries, h in {2, 4}, w in {1, 2} (w splits the rows of B*C);
* dx of the window adjoints, added in rank order as the halo's adjoint adds them, stays within the bound of tests/test_gpu_disco.py
  (c n 2^-24 sum |psi| |dX|) against an fp64 contraction of the plan's fp32 psi_hat, and is identical run to run;
* the module's arithmetic on every rank (window contraction, the pixels of the rank, grouped GEMM and bias; transposes and halo as slicing)
  against the single-GPU module: y, dx, dW and dbias at fp32 (rtol 1e-5) and TF32 (relative L2 < 5e-3);
* the resampling's forward and adjoint over the planes of every rank bit-identical to the single-GPU kernels at FCN3's decoder shape
  (360 x 720 Legendre-Gauss -> 721 x 1440, 585 planes, 4 x 2).
The modules themselves (DistributedDiscreteContinuousConvS2 and its autograd function, DistributedResampleS2) need process groups and do not run
here: the module-level test above runs their per-rank arithmetic with the CUDA stages, re-composed in one process.  The modules with their
collectives and autograd are covered on CPU, with oracle stages, by tests/test_distributed_disco_cpu.py and
tests/reference_suites/run_reference_distributed_fcn3.py."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import makani_b200.distributed as mbd
from makani_b200 import disco as D
from makani_b200 import resample as R
from makani_b200.distributed import disco as DD
from makani_b200.distributed.resample import CudaResampleLocalOps
from oracle import makani_disco_oracle as O
from test_gpu_disco import C_SUM, TF32_REL_L2, _dense32, _rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

FCN3 = {
    "encoder": ((721, 1440), (360, 720), "equiangular", "legendre-gauss", (3 + 1) * 0.5 * math.pi / 720),
    "processor": ((360, 720), (360, 720), "legendre-gauss", "legendre-gauss", 2 * (3 + 1) * 0.5 * math.pi / 359),
}


def _key(ish, osh, gi, go, cutoff, kernel_shape=(3, 3), norm="mean"):
    return (tuple(kernel_shape), "morlet", norm, tuple(ish), tuple(osh), gi, go, float(cutoff))


def _ops(key, window):
    return DD.CudaDiscoLocalOps(SimpleNamespace(_key=key, window=window))


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("w", [1, 2])
@pytest.mark.parametrize("h", [2, 4])
@pytest.mark.parametrize("what", ["encoder", "processor"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_window_X_is_the_single_gpu_slice(dtype, what, h, w):
    key = _key(*FCN3[what])
    psi = D.get_psi(*key)
    (hi, wi), (ho, wo) = key[3], key[4]
    BC = 6
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(BC, hi, wi, generator=g, device=DEV).to(dtype)
    Xs = D.get_plan(key, DEV).forward(x.view(BC, 1, hi, wi)).view(BC, psi.kernel_size, ho, wo)
    wins = DD.disco_windows(psi, mbd.compute_split_shapes(ho, h))
    assert wins[0].lo == 0 and wins[-1].hi == hi
    r0 = 0
    for rows in mbd.compute_split_shapes(BC, w):
        for win in wins:
            X = _ops(key, win).contract(x[r0 : r0 + rows, win.lo : win.hi])
            assert torch.equal(_bits(X), _bits(Xs[r0 : r0 + rows, :, win.t0 : win.t1])), (what, h, w, win.t0, win.lo, win.hi)
        r0 += rows


def _summed_adjoint(key, wins, dX):
    """every rank's window adjoint, added into the owners' rows in rank order (the order of halo_adjoint)"""
    (hi, wi) = key[3]
    dx = torch.zeros(dX.shape[0], hi, wi, device=DEV)
    for win in wins:
        dx[:, win.lo : win.hi] += _ops(key, win).adjoint(dX[:, :, win.t0 : win.t1].contiguous())
    return dx


@pytest.mark.parametrize("h", [2, 3, 4])
@pytest.mark.parametrize("geom", [((91, 180), (46, 90), "equiangular", "legendre-gauss", 6.0), ((33, 64), (33, 64), "equiangular", "equiangular", 5.0)])
def test_summed_window_adjoints_within_bound_and_deterministic(geom, h):
    ish, osh, gi, go, u = geom
    key = _key(ish, osh, gi, go, u * math.pi / (ish[0] - 1))
    psi = D.get_psi(*key)
    (hi, wi), (ho, wo), K = ish, osh, psi.kernel_size
    wins = DD.disco_windows(psi, mbd.compute_split_shapes(ho, h))
    dX = torch.randn(7, K, ho, wo, generator=torch.Generator(device=DEV).manual_seed(9), device=DEV)
    dx = _summed_adjoint(key, wins, dX)
    assert torch.equal(dx, _summed_adjoint(key, wins, dX))
    P = _dense32(psi)
    ref = O.adjoint(dX.double().unsqueeze(1), P, hi, wi)[:, 0]
    mag = O.adjoint(dX.double().abs().unsqueeze(1), P.abs(), hi, wi)[:, 0]
    n_a = int(np.bincount(psi.col // wi, minlength=hi).max())
    need = ((dx.double() - ref).abs() / (n_a * 2.0**-24 * mag + 1e-300)).max().item()
    print(f"\nC needed, window adjoints summed over {h} ranks {ish}->{osh}: {need:.3g}")
    assert need <= C_SUM, need


class _Contract(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xwin, ops):
        ctx.ops = ops
        return ops.contract(xwin)

    @staticmethod
    def backward(ctx, g):
        return ctx.ops.adjoint(g.contiguous()), None


def emulated_conv(mod, x, h, w):
    """the forward of DistributedDiscreteContinuousConvS2 on h x w virtual ranks: rows of B*C split over w, halo and transposes as slicing"""
    B, C = x.shape[:2]
    psi = D.get_psi(*mod._key)
    wins = DD.disco_windows(psi, mbd.compute_split_shapes(mod.nlat_out, h))
    rows = x.reshape(B * C, mod.nlat_in, mod.nlon_in)
    Wg = D._grouped(mod.weight, mod.groups)
    out = []
    for win in wins:
        X = torch.cat([_Contract.apply(r[:, win.lo : win.hi], _ops(mod._key, win))
                       for r in torch.split(rows, mbd.compute_split_shapes(B * C, w))])                  # (B*C, K, t1 - t0, nlon_out)
        ys = []
        for Xp in torch.split(X, mbd.compute_split_shapes(mod.nlon_out, w), dim=-1):              # the pixels of rank (ih, iw)
            nt, nl = Xp.shape[-2:]
            y = torch.matmul(Wg, Xp.reshape(B, mod.groups, -1, nt * nl)).view(B, -1, nt, nl)
            ys.append(y + mod.bias.view(1, -1, 1, 1) if mod.bias is not None else y)
        out.append(torch.cat(ys, dim=-1))
    return torch.cat(out, dim=-2)


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("h,w", [(2, 1), (2, 2), (4, 2)])
@pytest.mark.parametrize("case", [(6, 8, (91, 180), (46, 90), 2, True, "equiangular", "legendre-gauss"),
                                  (5, 7, (46, 90), (46, 90), 1, False, "legendre-gauss", "legendre-gauss")])
def test_virtual_ranks_match_single_gpu_module(case, h, w, tf32):
    cin, cout, ish, osh, G, bias, gi, go = case
    torch.manual_seed(11)
    kw = dict(basis_type="morlet", groups=G, grid_in=gi, grid_out=go, bias=bias, theta_cutoff=5 * math.pi / (ish[0] - 1))
    mod = D.DiscreteContinuousConvS2(cin, cout, ish, osh, (3, 3), **kw).to(DEV)
    if bias:
        with torch.no_grad():
            mod.bias.normal_()
    x = torch.randn(2, cin, *ish, device=DEV)
    gy = torch.randn(2, cout, *osh, device=DEV)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        grads = []
        for f in (mod, lambda t: emulated_conv(mod, t, h, w)):
            mod.zero_grad()
            xd = x.clone().requires_grad_(True)
            y = f(xd)
            y.backward(gy)
            grads.append([y.detach(), xd.grad, mod.weight.grad.clone()] + ([mod.bias.grad.clone()] if bias else []))
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    for what, a, b in zip(("y", "dx", "dw", "db"), grads[1], grads[0]):
        if tf32:
            rel = _rel_l2(a, b.double().cpu())
            print(f"\nTF32 rel L2 {h}x{w} {ish}->{osh} {what}: {rel:.3g}")
            assert rel < TF32_REL_L2, (what, rel)
        else:
            err = (a - b).abs().max().item()
            assert err <= 1e-5 * b.abs().max().item(), (what, err, b.abs().max().item())


def test_resample_ranks_bit_identical_at_decoder_shape():
    key = (360, 720, 721, 1440, "legendre-gauss", "equiangular")
    plan = R.get_plan(key, DEV)
    ops = CudaResampleLocalOps(SimpleNamespace(_key=key))
    g = torch.Generator(device=DEV).manual_seed(4)
    x = torch.randn(585, 360, 720, generator=g, device=DEV)
    dy = torch.randn(585, 721, 1440, generator=g, device=DEV)
    ys, dxs = plan.forward(x), plan.adjoint(dy)
    h, w, p0 = 4, 2, 0
    for ph in mbd.compute_split_shapes(585, h):
        for pw in mbd.compute_split_shapes(ph, w):
            sl = slice(p0, p0 + pw)
            assert torch.equal(_bits(ops.forward(x[sl])), _bits(ys[sl])), sl
            assert torch.equal(_bits(ops.adjoint(dy[sl])), _bits(dxs[sl])), sl
            p0 += pw
    assert p0 == 585

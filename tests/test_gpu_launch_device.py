"""Launches on a device other than the current one: with cuda:0 current, operators on cuda:1 tensors give bit for bit what they give with cuda:1
current.  The library keeps per-device state (scratch buffers, SM count, tensor-core setup) by the current device, so `_lib.call` makes the
stream's device current around each launch; this runs every kind of call path -- several launches on one stream (the SHT's analysis and
synthesis pairs, the bias gradient), the one-call SpectralConv entry points, plan creation (SHT, DISCO), and the norm kernels.  Needs two GPUs."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import makani_b200 as mb  # noqa: E402
from makani_b200.norm import InstanceNorm2d  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two CUDA devices")]

DEV = torch.device("cuda", 1)
NLAT, NLON, B, C = 33, 64, 2, 8


def _rand(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _sht(precision):
    f = mb.RealSHT(NLAT, NLON, precision=precision)
    i = mb.InverseRealSHT(NLAT, NLON, precision=precision)
    assert precision != "tf32" or f.plan(DEV).dft_ok       # the TF32 runs take the tiled synthesis pair
    x = _rand(B, C, NLAT, NLON, seed=1).to(DEV).requires_grad_(True)
    bias = _rand(1, C, 1, 1, seed=2).to(DEV).requires_grad_(True)
    y = i.forward_packed(f.forward_packed(x), B, C, torch.float32, bias=bias)      # packed analysis + synthesis, bias in the epilogue
    z = i(f(x))                                                                      # through the complex (B, C, L, M) coefficients
    ((y * _rand(*y.shape, seed=3).to(DEV)).sum() + (z * _rand(*z.shape, seed=4).to(DEV)).sum()).backward()
    return y, z, x.grad, bias.grad


def _spectral_conv(precision):
    f = mb.RealSHT(NLAT, NLON, precision=precision)
    i = mb.InverseRealSHT(NLAT, NLON, precision=precision)
    torch.manual_seed(5)
    conv = mb.SpectralConv(f, i, C, C, operator_type="dhconv", bias=True, precision=precision).to(DEV)
    x = _rand(B, C, NLAT, NLON, seed=6).to(DEV).requires_grad_(True)
    y, _ = conv(x)
    y.backward(_rand(*y.shape, seed=7).to(DEV))
    return y, x.grad, conv.weight.grad, conv.bias.grad


def _disco():
    torch.manual_seed(8)
    conv = mb.DiscreteContinuousConvS2(4, 6, (NLAT, NLON), (17, 32), (3, 3), basis_type="morlet", groups=2, grid_in="equiangular",
                                       grid_out="legendre-gauss", theta_cutoff=0.3).to(DEV)
    x = _rand(B, 4, NLAT, NLON, seed=9).to(DEV).requires_grad_(True)
    y = conv(x)
    y.backward(_rand(*y.shape, seed=10).to(DEV))
    return y, x.grad, conv.weight.grad, conv.bias.grad


def _instance_norm():
    nrm = InstanceNorm2d(C, eps=1e-6, affine=True).to(DEV)
    with torch.no_grad():
        nrm.weight.copy_(_rand(C, seed=11))
        nrm.bias.copy_(_rand(C, seed=12))
    x = _rand(B, C, NLAT, NLON, seed=13).to(DEV).requires_grad_(True)
    y = nrm(x, gelu=True)
    y.backward(_rand(*y.shape, seed=14).to(DEV))
    return y, x.grad, nrm.weight.grad, nrm.bias.grad


CASES = {
    "sht-fp32": lambda: _sht("fp32"),
    "sht-tf32": lambda: _sht("tf32"),
    "spectral_conv-fp32": lambda: _spectral_conv("fp32"),
    "spectral_conv-tf32": lambda: _spectral_conv("tf32"),
    "disco": _disco,
    "instance_norm": _instance_norm,
}


@pytest.mark.parametrize("case", list(CASES))
def test_other_device_matches_current_device(case):
    with torch.cuda.device(0):
        other = CASES[case]()
        torch.cuda.synchronize(DEV)
        assert torch.cuda.current_device() == 0
    with torch.cuda.device(DEV):
        same = CASES[case]()
        torch.cuda.synchronize(DEV)
    for k, (a, b) in enumerate(zip(other, same)):
        assert a.device == DEV and torch.equal(a, b), f"{case}: output {k} differs from the run with cuda:1 current"

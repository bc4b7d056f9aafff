"""GPU parity of the tensor-core (TF32) path: same checks as test_gpu_parity.py at the tolerance BASELINE.json states for the
reduced-precision path (rtol 1e-3), plus kernel-by-kernel agreement with the fp32 CUDA-core kernels."""
import os
import subprocess
import sys

import pytest
import torch

import makani_b200 as mb
from test_gpu_parity import CONV_CASES, SHT_CASES, _run_conv_case, close, oracle_pair

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tcgen05_path_is_available():
    plan = mb.get_plan(33, 64, 16, 17, "equiangular", True, torch.device(DEV))
    assert plan.umma_ok, "tensor-core path unavailable on this device"


@pytest.mark.parametrize("case", ["small", "odd", "tiles", "wide", "cfg2c"])
def test_umma_kernels_agree_with_fp32_kernels(case):
    """each tensor-core kernel against the fp32 CUDA-core kernel on identical inputs (own process: a trap cannot poison the suite)"""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "umma_diag.py"), "all", case], capture_output=True, text=True, timeout=900)
    print(r.stdout[-3000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-1000:]


@pytest.mark.parametrize("grid,nlat,nlon,lmax,mmax,B,C", SHT_CASES)
def test_real_sht_tf32(grid, nlat, nlon, lmax, mmax, B, C):
    torch.manual_seed(333)
    sht = mb.RealSHT(nlat, nlon, lmax, mmax, grid, precision="tf32")
    isht = mb.InverseRealSHT(nlat, nlon, sht.lmax, sht.mmax, grid, precision="tf32")
    osht, oisht = oracle_pair(nlat, nlon, nlat, nlon, sht.lmax, sht.mmax, grid, grid)
    x = torch.randn(B, C, nlat, nlon)
    close(sht(x.to(DEV)), osht(x.double()), 1e-3, f"RealSHT tf32 {grid} {nlat}x{nlon}")
    cin = torch.randn(B, C, sht.lmax, sht.mmax, dtype=torch.complex64)
    close(isht(cin.to(DEV)), oisht(cin.to(torch.complex128)), 1e-3, f"InverseRealSHT tf32 {grid} {nlat}x{nlon}")


@pytest.mark.parametrize("case", CONV_CASES[:3])
def test_spectral_conv_fwd_bwd_tf32(case):
    _run_conv_case(case, "tf32", 1e-3)


# more than 256 channels: the mix GEMMs split their columns into several equal tiles (ragged last tile, 300 != 330)
WIDE_CASE = (24, 48, "legendre-gauss", 24, 48, "legendre-gauss", 16, 17, 1, 300, 330, 1, "dhconv", False, True)


def test_spectral_conv_many_channels_tf32():
    _run_conv_case(WIDE_CASE, "tf32", 1e-3)


def test_spectral_conv_bf16_tf32():
    _run_conv_case(CONV_CASES[1], "tf32", 1e-3, act_dtype=torch.bfloat16)

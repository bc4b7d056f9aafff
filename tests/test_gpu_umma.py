"""GPU parity of the tensor-core (TF32) path: same checks as test_gpu_parity.py at the tolerance BASELINE.json states for the
reduced-precision path (rtol 1e-3).  The tensor-core kernels one by one, against fp64 references of their exact operands, are in
test_gpu_engine.py."""
import pytest
import torch

import makani_b200 as mb
from makani_b200 import _lib
from test_gpu_parity import CONV_CASES, SHT_CASES, _run_conv_case, close, oracle_pair

pytestmark = pytest.mark.gpu
DEV = "cuda"


def test_tcgen05_path_is_available():
    plan = mb.get_plan(33, 64, 16, 17, "equiangular", True, torch.device(DEV))
    assert plan.umma_ok, "tensor-core path unavailable on this device"


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


# grouped dhconv whose group slices and batch the tensor-core mix addresses (G = 2, 16 -> 24 channels, B = 4)
GROUPED_TC_CASE = (48, 96, "legendre-gauss", 48, 96, "legendre-gauss", 32, 33, 4, 16, 24, 2, "dhconv", False, True)


@pytest.mark.parametrize("case", CONV_CASES[:3] + [GROUPED_TC_CASE])
def test_spectral_conv_fwd_bwd_tf32(case):
    if case == GROUPED_TC_CASE:
        B, Cin, Cout, G = case[8:12]
        assert _lib.load().b200sht_mix_uses_tensor_cores(_lib.OP_DHCONV, B, G, Cin, Cout, _lib.PREC_TF32) == 1
    _run_conv_case(case, "tf32", 1e-3)


# more than 256 channels: the mix GEMMs split their columns into several equal tiles (ragged last tile, 300 != 330)
WIDE_CASE = (24, 48, "legendre-gauss", 24, 48, "legendre-gauss", 16, 17, 1, 300, 330, 1, "dhconv", False, True)


def test_spectral_conv_many_channels_tf32():
    _run_conv_case(WIDE_CASE, "tf32", 1e-3)


def test_spectral_conv_bf16_tf32():
    _run_conv_case(CONV_CASES[1], "tf32", 1e-3, act_dtype=torch.bfloat16)

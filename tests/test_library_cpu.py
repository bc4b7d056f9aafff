"""CPU tests of the C-ABI library and the host logic: the .so loads and exports every declared symbol, and the
__host__ __device__ FFT / Legendre-recurrence code (the same code the kernels run) matches numpy / the oracle."""
import ctypes

import numpy as np
import pytest
import torch

from makani_b200 import _lib, quadrature
from oracle import makani_oracle as O

_VP = ctypes.c_void_p


def _p(a):
    return a.ctypes.data_as(_VP)


def test_library_loads_and_exports_all_declared_symbols():
    lib = _lib.load()
    names = _lib.declared_symbols()
    assert len(names) >= 30
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing
    assert lib.b200sht_version() >= 100
    # every bound signature is declared in the header (the binding cannot drift from include/b200sht.h)
    assert set(_lib._SIGNATURES) <= set(names), set(_lib._SIGNATURES) - set(names)


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.B200ShtError):
        _lib.load()


def test_cpu_tensor_is_rejected():
    import makani_b200

    sht = makani_b200.RealSHT(16, 32)
    with pytest.raises(_lib.B200ShtError):
        sht(torch.randn(1, 2, 16, 32))


@pytest.mark.parametrize("N", [1440, 720, 480, 360, 128, 72, 64, 180, 256, 512, 2 * 7 * 11 * 13, 96, 10, 6, 2880])
def test_fft_plan_factorisation(N):
    lib = _lib.load()
    rad = np.zeros(20, dtype=np.int32)
    n = lib.b200sht_debug_fft_plan(N, _p(rad), 20)
    assert n > 0 and int(np.prod(rad[:n])) == N
    assert set(rad[:n].tolist()) <= {2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15, 16}
    assert list(rad[:n]) == sorted(rad[:n], reverse=True)


def test_fft_plan_rejects_large_primes():
    rad = np.zeros(20, dtype=np.int32)
    assert _lib.load().b200sht_debug_fft_plan(2 * 17, _p(rad), 20) < 0


@pytest.mark.parametrize("N,mmax", [(1440, 241), (480, 241), (720, 361), (128, 65), (72, 37), (360, 120), (64, 33), (2002, 100), (30, 16), (10, 6), (6, 2)])
def test_fft_host_code_matches_numpy(N, mmax):
    lib = _lib.load()
    rng = np.random.default_rng(333)
    a = rng.standard_normal(N).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    xa = np.zeros(2 * mmax, dtype=np.float32)
    xb = np.zeros(2 * mmax, dtype=np.float32)
    assert lib.b200sht_debug_fft_host(N, mmax, 0, _p(a), _p(b), _p(xa), _p(xb)) == 0
    ra = np.fft.rfft(a.astype(np.float64))[:mmax]
    rb = np.fft.rfft(b.astype(np.float64))[:mmax]
    scale = np.sqrt(N)
    assert np.abs(xa.view(np.complex64) - ra).max() / scale < 3e-6
    assert np.abs(xb.view(np.complex64) - rb).max() / scale < 3e-6
    # inverse: irfft(norm="forward") of a truncated spectrum; imaginary parts of m = 0 / Nyquist are ignored
    za = (rng.standard_normal(mmax) + 1j * rng.standard_normal(mmax)).astype(np.complex64)
    zb = (rng.standard_normal(mmax) + 1j * rng.standard_normal(mmax)).astype(np.complex64)
    ya = np.zeros(N, dtype=np.float32)
    yb = np.zeros(N, dtype=np.float32)
    assert lib.b200sht_debug_fft_host(N, mmax, 1, _p(za.view(np.float32)), _p(zb.view(np.float32)), _p(ya), _p(yb)) == 0
    ea = torch.fft.irfft(torch.from_numpy(za.astype(np.complex128)), n=N, norm="forward").numpy()
    eb = torch.fft.irfft(torch.from_numpy(zb.astype(np.complex128)), n=N, norm="forward").numpy()
    tol = 3e-6 * np.sqrt(mmax) * 4
    assert np.abs(ya - ea).max() < tol and np.abs(yb - eb).max() < tol


@pytest.mark.parametrize("grid,nlat,lmax,mmax", [("equiangular", 33, 20, 21), ("legendre-gauss", 48, 48, 25), ("equiangular", 91, 91, 46)])
def test_table_host_code_matches_oracle(grid, nlat, lmax, mmax):
    lib = _lib.load()
    cost, w = quadrature._grid_np(nlat, grid)
    tab = np.zeros((mmax, lmax, nlat), dtype=np.float32)
    assert lib.b200sht_debug_table_host(nlat, lmax, mmax, _p(np.ascontiguousarray(cost)), 1, _p(tab)) == 0
    th, _ = O.precompute_latitudes(nlat, grid)
    ref = O.legpoly(mmax, lmax, np.cos(th))
    assert np.abs(tab - ref).max() < 2e-6
    # without the Condon-Shortley phase the odd orders flip sign
    tab2 = np.zeros_like(tab)
    lib.b200sht_debug_table_host(nlat, lmax, mmax, _p(np.ascontiguousarray(cost)), 0, _p(tab2))
    assert np.array_equal(tab2[1::2], -tab[1::2]) and np.array_equal(tab2[0::2], tab[0::2])


def test_table_host_large_orders_underflow_gracefully():
    lib = _lib.load()
    cost, _ = quadrature._grid_np(721, "equiangular")
    tab = np.zeros((241, 240, 721), dtype=np.float32)
    assert lib.b200sht_debug_table_host(721, 240, 241, _p(np.ascontiguousarray(cost)), 1, _p(tab)) == 0
    assert np.isfinite(tab).all()
    ref = O.legpoly(241, 240, cost)
    assert np.abs(tab - ref).max() < 5e-6


@pytest.mark.parametrize("grid", ["equiangular", "legendre-gauss"])
def test_quadrature_module_matches_oracle(grid):
    for n in (32, 33, 240, 721):
        th, w = quadrature.precompute_latitudes(n, grid)
        tho, wo = O.precompute_latitudes(n, grid)
        assert isinstance(th, torch.Tensor) and th.dtype == torch.float64
        assert np.abs(th.numpy() - tho).max() < 1e-12 and np.abs(w.numpy() - wo).max() < 1e-13
    x, w = quadrature.clenshaw_curtiss_weights(33)
    xo, wo = O.clenshaw_curtiss_weights(33)
    assert np.allclose(x.numpy(), xo) and np.allclose(w.numpy(), wo, atol=1e-14)
    x, w = quadrature.legendre_gauss_weights(33)
    assert abs(w.sum().item() - 2.0) < 1e-12


def test_spectral_conv_constructor_contract():
    """Parameter names / shapes / tags and ValueErrors of the reference ctor (spectral_convolution.py:116-211)."""
    import makani_b200 as mb

    f = mb.RealSHT(33, 64, lmax=16, mmax=17, grid="equiangular")
    i = mb.InverseRealSHT(24, 48, lmax=16, mmax=17, grid="legendre-gauss")
    conv = mb.SpectralConv(f, i, 6, 4, num_groups=2, operator_type="dhconv", bias=True)
    assert conv.weight.shape == (2, 3, 2, 16) and conv.weight.dtype == torch.complex64
    assert conv.weight.is_shared_mp == ["matmul", "w"] and conv.weight.sharded_dims_mp == [None, None, None, "h"]
    assert conv.bias.shape == (1, 4, 1, 1) and conv.bias.is_shared_mp == ["model"]
    assert conv.scale_residual and set(dict(conv.named_parameters())) == {"weight", "bias"}
    assert not list(conv.state_dict().keys() - {"weight", "bias"})  # no transform tables in checkpoints
    d = mb.SpectralConv(f, i, 6, 6, operator_type="diagonal")
    assert d.weight.shape == (1, 6, 6, 16, 17) and d.weight.sharded_dims_mp == [None, None, None, "h", "w"]
    s = mb.SpectralConv(f, i, 6, 6, operator_type="dhconv", separable=True)
    assert s.weight.shape == (1, 6, 16)
    with pytest.raises(ValueError):
        mb.SpectralConv(f, i, 5, 4, num_groups=2)
    with pytest.raises(ValueError):
        mb.SpectralConv(f, i, 4, 4, operator_type="nope")
    with pytest.raises(ValueError):
        mb.SpectralConv(f, mb.InverseRealSHT(24, 48, lmax=12, mmax=13), 4, 4)
    a = mb.SpectralAttention(f, i, 4, 6, operator_type="l-dependant", spectral_layers=2, bias=True, complex_activation="modulus")
    assert a.w[0].shape == (16, 4, 8) and a.w[1].shape == (16, 8, 8) and a.wout.shape == (16, 8, 6) and a.b[0].shape == (8, 1, 1)
    assert a.activations[0].bias.shape == (8, 1, 1)
    # default mode counts follow torch-harmonics: lmax = nlat, mmax = nlon // 2 + 1
    t = mb.RealSHT(64, 128)
    assert (t.lmax, t.mmax, t.grid) == (64, 65, "equiangular")


def test_mix_tensor_core_shape_query_and_pdl_switch():
    """pure host logic of the C ABI: which shapes the tcgen05 mix serves (the caller then packs the weight for that precision), workspace sizes of the
    pointwise kernels, and the run-time PDL switch returns its previous value"""
    lib = _lib.load()
    q = lib.b200sht_mix_uses_tensor_cores
    assert q(_lib.OP_DHCONV, 1, 1, 73, 73, _lib.PREC_TF32) == 1
    assert q(_lib.OP_DHCONV, 32, 1, 384, 384, _lib.PREC_TF32) == 1
    assert q(_lib.OP_DHCONV, 3, 1, 73, 73, _lib.PREC_TF32) == 0        # batch must divide 32
    assert q(_lib.OP_DHCONV, 1, 2, 6, 6, _lib.PREC_TF32) == 0          # group slices of 3 channels are not 16-byte aligned
    assert q(_lib.OP_DHCONV, 1, 2, 8, 8, _lib.PREC_TF32) == 1
    assert q(_lib.OP_DIAGONAL, 1, 1, 73, 73, _lib.PREC_TF32) == 0      # per-mode operators are bandwidth bound: one (fp32) path
    assert q(_lib.OP_DHCONV, 1, 1, 73, 73, _lib.PREC_FP32) == 0
    assert q(_lib.OP_DHCONV | _lib.DENSE_FLAG, 1, 1, 73, 73, _lib.PREC_TF32) == 1
    w = lib.b200sht_pointwise_workspace_floats
    assert w(1, 384, 721 * 1440) >= 2 * 384 and w(1, 384, 721 * 1440) % (2 * 384) == 0
    assert w(2, 5, 63) == 2 * 10                                       # short rows: one split
    assert w(0, 5, 63) < 0
    old = lib.b200sht_debug_set_pdl(0)
    assert lib.b200sht_debug_set_pdl(old) == 0


def test_pointwise_modules_on_cpu_are_the_torch_operators():
    """makani_b200.norm / sfno.Conv1x1 on CPU tensors (oracle-backend reference arm, golden tests): PyTorch's own operators, same parameters and state dict"""
    import torch.nn as nn
    import torch.nn.functional as F

    from makani_b200 import norm as mnorm
    from makani_b200.sfno import Conv1x1, MLP

    torch.manual_seed(333)
    x = torch.randn(2, 6, 9, 14)
    m, r = mnorm.InstanceNorm2d(6, eps=1e-6, affine=True), nn.InstanceNorm2d(6, eps=1e-6, affine=True)
    assert list(m.state_dict()) == list(r.state_dict())
    assert torch.allclose(m(x), r(x)) and torch.allclose(m(x, gelu=True), F.gelu(r(x)))
    b = torch.randn(6)
    assert torch.allclose(mnorm.bias_gelu(x, b), F.gelu(x + b.view(1, -1, 1, 1)))
    c = Conv1x1(6, 10, 1, bias=True)
    assert torch.allclose(c(x), F.conv2d(x, c.weight, c.bias), atol=1e-6)
    mlp = MLP(6, 12, act_layer=nn.GELU)
    assert list(mlp.state_dict()) == ["fwd.0.weight", "fwd.0.bias", "fwd.3.weight", "fwd.3.bias"]
    ref = F.conv2d(F.gelu(F.conv2d(x, mlp.fwd[0].weight, mlp.fwd[0].bias)), mlp.fwd[3].weight, mlp.fwd[3].bias)
    assert torch.allclose(mlp(x), ref, atol=1e-5)

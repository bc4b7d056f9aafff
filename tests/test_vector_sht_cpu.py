"""CPU tests of the vector SHT (RealVectorSHT / InverseRealVectorSHT): the oracle's tables D = dP/dtheta and Q = m P / sin(theta) against
scipy's spherical harmonics, the library's host table recurrence (the same __host__ __device__ code the vector plan's build kernel runs)
against the oracle, and the oracle's transforms against the identities the contract implies (surface gradient, -r x grad g, round trip)."""
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy.special import sph_harm_y

import makani_b200 as mb
from makani_b200 import _lib
from oracle import makani_oracle as O
from oracle import makani_vector_oracle as V

_VP = ctypes.c_void_p
GRIDS = ["equiangular", "legendre-gauss"]


def _p(a):
    return a.ctypes.data_as(_VP)


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("csphase", [True, False])
def test_oracle_tables_match_scipy(grid, csphase):
    theta, _ = O.precompute_latitudes(19, grid)
    M, L = 14, 17
    D, Q = V.vector_legpoly(M, L, theta, csphase=csphase)
    s = np.sin(theta)
    inner = s > 1e-12
    for m in range(M):
        sgn = 1.0 if (csphase or m % 2 == 0) else -1.0
        for l in range(L):
            y, g = sph_harm_y(l, m, theta, 0.0, diff_n=1)
            dref = sgn * np.real(g[..., 0]) if l >= m else np.zeros_like(theta)
            qref = sgn * m * np.real(y) / np.where(inner, s, 1.0) if l >= m else np.zeros_like(theta)
            np.testing.assert_allclose(D[m, l], dref, rtol=0, atol=1e-13, err_msg=f"D m={m} l={l}")
            np.testing.assert_allclose(Q[m, l][inner], qref[inner], rtol=0, atol=1e-13, err_msg=f"Q m={m} l={l}")
    assert not D[:, 0].any() and not Q[:, 0].any()


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("csphase", [True, False])
def test_host_vector_table_matches_oracle(grid, csphase):
    nlat, L, M = 33, 33, 40
    theta, _ = O.precompute_latitudes(nlat, grid)
    cost = np.ascontiguousarray(np.cos(theta))
    D = np.zeros((M, L, nlat), np.float32)
    Q = np.zeros_like(D)
    assert _lib.load().b200sht_debug_vector_table_host(nlat, L, M, _p(cost), int(csphase), _p(D), _p(Q)) == 0
    Dr, Qr = V.vector_legpoly(M, L, theta, csphase=csphase)
    for got, ref, name in ((D, Dr, "D"), (Q, Qr, "Q")):
        err = np.abs(got.astype(np.float64) - ref)
        assert (err <= 2 ** -23 * np.abs(ref) + 1e-6 * np.abs(ref).max()).all(), (name, err.max())


def test_host_vector_table_large_orders_near_poles():
    """721 latitudes (equiangular, poles included) at the largest orders: finite values, exact zeros for l < m"""
    nlat, L, M = 721, 721, 721
    theta, _ = O.precompute_latitudes(nlat, "equiangular")
    cost = np.ascontiguousarray(np.cos(theta))
    D = np.zeros((M, L, nlat), np.float32)
    Q = np.zeros_like(D)
    assert _lib.load().b200sht_debug_vector_table_host(nlat, L, M, _p(cost), 1, _p(D), _p(Q)) == 0
    assert np.isfinite(D).all() and np.isfinite(Q).all()
    lower = np.tril(np.ones((M, L), bool), -1)   # [m][l]: l < m
    assert not D[lower].any() and not Q[lower].any()
    # spot check against the oracle on a few orders, including the Nyquist-side ones
    for m in (0, 1, 2, 360, 719, 720):
        Dr, Qr = V.vector_legpoly(m + 1, L, theta)
        np.testing.assert_allclose(D[m], Dr[m], rtol=0, atol=2e-6 * max(1.0, np.abs(Dr[m]).max()))
        np.testing.assert_allclose(Q[m], Qr[m], rtol=0, atol=2e-6 * max(1.0, np.abs(Qr[m]).max()))


def _grid(nlat, nlon, grid):
    theta, _ = O.precompute_latitudes(nlat, grid)
    phi = 2 * math.pi * np.arange(nlon) / nlon
    return np.meshgrid(theta, phi, indexing="ij")


def _band_limited(nlat, nlon, L, M, seed, grid):
    g = torch.Generator().manual_seed(seed)
    c = torch.randn(3, L, M, dtype=torch.complex128, generator=g) * torch.tril(torch.ones(L, M, dtype=torch.float64))
    c[..., 0] = c[..., 0].real
    return c


@pytest.mark.parametrize("grid,nlat,nlon", [("equiangular", 33, 64), ("legendre-gauss", 32, 64)])
def test_oracle_gradient_identity(grid, nlat, nlon):
    """ivsht([f_lm, 0]) = (df/dtheta, df/dphi / sin theta): analytic Y_1^0, Re Y_2^1, and a random band-limited f through the scalar oracle"""
    T, P = _grid(nlat, nlon, grid)
    # truncated to 12 degrees: the Clenshaw-Curtis quadrature then integrates every product of the analysis exactly
    ivsht = V.InverseRealVectorSHT(nlat, nlon, 12, 12, grid=grid, dtype=torch.float64)
    sht = O.RealSHT(nlat, nlon, 12, 12, grid=grid, dtype=torch.float64)
    c10 = math.sqrt(3 / (4 * math.pi))
    c21 = -math.sqrt(15 / (8 * math.pi))   # Condon-Shortley phase
    fields = [
        (c10 * np.cos(T), -c10 * np.sin(T), 0 * T),
        (c21 * np.sin(T) * np.cos(T) * np.cos(P), c21 * np.cos(2 * T) * np.cos(P), -c21 * np.cos(T) * np.sin(P)),
    ]
    for f, dt, dp in fields:
        flm = sht(torch.from_numpy(f))
        u = ivsht(torch.stack([flm, torch.zeros_like(flm)]))
        np.testing.assert_allclose(u[0].numpy(), dt, atol=1e-10)
        np.testing.assert_allclose(u[1].numpy(), dp, atol=1e-10)
    # random band-limited f: the gradient's phi component times sin(theta) is the phi derivative of f, computed spectrally (i m f_m)
    L = 14   # well inside the band limit the equiangular quadrature integrates exactly
    c = _band_limited(nlat, nlon, L, nlon // 2 + 1, 7, grid)[0]
    ivsht = V.InverseRealVectorSHT(nlat, nlon, L, nlon // 2 + 1, grid=grid, dtype=torch.float64)
    isht = O.InverseRealSHT(nlat, nlon, L, nlon // 2 + 1, grid=grid, dtype=torch.float64)
    u = ivsht(torch.stack([c, torch.zeros_like(c)]))
    m = torch.arange(nlon // 2 + 1, dtype=torch.float64)
    dfdphi = isht(c * 1j * m)
    np.testing.assert_allclose((u[1] * torch.from_numpy(np.sin(T))).numpy(), dfdphi.numpy(), atol=1e-9)
    # its theta component integrates back: the spheroidal analysis of the gradient returns f (l >= 1)
    vsht = V.RealVectorSHT(nlat, nlon, L, nlon // 2 + 1, grid=grid, dtype=torch.float64)
    back = vsht(u)
    c0 = c.clone()
    c0[0] = 0
    assert (back[0] - c0).abs().max() < 1e-9 * c.abs().max() and back[1].abs().max() < 1e-9 * c.abs().max()


@pytest.mark.parametrize("grid", GRIDS)
def test_oracle_toroidal_identity(grid):
    """ivsht([0, g_lm]) = -r x grad g = (df/dphi / sin theta, -df/dtheta) for g = Re Y_2^1"""
    nlat, nlon = 33 if grid == "equiangular" else 32, 64
    T, P = _grid(nlat, nlon, grid)
    sht = O.RealSHT(nlat, nlon, 12, 12, grid=grid, dtype=torch.float64)
    ivsht = V.InverseRealVectorSHT(nlat, nlon, 12, 12, grid=grid, dtype=torch.float64)
    c21 = -math.sqrt(15 / (8 * math.pi))
    g = c21 * np.sin(T) * np.cos(T) * np.cos(P)
    gt, gp = c21 * np.cos(2 * T) * np.cos(P), -c21 * np.cos(T) * np.sin(P)
    glm = sht(torch.from_numpy(g))
    u = ivsht(torch.stack([torch.zeros_like(glm), glm]))
    np.testing.assert_allclose(u[0].numpy(), gp, atol=1e-10)
    np.testing.assert_allclose(u[1].numpy(), -gt, atol=1e-10)


@pytest.mark.parametrize("grid,nlat,nlon", [("equiangular", 33, 64), ("legendre-gauss", 32, 64), ("equiangular", 46, 90)])
def test_oracle_round_trip(grid, nlat, nlon):
    """vsht(ivsht(S, T)) = (S, T) on band-limited coefficients with zero l = 0 terms"""
    L, M = nlat // 2, nlon // 4
    g = torch.Generator().manual_seed(11)
    c = torch.randn(2, 2, L, M, dtype=torch.complex128, generator=g) * torch.tril(torch.ones(L, M, dtype=torch.float64))
    c[..., 0] = c[..., 0].real
    c[..., 0, :] = 0
    vsht = V.RealVectorSHT(nlat, nlon, L, M, grid=grid, dtype=torch.float64)
    ivsht = V.InverseRealVectorSHT(nlat, nlon, L, M, grid=grid, dtype=torch.float64)
    back = vsht(ivsht(c))
    assert (back - c).abs().max() < 1e-10 * c.abs().max()


def test_shim_exports_vector_classes():
    import sys

    from makani_b200 import compat

    saved = {k: sys.modules[k] for k in list(sys.modules) if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        th = compat.install_torch_harmonics_shim(force=True)
        assert th.RealVectorSHT is mb.RealVectorSHT and th.InverseRealVectorSHT is mb.InverseRealVectorSHT
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_module_attributes_and_defaults():
    v = mb.RealVectorSHT(32, 64)
    iv = mb.InverseRealVectorSHT(32, 64, lmax=20, mmax=10, grid="legendre-gauss", csphase=False)
    assert (v.nlat, v.nlon, v.lmax, v.mmax, v.grid, v.norm, v.csphase) == (32, 64, 32, 33, "equiangular", "ortho", True)
    assert (iv.lmax, iv.mmax, iv.grid, iv.csphase) == (20, 10, "legendre-gauss", False)
    with pytest.raises(NotImplementedError):
        mb.RealVectorSHT(32, 64, norm="schmidt")


def test_cpu_tensor_is_rejected():
    with pytest.raises(_lib.B200ShtError):
        mb.RealVectorSHT(16, 32)(torch.randn(1, 2, 16, 32))
    with pytest.raises(_lib.B200ShtError):
        mb.InverseRealVectorSHT(16, 32)(torch.zeros(1, 2, 16, 17, dtype=torch.complex64))

"""Transposed DISCO convolution on the CPU: the product's psi_T builder (`precompute_psi(..., transpose=True)`) against the independent fp64
oracle (tests/disco_transpose_oracle.py), the identities that pin the restated contract without torch-harmonics (the adjoint identity to the
forward convolution under the quadrature inner products, the constant field, longitude equivariance), the autograd function's channel mix
and gradients on oracle contractions, and the module's constructor contract and shim names.  Needs neither a GPU nor torch-harmonics."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import makani_b200 as mb  # noqa: E402
from makani_b200 import disco as D  # noqa: E402
from makani_b200._lib import B200ShtError  # noqa: E402
from makani_b200.quadrature import precompute_latitudes  # noqa: E402
from oracle import makani_disco_oracle as O  # noqa: E402
import disco_transpose_oracle as TO  # noqa: E402

# (in_shape, out_shape, grid_in, grid_out, cutoff in units of the out-grid spacing pi / (nlat_out - 1)): equal grids, s = 2 between equiangular
# grids, Legendre-Gauss <-> equiangular both ways
GEOMETRIES = [
    ((17, 32), (17, 32), "equiangular", "equiangular", 2.5),
    ((17, 32), (33, 64), "equiangular", "equiangular", 3.0),
    ((16, 32), (31, 64), "legendre-gauss", "equiangular", 3.0),
    ((21, 40), (20, 40), "equiangular", "legendre-gauss", 2.0),
]


def _cutoff(geom):
    return geom[4] * math.pi / (geom[1][0] - 1)


def _psi_T(geom, kernel_shape=(3, 3), norm="mean"):
    """the product's psi_T as a dense (K, nlat_in, nlat_out, nlon_out) array"""
    ish, osh, gi, go, _ = geom
    return D.psi_dense(D.precompute_psi(kernel_shape, "morlet", norm, osh, ish, go, gi, _cutoff(geom), True))


def _q(nlat, nlon, grid):
    """the quadrature weights 2 pi w / nlon of a grid as (nlat, 1)"""
    _, w = precompute_latitudes(nlat, grid)
    return torch.as_tensor(np.asarray(w), dtype=torch.float64)[:, None] * (2 * math.pi / nlon)


@pytest.mark.parametrize("geom", GEOMETRIES)
@pytest.mark.parametrize("kernel_shape", [(1, 1), (3, 3), (2, 3)])
@pytest.mark.parametrize("norm", D.NORM_MODES)
def test_builder_matches_oracle(geom, kernel_shape, norm):
    ish, osh, gi, go, _ = geom
    a = _psi_T(geom, kernel_shape, norm)
    b = TO.dense_psi_T(kernel_shape, norm, ish, osh, gi, go, _cutoff(geom)).numpy()
    assert a.shape == b.shape == (kernel_shape[0] * kernel_shape[1], ish[0], osh[0], osh[1])
    assert np.abs(a - b).max() <= 1e-12 * max(1.0, np.abs(a).max())


def test_forward_keys_and_psi_unchanged():
    """transpose=False is the forward builder: same 8-element key, same psi_hat bit for bit"""
    args = ((3, 3), "morlet", "mean", (17, 32), (9, 16), "equiangular", "legendre-gauss", 0.4)
    assert D._psi_key(*args) == D._psi_key(*args, transpose=False) and len(D._psi_key(*args)) == 8
    assert D._psi_key(*args, transpose=True) == D._psi_key(*args) + (True,)
    a, b = D.precompute_psi(*args), D.precompute_psi(*args, transpose=False)
    for f in ("row_ptr", "ker", "col", "val"):
        assert np.array_equal(getattr(a, f), getattr(b, f))


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_adjoint_to_forward_convolution(geom):
    """<y, z>_out = sum_k <Y_k, X_k>_in under the quadrature inner products, X the forward convolution's contraction of z from the out grid to
    the in grid (mode "none"): pins the geometry, the bearing and the quadrature of psi_T against the forward oracle"""
    ish, osh, gi, go, _ = geom
    K = 6
    psiT = torch.from_numpy(_psi_T(geom, (2, 3), "none")).reshape(K * ish[0], -1)
    psiF, _ = O.dense_psi((2, 3), "none", osh, ish, go, gi, _cutoff(geom))
    g = torch.Generator().manual_seed(4)
    Y = torch.randn(2, 3, K, *ish, dtype=torch.float64, generator=g)
    z = torch.randn(2, 3, *osh, dtype=torch.float64, generator=g)
    y = TO.transpose_contraction(Y, psiT, *osh)
    X = O.contraction(z, psiF.reshape(K * ish[0], -1), K, *ish)
    lhs = (y * z * _q(*osh, go)).sum()
    rhs = (Y * X * _q(*ish, gi)).sum()
    mag = (y.abs() * z.abs() * _q(*osh, go)).sum()
    assert abs(lhs - rhs) <= 1e-12 * mag, (lhs.item(), rhs.item())


@pytest.mark.parametrize("geom", [GEOMETRIES[0], ((16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 2.0)])
def test_constant_field_is_one(geom):
    """s = 1, "individual", morlet (1, 1): the transposed contraction of a constant is v / (v + 1e-9) = 1 up to the epsilon term"""
    ish, osh = geom[0], geom[1]
    psiT = torch.from_numpy(_psi_T(geom, (1, 1), "individual")).reshape(ish[0], -1)
    y = TO.transpose_contraction(torch.ones(1, 1, 1, *ish, dtype=torch.float64), psiT, *osh)
    raw = torch.from_numpy(_psi_T(geom, (1, 1), "none"))                           # psi (2 pi w_in / nlon_in) / (1 + 1e-9)
    v = raw.abs().sum(dim=(1, 3))[0] * (1 + D.NORM_EPS) * (ish[1] / osh[1])         # v[0, i]
    assert (v > 0).all()
    assert torch.allclose(y[0, 0], (v / (v + D.NORM_EPS))[:, None].expand(osh), rtol=0, atol=1e-12)
    assert (y - 1).abs().max() <= 2 * D.NORM_EPS / v.min()


def test_longitude_equivariance():
    """rolling the input by one in-grid longitude rolls the output by s = nlon_out / nlon_in out-grid longitudes"""
    geom = GEOMETRIES[1]
    ish, osh = geom[0], geom[1]
    s = osh[1] // ish[1]
    psiT = torch.from_numpy(_psi_T(geom, (2, 3))).reshape(6 * ish[0], -1)
    Y = torch.randn(2, 2, 6, *ish, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    y = TO.transpose_contraction(Y, psiT, *osh)
    for r in (1, 3):
        yr = TO.transpose_contraction(torch.roll(Y, r, dims=-1), psiT, *osh)
        assert torch.allclose(yr, torch.roll(y, s * r, dims=-1), rtol=0, atol=1e-14 * y.abs().max())


class _OraclePlan:
    """a stand-in for the device plan of psi_T: the oracle's transposed contraction as `adjoint`, its transpose as `forward` (fp64 inside)"""

    def __init__(self, psi, ish, osh):
        self.psi, self.K = psi, psi.shape[0] // ish[0]
        self.nlat_out, self.nlon_out, self.osh = ish[0], ish[1], osh

    def adjoint(self, Y, dtype=torch.float32):
        return TO.transpose_contraction(Y.double(), self.psi, *self.osh).to(dtype)

    def forward(self, gy):
        return O.contraction(gy.double(), self.psi, self.K, self.nlat_out, self.nlon_out).float()


@pytest.mark.parametrize("groups,bias,dtype", [(1, True, torch.float32), (2, False, torch.float32), (3, True, torch.bfloat16)])
def test_autograd_function_on_oracle_contractions(groups, bias, dtype):
    """the grouped channel mix, dx, dW and dbias of the module's autograd function, with the oracle's contractions in place of the kernels,
    against autograd through the oracle module"""
    geom = GEOMETRIES[2]
    ish, osh, gi, go, _ = geom
    cin, cout = 3 * groups, 2 * groups
    torch.manual_seed(5)
    ref = TO.DiscreteContinuousConvTransposeS2(cin, cout, ish, osh, (2, 2), basis_type="morlet", groups=groups, grid_in=gi, grid_out=go,
                                               bias=bias, theta_cutoff=_cutoff(geom)).double()
    if bias:
        with torch.no_grad():
            ref.bias.normal_()
    plan = _OraclePlan(ref.psi, ish, osh)
    x = torch.randn(2, cin, *ish).to(dtype)
    gy = torch.randn(2, cout, *osh, dtype=torch.float64)
    xr = x.double().requires_grad_(True)
    ref(xr).backward(gy)
    w = ref.weight.detach().float().requires_grad_(True)
    b = ref.bias.detach().float().requires_grad_(True) if bias else None
    xd = x.clone().requires_grad_(True)
    y = D._DiscoConvTranspose.apply(xd, w, b, plan, groups)
    y.backward(gy.float())
    assert y.dtype == torch.float32 and xd.grad.dtype == dtype
    pairs = [("y", y, ref(x.double())), ("dx", xd.grad, xr.grad), ("dw", w.grad, ref.weight.grad)] + ([("db", b.grad, ref.bias.grad)] if bias else [])
    for what, a, r in pairs:
        a, r = a.detach().double(), r.detach()
        tol = 1e-2 if (dtype == torch.bfloat16 and what == "dx") else 1e-5
        assert (a - r).abs().max() <= tol * r.abs().max(), what


def test_constructor_contract():
    torch.manual_seed(0)
    conv = D.DiscreteContinuousConvTransposeS2(12, 8, (17, 32), (33, 64), (3, 3), basis_type="morlet", groups=4, grid_in="legendre-gauss",
                                               theta_cutoff=0.3)
    assert conv.kernel_size == 9 and conv.groups == 4 and conv.groupsize == 3 and conv.kernel_shape == (3, 3)
    assert conv.basis_type == "morlet" and conv.basis_norm_mode == "mean" and conv.theta_cutoff == 0.3
    assert (conv.nlat_in, conv.nlon_in, conv.nlat_out, conv.nlon_out) == (17, 32, 33, 64)
    assert conv.weight.shape == (8, 3, 9) and conv.bias.shape == (8,) and not conv.bias.any()
    assert set(conv.state_dict()) == {"weight", "bias"}
    psi = D.get_psi(*conv._key)
    assert (psi.nlat_in, psi.nlon_in, psi.nlat_out, psi.nlon_out) == (33, 64, 17, 32)
    assert conv.psi_vals.shape == (len(psi.val),)
    big = D.DiscreteContinuousConvTransposeS2(64, 64, (17, 32), (17, 32), (3, 3), basis_type="morlet", bias=False, theta_cutoff=0.3)
    assert big.bias is None and set(big.state_dict()) == {"weight"}
    assert abs(big.weight.std().item() / math.sqrt(1 / 64 / 9) - 1) < 0.05
    conv.load_state_dict({"weight": torch.zeros(8, 3, 9), "bias": torch.ones(8)})
    for cutoff in (None, 0.0, -0.1):
        with pytest.raises(ValueError):
            D.DiscreteContinuousConvTransposeS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type="morlet", theta_cutoff=cutoff)
    for basis in ("piecewise linear", "zernike", "harmonic"):
        with pytest.raises(NotImplementedError, match=basis):
            D.DiscreteContinuousConvTransposeS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type=basis, theta_cutoff=0.3)
    with pytest.raises(NotImplementedError, match="nodal"):
        D.DiscreteContinuousConvTransposeS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type="morlet", basis_norm_mode="nodal", theta_cutoff=0.3)
    with pytest.raises(ValueError):
        D.DiscreteContinuousConvTransposeS2(6, 4, (17, 32), (17, 32), (3, 3), basis_type="morlet", groups=4, theta_cutoff=0.3)
    with pytest.raises(ValueError, match="multiple of nlon_in"):
        D.DiscreteContinuousConvTransposeS2(4, 4, (17, 32), (17, 48), (3, 3), basis_type="morlet", theta_cutoff=0.3)
    with pytest.raises(ValueError, match="multiple of nlon_in"):
        D.DiscreteContinuousConvTransposeS2(4, 4, (33, 64), (17, 32), (3, 3), basis_type="morlet", theta_cutoff=0.3)
    with pytest.raises(B200ShtError):
        conv(torch.randn(1, 12, 17, 32))


def test_shim_and_package_names():
    import importlib

    import makani_b200.compat as compat
    import makani_b200.distributed as mbd

    assert mb.DiscreteContinuousConvTransposeS2 is D.DiscreteContinuousConvTransposeS2
    assert D.DistributedDiscreteContinuousConvTransposeS2 is mbd.DistributedDiscreteContinuousConvTransposeS2
    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        th = compat.install_torch_harmonics_shim()
        assert th.DiscreteContinuousConvTransposeS2 is D.DiscreteContinuousConvTransposeS2
        thd = importlib.import_module("torch_harmonics.distributed")
        assert thd.DistributedDiscreteContinuousConvTransposeS2 is mbd.DistributedDiscreteContinuousConvTransposeS2
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_oracle_sparse_matches_dense():
    geom = GEOMETRIES[2]
    ish, osh, gi, go, _ = geom
    args = ((3, 3), "support", ish, osh, gi, go, _cutoff(geom))
    dense = TO.dense_psi_T(*args).reshape(9 * ish[0], -1)
    assert torch.equal(TO.sparse_psi_T(*args).to_dense(), dense)
    Y = torch.randn(1, 2, 9, *ish, dtype=torch.float64)
    assert torch.allclose(TO.transpose_contraction(Y, TO.sparse_psi_T(*args), *osh), TO.transpose_contraction(Y, dense, *osh),
                          rtol=1e-13, atol=1e-13)


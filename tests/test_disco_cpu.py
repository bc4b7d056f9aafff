"""DISCO convolution on the CPU: the product's psi_hat builder (makani_b200/disco.py) against the independent fp64 oracle
(oracle/makani_disco_oracle.py), and the identities that pin the restated contract without torch-harmonics: support, normalisation, longitude
equivariance, Funk-Hecke on the isotropic function, the adjoint identity.  Plus the module's constructor contract, the shim names and the build
log of the two kernels (no register spills).  Needs neither a GPU nor torch-harmonics."""
import math
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from makani_b200 import disco as D  # noqa: E402
from makani_b200._lib import B200ShtError  # noqa: E402
from makani_b200.quadrature import precompute_latitudes  # noqa: E402
from oracle import makani_disco_oracle as O  # noqa: E402
from oracle import makani_oracle as SO  # noqa: E402

# (in_shape, out_shape, grid_in, grid_out, cutoff in units of the input spacing pi / (nlat_in - 1))
GEOMETRIES = [
    ((17, 32), (17, 32), "equiangular", "equiangular", 2.5),
    ((17, 32), (9, 16), "equiangular", "legendre-gauss", 3.0),
    ((16, 32), (16, 16), "legendre-gauss", "legendre-gauss", 2.0),
    ((21, 40), (11, 20), "equiangular", "equiangular", 4.0),
]
KERNELS = [(1, 1), (3, 3), (5, 4), (2, 3)]


def _cutoff(in_shape, units):
    return units * math.pi / (in_shape[0] - 1)


def _psi(geom, kernel_shape=(3, 3), norm="mean"):
    ish, osh, gi, go, u = geom
    return D.precompute_psi(kernel_shape, "morlet", norm, ish, osh, gi, go, _cutoff(ish, u))


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_support_matches_haversine_distance(geom):
    """every entry lies within r_c of its output point, every grid point within r_c is present (pole rows included)"""
    ish, osh, gi, go, u = geom
    psi = _psi(geom)
    rc = (1 + D.CUTOFF_SLACK) * _cutoff(ish, u)
    th_i, _ = precompute_latitudes(ish[0], gi)
    th_o, _ = precompute_latitudes(osh[0], go)
    th_i, th_o = th_i.numpy(), th_o.numpy()
    lon = 2 * np.pi * np.arange(ish[1]) / ish[1]
    # haversine: 2 asin sqrt(sin^2(dlat / 2) + cos lat1 cos lat2 sin^2(dlon / 2)), latitudes = pi / 2 - colatitudes
    la_i, la_o = np.pi / 2 - th_i, np.pi / 2 - th_o
    hav = (np.sin((la_i[None, :, None] - la_o[:, None, None]) / 2) ** 2
           + np.cos(la_o)[:, None, None] * np.cos(la_i)[None, :, None] * np.sin(lon[None, None, :] / 2) ** 2)
    dist = 2 * np.arcsin(np.sqrt(np.clip(hav, 0, 1)))                                    # (nlat_out, nlat_in, nlon_in)
    present = np.zeros(dist.shape, dtype=bool)
    present.reshape(osh[0], -1)[D.psi_lat_out(psi), psi.col] = True
    inside = dist <= rc
    margin = np.abs(dist - rc) > 1e-12                                                   # no point sits on the boundary
    assert margin.all()
    assert np.array_equal(present, inside)
    # the pole rows of an equiangular output grid see whole input rows
    if go == "equiangular":
        assert present[0, 0].all() and present[-1, -1].all()
    # every k carries every support point
    counts = np.bincount(psi.ker, minlength=psi.kernel_size)
    assert (counts == inside.sum()).all()


@pytest.mark.parametrize("geom", GEOMETRIES)
@pytest.mark.parametrize("kernel_shape", KERNELS)
@pytest.mark.parametrize("norm", D.NORM_MODES)
def test_builder_matches_oracle(geom, kernel_shape, norm):
    ish, osh, gi, go, u = geom
    a = D.psi_dense(_psi(geom, kernel_shape, norm))
    b, _ = O.dense_psi(kernel_shape, norm, ish, osh, gi, go, _cutoff(ish, u))
    assert a.shape == tuple(b.shape)
    assert np.abs(a - b.numpy()).max() <= 1e-12 * max(1.0, np.abs(a).max())


def test_entries_sorted_by_output_latitude_then_point():
    psi = _psi(GEOMETRIES[1], (5, 4))
    for t in range(psi.nlat_out):
        s = slice(psi.row_ptr[t], psi.row_ptr[t + 1])
        key = psi.col[s].astype(np.int64) * psi.kernel_size + psi.ker[s]
        assert np.all(np.diff(key) > 0)


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_normalisation(geom):
    ish, osh, gi, go, u = geom
    a = np.abs(D.psi_dense(_psi(geom, (3, 3), "mean"))).sum(axis=(2, 3))                 # (K, nlat_out)
    assert np.allclose(a.mean(axis=1), 1.0, rtol=0, atol=1e-7)
    b = np.abs(D.psi_dense(_psi(geom, (3, 3), "individual"))).sum(axis=(2, 3))
    assert np.allclose(b, 1.0, rtol=0, atol=1e-7)
    # a constant field through k = 0 gives v[0, t] / mean_t v[0, t]
    psi = D.psi_dense(_psi(geom, (3, 3), "mean"))
    raw = D.psi_dense(_psi(geom, (3, 3), "none"))
    v = np.abs(raw[0]).sum(axis=(1, 2))
    out = psi[0].sum(axis=(1, 2))
    assert np.allclose(out, v / (v.mean() + D.NORM_EPS), rtol=1e-13, atol=0)


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_longitude_equivariance(geom):
    ish, osh = geom[0], geom[1]
    psi = torch.from_numpy(D.psi_dense(_psi(geom, (2, 3)))).reshape(6 * osh[0], -1)
    ps = ish[1] // osh[1]
    x = torch.randn(2, 3, *ish, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    X = O.contraction(x, psi, 6, *osh)
    for s in (1, 3):
        Xs = O.contraction(torch.roll(x, -ps * s, dims=-1), psi, 6, *osh)
        assert torch.allclose(Xs, torch.roll(X, -s, dims=-1), rtol=0, atol=1e-14 * X.abs().max())


def _funk_hecke(nlat, grid, l, m, cutoff):
    nlon = 2 * (nlat - 1) if grid == "equiangular" else 2 * nlat
    isht = SO.InverseRealSHT(nlat, nlon, l + 1, m + 1, grid, dtype=torch.float64)
    c = torch.zeros(l + 1, m + 1, dtype=torch.complex128)
    c[l, m] = 1.0
    f = isht(c)[None, None]
    psi = torch.from_numpy(D.psi_dense(D.precompute_psi((1, 1), "morlet", "none", (nlat, nlon), (nlat, nlon), grid, grid, cutoff))).reshape(nlat, -1)
    g = O.contraction(f, psi, 1, nlat, nlon)[0, 0, 0]
    lam = (g * f[0, 0]).sum() / (f * f).sum()
    return lam.item(), ((g - lam * f[0, 0]).norm() / g.norm()).item()


@pytest.mark.parametrize("grid", ["equiangular", "legendre-gauss"])
def test_funk_hecke_isotropic_kernel(grid):
    """the isotropic k = 0 function maps Y_l^m to lambda_l Y_l^m with lambda_l independent of m; the residual shrinks under refinement.
    This pins the distance formula and the north / south orientation of both grids."""
    cutoff, l = 0.35, 4
    res = {}
    for nlat in (33, 65):
        lams = []
        for m in (0, 2, 4):
            lam, r = _funk_hecke(nlat, grid, l, m, cutoff)
            lams.append(lam)
            res.setdefault(nlat, []).append(r)
        spread = (max(lams) - min(lams)) / abs(np.mean(lams))
        res[nlat].append(spread)
    assert max(res[65]) < 0.5 * max(res[33]), res
    assert max(res[65]) < 2e-2, res


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_adjoint_identity(geom):
    ish, osh = geom[0], geom[1]
    psi = torch.from_numpy(D.psi_dense(_psi(geom, (3, 3)))).reshape(9 * osh[0], -1)
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 2, *ish, dtype=torch.float64, generator=g)
    y = torch.randn(2, 2, 9, *osh, dtype=torch.float64, generator=g)
    lhs = (O.contraction(x, psi, 9, *osh) * y).sum()
    rhs = (x * O.adjoint(y, psi, *ish)).sum()
    assert abs(lhs - rhs) <= 1e-12 * abs(lhs)
    # and the oracle module's autograd agrees with the explicit adjoint
    xr = x.clone().requires_grad_(True)
    (O.contraction(xr, psi, 9, *osh) * y).sum().backward()
    assert torch.allclose(xr.grad, O.adjoint(y, psi, *ish), rtol=1e-12, atol=1e-14)


def test_constructor_contract():
    torch.manual_seed(0)
    conv = D.DiscreteContinuousConvS2(12, 8, (33, 64), (17, 32), (3, 3), basis_type="morlet", groups=4, grid_out="legendre-gauss",
                                      theta_cutoff=0.3)
    assert conv.kernel_size == 9 and conv.groups == 4 and conv.groupsize == 3
    assert (conv.nlat_in, conv.nlon_in, conv.nlat_out, conv.nlon_out) == (33, 64, 17, 32)
    assert conv.weight.shape == (8, 3, 9) and conv.bias.shape == (8,) and not conv.bias.any()
    assert set(conv.state_dict()) == {"weight", "bias"}
    big = D.DiscreteContinuousConvS2(64, 64, (17, 32), (17, 32), (3, 3), basis_type="morlet", bias=False, theta_cutoff=0.3)
    assert big.bias is None and set(big.state_dict()) == {"weight"}
    assert abs(big.weight.std().item() / math.sqrt(1 / 64 / 9) - 1) < 0.05
    # an FCN3 state dict loads into the same constructor
    conv.load_state_dict({"weight": torch.zeros(8, 3, 9), "bias": torch.ones(8)})
    with pytest.raises(ValueError):
        D.DiscreteContinuousConvS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type="morlet")
    for basis in ("piecewise linear", "zernike", "harmonic"):
        with pytest.raises(NotImplementedError, match=basis):
            D.DiscreteContinuousConvS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type=basis, theta_cutoff=0.3)
    with pytest.raises(NotImplementedError, match="nodal"):
        D.DiscreteContinuousConvS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type="morlet", basis_norm_mode="nodal", theta_cutoff=0.3)
    with pytest.raises(ValueError):
        D.DiscreteContinuousConvS2(4, 4, (17, 32), (17, 24), (3, 3), basis_type="morlet", theta_cutoff=0.3)
    with pytest.raises(B200ShtError):
        conv(torch.randn(1, 12, 33, 64))


def test_shim_names_resolve():
    import importlib

    import makani_b200.compat as compat

    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        th = compat.install_torch_harmonics_shim()
        assert th.DiscreteContinuousConvS2 is D.DiscreteContinuousConvS2
        fb = importlib.import_module("torch_harmonics.filter_basis")
        assert fb.get_filter_basis((3, 3), "morlet").kernel_size == 9 and th.filter_basis is fb
        with pytest.raises(NotImplementedError):
            fb.get_filter_basis((3, 3), "harmonic")
        thd = importlib.import_module("torch_harmonics.distributed")
        with pytest.raises(NotImplementedError, match="distributed DISCO"):
            thd.DistributedDiscreteContinuousConvS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type="morlet", theta_cutoff=0.3)
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc is not available")
def test_disco_kernels_do_not_spill():
    """every instantiation of the forward and the adjoint kernel keeps its accumulators in registers"""
    csrc = os.path.join(ROOT, "makani_b200", "csrc")
    log = os.path.join(ROOT, "makani_b200", "build", "disco.o.log")
    sources = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh"))]
    if os.path.exists(log) and os.path.getmtime(log) >= max(os.path.getmtime(s) for s in sources):
        report = open(log).read()
    else:
        from makani_b200 import build as _build

        nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
        with tempfile.TemporaryDirectory() as tmp:
            r = subprocess.run([nvcc] + _build.FLAGS + ["-c", os.path.join(csrc, "disco.cu"), "-o", os.path.join(tmp, "disco.o")],
                               capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        report = r.stdout + r.stderr
    pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?Function properties for \1\n\s+(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    kernels = {m.group(1): (int(m.group(3)), int(m.group(4))) for m in pat.finditer(report) if "disco_" in m.group(1)}
    assert sum("disco_forward_kernel" in k for k in kernels) == 8 and sum("disco_adjoint_kernel" in k for k in kernels) == 1, kernels
    spilling = {k: v for k, v in kernels.items() if v[0] or v[1]}
    assert not spilling, spilling

"""Neighbourhood attention on the CPU: the neighbourhood builder (makani_b200/attention.py) against the DISCO support of precompute_psi, the
invariants of the fp64 oracle (tests/attention_oracle.py) that pin the restated contract without torch-harmonics, the module's constructor
contract, the shim name and the build log of the kernels (no register spills).  Needs neither a GPU nor torch-harmonics."""
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
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import attention_oracle as AO  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200 import disco as D  # noqa: E402
from makani_b200._lib import B200ShtError  # noqa: E402
from makani_b200.quadrature import _grid_np  # noqa: E402

# (in_shape, out_shape, grid_in, grid_out, cutoff in units of the input spacing pi / (nlat_in - 1))
GEOMETRIES = [
    ((17, 32), (17, 32), "equiangular", "equiangular", 2.5),
    ((17, 32), (9, 16), "equiangular", "legendre-gauss", 3.0),
    ((16, 32), (16, 16), "legendre-gauss", "legendre-gauss", 2.0),
    ((21, 40), (11, 20), "equiangular", "equiangular", 4.0),
]


def _cutoff(in_shape, units):
    return units * math.pi / (in_shape[0] - 1)


def _nbhd(geom):
    ish, osh, gi, go, u = geom
    return A.neighbourhood(ish, osh, gi, go, _cutoff(ish, u))


def _omega(nlat, nlon, grid):
    return 2.0 * np.pi * _grid_np(nlat, grid)[1] / nlon


@pytest.mark.parametrize("geom", GEOMETRIES)
@pytest.mark.parametrize("kernel_shape", [(1, 1), (3, 3), (2, 3)])
def test_neighbourhood_is_the_disco_support(geom, kernel_shape):
    ish, osh, gi, go, u = geom
    nb = _nbhd(geom)
    psi = D.precompute_psi(kernel_shape, "morlet", "mean", ish, osh, gi, go, _cutoff(ish, u))
    first = psi.ker == 0
    assert np.array_equal(nb.row_ptr * psi.kernel_size, psi.row_ptr)
    assert np.array_equal(nb.col, psi.col[first]) and np.array_equal(D.psi_lat_out(nb), D.psi_lat_out(psi)[first])
    assert nb.kernel_size == 1 and not nb.ker.any()
    assert np.array_equal(nb.val, _omega(ish[0], ish[1], gi)[nb.col // ish[1]])


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_neighbourhood_ordered_and_symmetric(geom):
    ish = geom[0]
    nb = _nbhd(geom)
    for t in range(nb.nlat_out):
        c = nb.col[nb.row_ptr[t] : nb.row_ptr[t + 1]].astype(np.int64)
        assert len(c) and np.all(np.diff(c) > 0)                     # (i, j) order
        i, j = c // ish[1], c % ish[1]
        mirrored = np.sort(i * ish[1] + (-j) % ish[1])
        assert np.array_equal(mirrored, c)                           # symmetric in longitude


def test_poles_see_whole_rings():
    nb = A.neighbourhood((17, 32), (17, 32), "equiangular", "equiangular", 1.5 * math.pi / 16)
    c = nb.col[nb.row_ptr[0] : nb.row_ptr[1]]
    assert np.array_equal(c[c < 32], np.arange(32))                  # the north pole ring, every longitude


def _rand(*shape, seed=0):
    return torch.randn(*shape, dtype=torch.float64, generator=torch.Generator().manual_seed(seed))


def test_oracle_global_limit_is_sdpa():
    """theta_cutoff >= pi: every output point sees every input point, i.e. attention with the additive mask log w"""
    ish, osh, gi, go = (9, 16), (7, 8), "equiangular", "legendre-gauss"
    nb = A.neighbourhood(ish, osh, gi, go, math.pi)
    assert np.all(np.diff(nb.row_ptr) == ish[0] * ish[1])
    B, H, ek, ev = 2, 2, 3, 5
    q, k, v = _rand(B, 56, H * ek, seed=1), _rand(B, 144, H * ek, seed=2), _rand(B, 144, H * ev, seed=3)
    om = _omega(ish[0], ish[1], gi)
    y, lse = AO.attention(q, k, v, nb.row_ptr, nb.col, om, ish[1], osh[1], H, 0.7)
    mask = torch.from_numpy(np.log(np.repeat(om, ish[1]))).view(1, -1)
    split = lambda x, e: x.view(B, -1, H, e).transpose(1, 2)       # noqa: E731
    ref = F.scaled_dot_product_attention(split(q, ek), split(k, ek), split(v, ev), attn_mask=mask, scale=0.7)
    assert torch.allclose(y, ref.transpose(1, 2).reshape(B, -1, H * ev), rtol=1e-12, atol=1e-12)
    lref = torch.logsumexp(0.7 * split(q, ek) @ split(k, ek).transpose(-1, -2) + mask, -1)
    assert torch.allclose(lse, lref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("geom", GEOMETRIES[:2])
def test_oracle_zero_keys_give_the_disk_mean(geom):
    ish, osh, gi = geom[0], geom[1], geom[2]
    nb = _nbhd(geom)
    B, H, ev = 1, 2, 3
    v = _rand(B, ish[0] * ish[1], H * ev, seed=4)
    q = _rand(B, osh[0] * osh[1], H * 4, seed=5)
    k = torch.zeros(B, ish[0] * ish[1], H * 4, dtype=torch.float64)
    om = _omega(ish[0], ish[1], gi)
    y, _ = AO.attention(q, k, v, nb.row_ptr, nb.col, om, ish[1], osh[1], H, 1.0)
    for t in (0, osh[0] // 2, osh[0] - 1):
        p, n = AO.pairs(nb.row_ptr, nb.col, ish[1], osh[1], t)
        w = torch.from_numpy(om[n // ish[1]])
        for pp in (0, osh[1] - 1):
            sel = torch.from_numpy(p == pp)
            ref = (w[sel, None] * v[0, torch.from_numpy(n)[sel]]).sum(0) / w[sel].sum()
            assert torch.allclose(y[0, t * osh[1] + pp], ref, rtol=1e-13, atol=1e-14)


@pytest.mark.parametrize("geom", GEOMETRIES)
def test_oracle_longitude_equivariance(geom):
    ish, osh, gi = geom[0], geom[1], geom[2]
    nb = _nbhd(geom)
    s = ish[1] // osh[1]
    B, H, ek, ev = 2, 2, 4, 3
    q = _rand(B, *osh, H * ek, seed=6)
    k, v = _rand(B, *ish, H * ek, seed=7), _rand(B, *ish, H * ev, seed=8)
    om = _omega(ish[0], ish[1], gi)
    flat = lambda x: x.reshape(B, -1, x.shape[-1])                  # noqa: E731
    y, _ = AO.attention(flat(q), flat(k), flat(v), nb.row_ptr, nb.col, om, ish[1], osh[1], H, 0.5)
    for d in (1, 3):
        ys, _ = AO.attention(flat(torch.roll(q, d, 2)), flat(torch.roll(k, s * d, 2)), flat(torch.roll(v, s * d, 2)), nb.row_ptr, nb.col, om,
                             ish[1], osh[1], H, 0.5)
        ref = torch.roll(y.view(B, *osh, -1), d, 2).reshape(B, -1, H * ev)
        assert torch.allclose(ys, ref, rtol=1e-12, atol=1e-13)


def test_oracle_gradcheck():
    ish, osh, gi, go = (7, 8), (4, 4), "equiangular", "legendre-gauss"
    nb = A.neighbourhood(ish, osh, gi, go, 2.0 * math.pi / 6)
    om = _omega(ish[0], ish[1], gi)
    H, ek, ev = 2, 2, 3
    q = _rand(1, 16, H * ek, seed=9).requires_grad_(True)
    k = _rand(1, 56, H * ek, seed=10).requires_grad_(True)
    v = _rand(1, 56, H * ev, seed=11).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda q, k, v: AO.attention(q, k, v, nb.row_ptr, nb.col, om, ish[1], osh[1], H, 0.8), (q, k, v))


def test_constructor_contract():
    torch.manual_seed(0)
    att = A.NeighborhoodAttentionS2(12, (17, 32), (9, 16), grid_out="legendre-gauss", num_heads=4, theta_cutoff=0.5, k_channels=8,
                                    out_channels=20)
    assert (att.k_channels, att.out_channels, att.num_heads) == (8, 20, 4)
    assert att.scale == pytest.approx(1 / math.sqrt(2))
    shapes = {k: tuple(v.shape) for k, v in att.state_dict().items()}
    assert shapes == {"q_weights": (8, 12, 1, 1), "k_weights": (8, 12, 1, 1), "v_weights": (20, 12, 1, 1), "proj_weights": (20, 20, 1, 1),
                      "q_bias": (8,), "k_bias": (8,), "v_bias": (20,), "proj_bias": (20,)}
    assert not any(att.state_dict()[k].any() for k in ("q_bias", "k_bias", "v_bias", "proj_bias"))
    bound = math.sqrt(6 / (12 + 20))                                 # xavier-uniform of (20, 12, 1, 1)
    assert att.v_weights.abs().max() <= bound and att.v_weights.abs().max() > 0.8 * bound
    assert {n for n, _ in att.named_buffers()} == {"psi_row_ptr", "psi_col_idx", "quad_weights"}
    nob = A.NeighborhoodAttentionS2(8, (17, 32), (17, 32), bias=False, theta_cutoff=0.5, scale=0.25, optimized_kernel=False)
    assert set(nob.state_dict()) == {"q_weights", "k_weights", "v_weights", "proj_weights"} and nob.scale == 0.25
    with pytest.raises(ValueError, match="theta_cutoff"):
        A.NeighborhoodAttentionS2(8, (17, 32), (17, 32))
    with pytest.raises(ValueError, match="positive"):
        A.NeighborhoodAttentionS2(8, (17, 32), (17, 32), theta_cutoff=0.0)
    with pytest.raises(ValueError, match="divisible"):
        A.NeighborhoodAttentionS2(8, (17, 32), (17, 32), num_heads=3, theta_cutoff=0.5)
    with pytest.raises(ValueError, match="divisible"):
        A.NeighborhoodAttentionS2(8, (17, 32), (17, 32), num_heads=2, theta_cutoff=0.5, out_channels=5)
    with pytest.raises(ValueError, match="multiple"):
        A.NeighborhoodAttentionS2(8, (17, 32), (17, 24), theta_cutoff=0.5)
    with pytest.raises(ValueError, match="output latitude"):
        A.NeighborhoodAttentionS2(8, (17, 32), (16, 32), grid_out="legendre-gauss", theta_cutoff=0.01)
    with pytest.raises(NotImplementedError, match="64"):
        A.NeighborhoodAttentionS2(130, (17, 32), (17, 32), theta_cutoff=0.5)
    with pytest.raises(ValueError, match="in_shape == out_shape"):
        A.NeighborhoodAttentionS2(8, (17, 32), (9, 16), theta_cutoff=0.5)(torch.randn(1, 8, 9, 16))
    with pytest.raises(B200ShtError):
        nob(torch.randn(1, 8, 17, 32))
    # "zernike" keeps raising in the DISCO convolution: the neighbourhood does not go through the filter bases
    with pytest.raises(NotImplementedError, match="zernike"):
        D.DiscreteContinuousConvS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type="zernike", theta_cutoff=0.3)


def test_shim_name_resolves():
    import makani_b200 as mb
    import makani_b200.compat as compat

    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        th = compat.install_torch_harmonics_shim()
        assert th.NeighborhoodAttentionS2 is mb.NeighborhoodAttentionS2 is A.NeighborhoodAttentionS2
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_product_path_does_not_import_the_attention_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "makani_b200")):
        for f in files:
            if f.endswith(".py"):
                assert "attention_oracle" not in open(os.path.join(dirpath, f)).read(), f


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc is not available")
def test_attention_kernels_do_not_spill():
    """every instantiation of the three attention kernels keeps its rows and accumulators in registers"""
    csrc = os.path.join(ROOT, "makani_b200", "csrc")
    log = os.path.join(ROOT, "makani_b200", "build", "attention.o.log")
    sources = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh"))]
    if os.path.exists(log) and os.path.getmtime(log) >= max(os.path.getmtime(s) for s in sources):
        report = open(log).read()
    else:
        from makani_b200 import build as _build

        nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
        with tempfile.TemporaryDirectory() as tmp:
            r = subprocess.run([nvcc] + _build.FLAGS + ["-c", os.path.join(csrc, "attention.cu"), "-o", os.path.join(tmp, "attention.o")],
                               capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        report = r.stdout + r.stderr
    pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?Function properties for \1\n\s+(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    kernels = {m.group(1): (int(m.group(3)), int(m.group(4))) for m in pat.finditer(report) if "attn_" in m.group(1)}
    # head-dim classes 4 .. 64, vector and scalar paths: forward, query side, key/value side
    assert sum("attn_query_kernel" in k for k in kernels) == 20 and sum("attn_kv_kernel" in k for k in kernels) == 10, kernels
    spilling = {k: v for k, v in kernels.items() if v[0] or v[1]}
    assert not spilling, spilling

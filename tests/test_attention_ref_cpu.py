"""The exact-operand references of tests/attention_ref.py on the CPU: on fp64 operands (the scaled query taken as scale q) they are the
contract oracle of tests/attention_oracle.py, forward and autograd backward, and their bounds are well formed."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import attention_oracle as AO  # noqa: E402
import attention_ref as AR  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.quadrature import _grid_np  # noqa: E402

# (in_shape, out_shape, grid_in, grid_out, cutoff in input spacings or None for pi, B, heads, ek, ev): s = 1, 2, 3; pole rings; single-point
# neighbourhoods; the global limit
GEOMETRIES = [
    ((17, 32), (17, 32), "equiangular", "equiangular", 2.5, 2, 2, 3, 5),
    ((16, 96), (16, 32), "legendre-gauss", "legendre-gauss", 2.5, 1, 2, 4, 4),
    ((21, 40), (11, 20), "equiangular", "equiangular", 4.0, 1, 1, 8, 6),
    ((16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 0.05, 1, 3, 12, 16),
    ((9, 16), (7, 8), "equiangular", "legendre-gauss", None, 2, 2, 8, 3),
]


def _case(geom, seed=0):
    ish, osh, gi, go, units, B, H, ek, ev = geom
    cutoff = math.pi if units is None else units * math.pi / (ish[0] - 1)
    nb = A.get_neighbourhood(ish, osh, gi, go, cutoff)
    omega = 2.0 * np.pi * _grid_np(ish[0], gi)[1] / ish[1]
    g = torch.Generator().manual_seed(seed)
    q = 2.0 * torch.randn(B, osh[0] * osh[1], H * ek, generator=g, dtype=torch.float64)
    k = 2.0 * torch.randn(B, ish[0] * ish[1], H * ek, generator=g, dtype=torch.float64)
    v = torch.randn(B, ish[0] * ish[1], H * ev, generator=g, dtype=torch.float64)
    dy = torch.randn(B, osh[0] * osh[1], H * ev, generator=g, dtype=torch.float64)
    return nb, omega, q, k, v, dy, ish[1], osh[1], H, 1.0 / math.sqrt(ek)


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-300)).item()


@pytest.mark.parametrize("geom", GEOMETRIES, ids=lambda g: f"{g[0][0]}x{g[0][1]}-{g[1][0]}x{g[1][1]}-{g[4]}")
def test_references_are_the_oracle_on_fp64_operands(geom):
    nb, omega, q, k, v, dy, nlon_in, nlon_out, H, scale = _case(geom)
    qr, kr, vr = (x.clone().requires_grad_(True) for x in (q, k, v))
    y, lse = AO.attention(qr, kr, vr, nb.row_ptr, nb.col, omega, nlon_in, nlon_out, H, scale)
    y.backward(dy)
    (yx, my), (lx, ml) = AR.forward(scale * q, k, v, nb.row_ptr, nb.col, omega, nlon_in, nlon_out, H)
    assert _rel(yx, y.detach()) < 1e-12 and _rel(lx, lse.detach()) < 1e-12
    bw = AR.backward(scale * q, k, v, y.detach(), lse.detach(), dy, nb.row_ptr, nb.col, omega, nlon_in, nlon_out, H, scale)
    B, ev = q.shape[0], v.shape[2] // H
    D = (dy * y.detach()).view(B, -1, H, ev).sum(-1).transpose(1, 2)
    for what, want in (("D", D), ("dq", qr.grad), ("dk", kr.grad), ("dv", vr.grad)):
        assert bw[what][0].shape == want.shape, what
        if what in ("dq", "dk") and geom[4] == 0.05:
            # single-point neighbourhoods: the exact dq and dk are zero, both sides are fp64 cancellation
            assert bw[what][0].abs().max() < 1e-12 * (q.abs().max() * v.abs().max() * dy.abs().max()).item(), what
            continue
        assert _rel(bw[what][0], want) < 1e-12, (what, _rel(bw[what][0], want))


@pytest.mark.parametrize("geom", GEOMETRIES, ids=lambda g: f"{g[0][0]}x{g[0][1]}-{g[1][0]}x{g[1][1]}-{g[4]}")
def test_bounds_are_well_formed(geom):
    """every magnitude term is finite and non-negative, and the bound is positive wherever the reference is not zero"""
    nb, omega, q, k, v, dy, nlon_in, nlon_out, H, scale = _case(geom, seed=1)
    (y, my), (lse, ml) = AR.forward(scale * q, k, v, nb.row_ptr, nb.col, omega, nlon_in, nlon_out, H)
    bw = AR.backward(scale * q, k, v, y, lse, dy, nb.row_ptr, nb.col, omega, nlon_in, nlon_out, H, scale)
    for what, (ref, mag) in [("y", (y, my)), ("lse", (lse, ml))] + list(bw.items()):
        assert ref.shape == mag.shape, what
        assert torch.isfinite(mag).all() and (mag >= 0).all(), what
        assert (mag[ref != 0] > 0).all(), what
        # the bound covers the rounding of the stored value itself: mag >= |ref|
        assert (mag >= ref.abs() * (1 - 1e-12)).all(), what


def test_need_measures_the_bound():
    ref = torch.tensor([1.0, -2.0, 0.0], dtype=torch.float64)
    mag = torch.tensor([4.0, 4.0, 0.0], dtype=torch.float64)
    got = ref + torch.tensor([2.0 ** -24, -2.0 ** -23, 0.0], dtype=torch.float64)
    assert AR.need(got, ref, mag) == pytest.approx(0.5)
    assert AR.need(torch.tensor([float("nan"), 0.0, 0.0]), ref, mag) == float("inf")
    assert AR.need(torch.tensor([1.0, -2.0, 1e-30]), ref, mag) > 1e200

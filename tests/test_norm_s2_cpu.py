"""CPU tests of the quadrature-weighted instance norm (makani_b200.norm.GeometricInstanceNormS2, makani_b200.quadrature's grid rules):

* the latitude weights of every rule, crop and polar-rank slice against the oracle's restatement of makani's GridQuadrature (full H x W tensors);
* the closed-form backward (dx, dgamma, dbeta) against fp64 autograd of the formula, with and without GELU, on full crops (D = S) and partial crops
  and the serial normaliser (D = 1 != S), and the module's torch-operator stages run through the same autograd Function in fp64;
* the constructor contract of makani's class: signature, TypeError on an unknown keyword (FCN3's `pole_mask`), NotImplementedError on a grid without
  a rule, parameter names, state-dict keys, the non-persistent weight buffer, the `is_shared_mp` tags of the distributed class;
* the CPU module path against the oracle, float32 and bfloat16 inputs.
The kernels are covered by tests/test_gpu_norm_s2.py."""
import inspect

import numpy as np
import pytest
import torch

from makani_b200 import norm as N
from makani_b200.quadrature import crop_quadrature_np
from oracle import makani_norm_oracle as O

GRIDS = ["equiangular", "legendre-gauss", "clenshaw-curtiss", "weatherbench2", "euclidean"]
# img_shape, crop_shape, crop_offset
CROPS = [((17, 32), (17, 32), (0, 0)), ((181, 360), (181, 360), (0, 0)), ((180, 360), (120, 200), (30, 100)), ((49, 97), (48, 96), (1, 0))]


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("crop", CROPS, ids=lambda c: f"{c[0][0]}x{c[0][1]}-crop{c[1][0]}x{c[1][1]}")
def test_weights_match_grid_quadrature(grid, crop):
    img, cs, co = crop
    for h in (1, 2, 3, 4):
        hs = O.split_shapes(cs[0], h)
        for ih in range(h):
            ref = O.grid_quadrature(grid, img, cs, co, h, ih, 2, 1)
            q = crop_quadrature_np(grid, img, cs, co, hs if h > 1 else None, ih)
            assert q.shape == (ref.shape[0],)
            got = np.tile(q[:, None], (1, ref.shape[1]))
            np.testing.assert_allclose(got, ref.numpy(), rtol=1e-12, atol=1e-18)
    assert abs(crop_quadrature_np(grid, img).sum() * img[1] - 1.0) < 1e-12


def test_unknown_grid_raises():
    with pytest.raises(NotImplementedError):
        N.GeometricInstanceNormS2((8, 16), (8, 16), (0, 0), "healpix", 4)


# img_shape, crop_shape, crop_offset, grid
FORMULA_CASES = [((9, 16), (9, 16), (0, 0), "equiangular"), ((8, 16), (8, 16), (0, 0), "legendre-gauss"), ((12, 20), (7, 11), (2, 4), "weatherbench2")]


@pytest.mark.parametrize("case", FORMULA_CASES, ids=lambda c: f"{c[3]}-{c[1][0]}x{c[1][1]}")
@pytest.mark.parametrize("gelu", [False, True])
@pytest.mark.parametrize("normaliser", ["serial", "distributed"])
def test_backward_formula_matches_autograd(case, gelu, normaliser):
    img, cs, co, grid = case
    q = O.grid_quadrature(grid, img, cs, co)
    D = 1.0 if normaliser == "serial" else float(q.sum())
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(2, 3, *cs, dtype=torch.float64, generator=g) + 0.3).requires_grad_(True)
    w = (1.0 + 0.2 * torch.randn(3, dtype=torch.float64, generator=g)).requires_grad_(True)
    b = (0.1 * torch.randn(3, dtype=torch.float64, generator=g)).requires_grad_(True)
    dy = torch.randn(2, 3, *cs, dtype=torch.float64, generator=g)
    y = O.forward(x, q, 1e-5, w, b, gelu, D=D)
    y.backward(dy)
    dx, dw, db = O.backward(x.detach(), dy, q, 1e-5, w.detach(), b.detach(), gelu, D=D)
    if normaliser == "serial" and cs != img:
        assert abs(D - float(q.sum())) > 0.1      # a partial crop with D = 1 != S: the correction term is live
    for a, ref in ((dx, x.grad), (dw, w.grad), (db, b.grad)):
        assert torch.allclose(a, ref, rtol=1e-12, atol=1e-12), (a - ref).abs().max()

    # the autograd Function on the oracle's fp64 stand-in stages (forward and backward), and the forward of the module's own torch-operator stages
    # (fp32 normalisation, at 1e-5; their backward: test_torch_stages_backward_match_autograd_partial_crop)
    xs = x.detach().clone().requires_grad_(True)
    ws_, bs = w.detach().float().requires_grad_(True), b.detach().float().requires_grad_(True)
    y2 = N._GeometricNormFn.apply(xs, ws_, bs, q[:, 0].float(), D, 1e-5, gelu, O.OracleStages(), N._gather_none)
    y2.backward(dy)
    assert torch.allclose(xs.grad, x.grad, rtol=1e-6, atol=1e-6 * x.grad.abs().max().item())
    y3 = O.forward(x.detach(), q[:, :1].float().double().expand_as(q), 1e-5, ws_.detach().double(), bs.detach().double(), gelu, D=D)
    assert torch.allclose(y2, y3, rtol=1e-12, atol=1e-12)
    y4 = N._GeometricNormFn.apply(x.detach().clone(), ws_.detach(), bs.detach(), q[:, 0].float(), D, 1e-5, gelu, N.TorchGeometricNormStages(),
                                  N._gather_none)
    assert torch.allclose(y4.double(), y3, rtol=1e-5, atol=1e-5)


def test_torch_stages_backward_match_autograd_partial_crop():
    img, cs, co, grid = FORMULA_CASES[2]
    q = O.grid_quadrature(grid, img, cs, co).float().double()
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 3, *cs, dtype=torch.float64, generator=g).requires_grad_(True)
    w = torch.randn(3, generator=g).requires_grad_(True)
    b = torch.randn(3, generator=g).requires_grad_(True)
    dy = torch.randn(2, 3, *cs, dtype=torch.float64, generator=g)
    for gelu in (False, True):
        for t in (x, w, b):
            t.grad = None
        N._GeometricNormFn.apply(x, w, b, q[:, 0].float(), 1.0, 1e-5, gelu, N.TorchGeometricNormStages(), N._gather_none).backward(dy)
        xr, wr, br = (t.detach().double().requires_grad_(True) for t in (x, w, b))
        O.forward(xr, q, 1e-5, wr, br, gelu).backward(dy)
        for a, ref in ((x.grad, xr.grad), (w.grad, wr.grad), (b.grad, br.grad)):
            assert torch.allclose(a.double(), ref, rtol=1e-5, atol=1e-5 * ref.abs().max().item()), (a.double() - ref).abs().max()


def test_constructor_contract():
    sig = inspect.signature(N.GeometricInstanceNormS2.__init__)
    assert [(p.name, p.default) for p in list(sig.parameters.values())[1:]] == [
        ("img_shape", inspect.Parameter.empty), ("crop_shape", inspect.Parameter.empty), ("crop_offset", inspect.Parameter.empty),
        ("grid_type", inspect.Parameter.empty), ("num_features", inspect.Parameter.empty), ("eps", 1e-05), ("affine", False)]
    with pytest.raises(TypeError):
        N.GeometricInstanceNormS2((9, 16), (9, 16), (0, 0), "equiangular", 4, eps=1e-6, affine=True, pole_mask=0)
    m = N.GeometricInstanceNormS2((9, 16), (9, 16), (0, 0), "equiangular", 4, eps=1e-6, affine=True)
    assert [n for n, _ in m.named_parameters()] == ["weight", "bias"]
    assert list(m.state_dict().keys()) == ["weight", "bias"]
    assert torch.equal(m.weight, torch.ones(4)) and torch.equal(m.bias, torch.zeros(4))
    assert m.quad_weight.shape == (9,) and "quad_weight" in dict(m.named_buffers())
    assert list(N.GeometricInstanceNormS2((9, 16), (9, 16), (0, 0), "equiangular", 4).state_dict().keys()) == []

    import makani_b200.distributed as mbd
    d = mbd.DistributedGeometricInstanceNormS2((9, 16), (9, 16), (0, 0), "equiangular", 4, affine=True)
    assert list(d.state_dict().keys()) == ["weight", "bias"]
    assert d.weight.is_shared_mp == ["spatial"] and d.bias.is_shared_mp == ["spatial"]
    assert not hasattr(m.weight, "is_shared_mp")
    with pytest.raises(TypeError):
        mbd.DistributedGeometricInstanceNormS2((9, 16), (9, 16), (0, 0), "equiangular", 4, pole_mask=0)


MODULE_CASES = [((17, 32), (17, 32), (0, 0), "equiangular", True), ((16, 32), (16, 32), (0, 0), "legendre-gauss", False),
                ((24, 40), (12, 30), (6, 5), "clenshaw-curtiss", True), ((49, 97), (49, 97), (0, 0), "weatherbench2", True)]


@pytest.mark.parametrize("case", MODULE_CASES, ids=lambda c: f"{c[3]}-{c[1][0]}x{c[1][1]}")
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_cpu_module_matches_oracle(case, dtype):
    img, cs, co, grid, affine = case
    m = N.GeometricInstanceNormS2(img, cs, co, grid, 5, eps=1e-6, affine=affine)
    g = torch.Generator().manual_seed(11)
    if affine:
        with torch.no_grad():
            m.weight.copy_(1.0 + 0.3 * torch.randn(5, generator=g))
            m.bias.copy_(0.2 * torch.randn(5, generator=g))
    x = (3.0 + torch.randn(2, 5, *cs, generator=g)).to(dtype)
    dy = torch.randn(2, 5, *cs, generator=g)
    q = O.grid_quadrature(grid, img, cs, co)
    for gelu in (False, True):
        xi = x.clone().requires_grad_(True)
        m.zero_grad()
        y = m(xi, gelu=gelu)
        assert y.dtype == dtype and y.shape == x.shape
        y.backward(dy.to(dtype))
        xr = x.double().requires_grad_(True)
        pr = [p.detach().double().requires_grad_(True) for p in m.parameters()]
        yr = O.serial(xr, q, 1e-6, *(pr if affine else (None, None)), gelu=gelu)
        yr.backward(dy.to(dtype).double())
        tol = 1e-5 if dtype == torch.float32 else 1e-2
        rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
        assert rel(y.detach(), yr.detach()) < tol
        assert rel(xi.grad, xr.grad) < (tol if dtype == torch.float32 else 2e-2)
        for p, r in zip(m.parameters(), pr):
            assert rel(p.grad, r.grad) < tol


def test_wrong_shape_is_refused():
    m = N.GeometricInstanceNormS2((17, 32), (16, 30), (0, 0), "equiangular", 4)
    with pytest.raises(ValueError):
        m(torch.randn(1, 4, 17, 32))


def test_sfno_instance_norm_s2_handles():
    """makani's per-block handles: first block (inp, mid) at (h, w), middle (mid, mid), last (out, out) at out_shape; model grid, eps 1e-6, affine;
    the network runs forward and backward on the oracle backend, and `instance_norm` still builds torch-compatible InstanceNorm2d modules"""
    from makani_b200.sfno import SphericalFourierNeuralOperatorNet
    from oracle.sfno_backend import OracleBackend

    kw = dict(inp_shape=(33, 64), out_shape=(17, 32), scale_factor=2, inp_chans=3, out_chans=2, embed_dim=8, num_layers=3, model_grid_type="equiangular",
              sht_grid_type="legendre-gauss", backend=OracleBackend())
    torch.manual_seed(0)
    net = SphericalFourierNeuralOperatorNet(normalization_layer="instance_norm_s2", **kw)
    shapes = [(b.norm0.img_shape, b.norm1.img_shape) for b in net.blocks]
    assert shapes == [((16, 32), (16, 32)), ((16, 32), (16, 32)), ((17, 32), (17, 32))]
    for b in net.blocks:
        for n in (b.norm0, b.norm1):
            assert type(n) is N.GeometricInstanceNormS2 and n.grid_type == "equiangular" and n.eps == 1e-6 and n.affine
            assert n.crop_shape == n.img_shape and n.crop_offset == (0, 0)
    x = torch.randn(2, 3, 33, 64)
    y = net(x)
    assert y.shape == (2, 2, 17, 32) and torch.isfinite(y).all()
    y.square().sum().backward()
    assert all(p.grad is not None for n, p in net.named_parameters() if "norm" in n)
    torch.manual_seed(0)
    plain = SphericalFourierNeuralOperatorNet(normalization_layer="instance_norm", **kw)
    assert all(type(b.norm0) is N.InstanceNorm2d and type(b.norm1) is N.InstanceNorm2d for b in plain.blocks)
    keys = set(plain.state_dict().keys())
    assert keys == set(net.state_dict().keys())

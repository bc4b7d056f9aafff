"""makani_b200/sfno.py with `normalization_layer="instance_norm_s2"` (makani_b200.norm.GeometricInstanceNormS2 in every block, makani's per-block
handles) against golden vectors produced by makani's OWN network class with makani's own GeometricInstanceNormS2 and GridQuadrature
(tests/golden/make_sfno_s2norm_golden.py): the network on the oracle backend loads the reference state dict strictly and reproduces its output,
input gradient and the gradients of the norm parameters, on an equiangular and a Legendre-Gauss model grid.  Also: the weights stay fp32 when the
module is cast.  The CUDA path against the same vectors: tests/test_gpu_norm_s2.py."""
import os
import sys

import numpy as np
import pytest
import torch

from makani_b200.norm import GeometricInstanceNormS2
from makani_b200.sfno import SphericalFourierNeuralOperatorNet
from oracle.sfno_backend import OracleBackend
from test_sfno_cpu import golden_state_dict

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_sfno_s2norm_golden import GRAD_KEYS, SFNO_S2NORM_GOLDEN_CASES  # noqa: E402

GOLD_S2NORM = os.path.join(os.path.dirname(__file__), "golden", "sfno_s2norm_golden.npz")


@pytest.mark.parametrize("name", sorted(SFNO_S2NORM_GOLDEN_CASES))
def test_network_on_oracle_backend_matches_reference_network(name):
    g = np.load(GOLD_S2NORM)
    torch.manual_seed(0)
    net = SphericalFourierNeuralOperatorNet(**SFNO_S2NORM_GOLDEN_CASES[name], backend=OracleBackend())
    assert all(type(b.norm0) is GeometricInstanceNormS2 for b in net.blocks)
    sd = golden_state_dict(g, name)
    assert sorted(net.state_dict().keys()) == sorted(sd.keys())
    net.load_state_dict(sd, strict=True)
    x = torch.from_numpy(g[f"{name}/x"]).requires_grad_(True)
    y = net(x)
    yref = torch.from_numpy(g[f"{name}/y"])
    assert torch.allclose(y, yref, rtol=1e-4, atol=1e-5), (y - yref).abs().max()
    (y * torch.from_numpy(g[f"{name}/g"])).sum().backward()
    assert torch.allclose(x.grad, torch.from_numpy(g[f"{name}/dx"]), rtol=1e-3, atol=1e-4)
    params = dict(net.named_parameters())
    for k in GRAD_KEYS:
        ref = torch.from_numpy(g[f"{name}/grad/{k}"])
        got = params[k].grad
        got = torch.view_as_real(got) if got.is_complex() else got
        assert torch.allclose(got, ref, rtol=1e-3, atol=1e-4 * ref.abs().max().item() + 1e-6), k


def test_weights_stay_fp32_when_the_module_is_cast():
    m = GeometricInstanceNormS2((33, 64), (33, 64), (0, 0), "equiangular", 4, affine=True)
    q = m.quad_weight.clone()
    m.to(torch.bfloat16)
    assert m.weight.dtype == torch.bfloat16 and m.quad_weight.dtype == torch.float32 and torch.equal(m.quad_weight, q)
    m.double()
    assert m.quad_weight.dtype == torch.float32 and torch.equal(m.quad_weight, q)
    assert m(torch.randn(2, 4, 33, 64, dtype=torch.bfloat16)).dtype == torch.bfloat16

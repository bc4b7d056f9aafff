"""CPU tests of the channel layer norm (makani_b200.norm.DistributedLayerNorm, makani's DistributedLayerNorm):

* the constructor contract of makani's class: signature, the `.norm` nn.LayerNorm submodule, parameter names and shapes, state-dict keys, the
  `is_shared_mp` / `sharded_dims_mp` tags, without affine and without bias, and the errors of a bad argument or input;
* CPU tensors take makani's formula (transpose -> nn.LayerNorm -> transpose), GELU applied after it, output dtypes with and without autocast;
* the SFNO network's `normalization_layer="layer_norm"` against golden vectors of makani's own network (tests/golden/sfno_layernorm_golden.npz) on
  the oracle backend, and the norm0 -> GELU fusion it takes;
* `compat.patch_makani_layer_norm()` repoints makani's names;
* the layer-norm kernels compile for sm_90a without register spills.
The kernels are covered by tests/test_gpu_layer_norm.py."""
import inspect
import os
import re
import shutil
import subprocess
import sys
import tempfile
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from makani_b200 import norm as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_sfno_layernorm_golden import GRAD_KEYS, SFNO_LAYERNORM_GOLDEN_CASES  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "sfno_layernorm_golden.npz")


def makani_formula(norm, x):
    """makani's DistributedLayerNorm.forward (makani/mpu/layer_norm.py:284-290)"""
    return torch.transpose(norm(torch.transpose(x, 1, 3)), 1, 3).contiguous()


def test_constructor_contract():
    sig = inspect.signature(N.DistributedLayerNorm.__init__)
    assert [(p.name, p.default) for p in list(sig.parameters.values())[1:]] == [
        ("normalized_shape", inspect.Parameter.empty), ("eps", 1e-05), ("elementwise_affine", True), ("bias", True), ("device", None), ("dtype", None)]
    m = N.DistributedLayerNorm(12, eps=1e-6)
    assert type(m.norm) is nn.LayerNorm and m.norm.normalized_shape == (12,) and m.norm.eps == 1e-6
    assert [(n, tuple(p.shape)) for n, p in m.named_parameters()] == [("norm.weight", (12,)), ("norm.bias", (12,))]
    assert list(m.state_dict().keys()) == ["norm.weight", "norm.bias"]
    assert torch.equal(m.norm.weight, torch.ones(12)) and torch.equal(m.norm.bias, torch.zeros(12))
    for p in (m.norm.weight, m.norm.bias):
        assert p.is_shared_mp == ["model"] and p.sharded_dims_mp == [None]

    nb = N.DistributedLayerNorm((7,), bias=False)
    assert list(nb.state_dict().keys()) == ["norm.weight"] and nb.norm.bias is None and nb.norm.weight.is_shared_mp == ["model"]
    na = N.DistributedLayerNorm(7, elementwise_affine=False)
    assert list(na.state_dict().keys()) == [] and na.norm.weight is None and na.norm.bias is None
    assert N.DistributedLayerNorm(5, dtype=torch.float64).norm.weight.dtype == torch.float64

    # a state dict of makani's layout loads strictly, and a wrong one is refused
    sd = {"norm.weight": torch.randn(12), "norm.bias": torch.randn(12)}
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.norm.weight, sd["norm.weight"])
    with pytest.raises(RuntimeError):
        m.load_state_dict({"weight": torch.randn(12), "bias": torch.randn(12)}, strict=True)
    with pytest.raises(TypeError):
        N.DistributedLayerNorm(12, affine=True)
    with pytest.raises(RuntimeError):
        m(torch.randn(2, 11, 4, 5))        # channels != normalized_shape, as nn.LayerNorm refuses it


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("affine,bias", [(True, True), (True, False), (False, False)])
def test_cpu_takes_makanis_formula(dtype, affine, bias):
    torch.manual_seed(0)
    m = N.DistributedLayerNorm(6, eps=1e-6, elementwise_affine=affine, bias=bias)
    if affine:
        with torch.no_grad():
            for p in m.parameters():
                p.add_(0.3 * torch.randn_like(p))
    x = (1e3 + torch.randn(2, 6, 5, 7)).to(dtype)
    for gelu in (False, True):
        xa, xb = x.clone().requires_grad_(True), x.clone().requires_grad_(True)
        y = m(xa, gelu=gelu)
        yr = makani_formula(m.norm, xb)
        yr = F.gelu(yr) if gelu else yr
        assert y.dtype == yr.dtype == dtype and y.is_contiguous()
        assert torch.equal(y, yr)
        dy = torch.randn_like(y)
        y.backward(dy)
        yr.backward(dy)
        assert torch.equal(xa.grad, xb.grad)


def test_output_dtype_under_autocast():
    """CPU autocast keeps a bf16 layer_norm in bf16 (CUDA autocast returns fp32: tests/test_gpu_layer_norm.py); the module follows makani either way"""
    m = N.DistributedLayerNorm(4)
    for dtype in (torch.float32, torch.bfloat16):
        x = torch.randn(1, 4, 3, 5, dtype=dtype)
        assert m(x).dtype == makani_formula(m.norm, x).dtype == dtype
        with torch.autocast("cpu", dtype=torch.bfloat16):
            assert m(x).dtype == makani_formula(m.norm, x).dtype
        assert N._layer_norm_out_dtype(x) == dtype


def golden_state_dict(g, name):
    sd = {}
    for k in g.files:
        if k.startswith(f"{name}/sd/"):
            v = torch.from_numpy(g[k])
            key = k[len(f"{name}/sd/"):]
            sd[key] = torch.view_as_complex(v.contiguous()) if (key.endswith("filter.filter.weight") and v.shape[-1] == 2 and v.dtype == torch.float32) else v
    return sd


@pytest.mark.parametrize("name", sorted(SFNO_LAYERNORM_GOLDEN_CASES))
def test_network_on_oracle_backend_matches_reference_network(name):
    from makani_b200.sfno import SphericalFourierNeuralOperatorNet
    from oracle.sfno_backend import OracleBackend

    g = np.load(GOLD)
    torch.manual_seed(0)
    cfg = SFNO_LAYERNORM_GOLDEN_CASES[name]
    net = SphericalFourierNeuralOperatorNet(**cfg, backend=OracleBackend())
    for b in net.blocks:
        for n in (b.norm0, b.norm1):
            assert type(n) is N.DistributedLayerNorm and n.norm.normalized_shape == (cfg["embed_dim"],) and n.norm.eps == 1e-6
            assert n.norm.elementwise_affine and n.norm.bias is not None
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


def test_sfno_fuses_norm0_and_gelu(monkeypatch):
    """with inner_skip "none" and exact GELU, the block calls norm0(x, gelu=True) for the layer norm as for the instance norms"""
    from makani_b200.sfno import SphericalFourierNeuralOperatorNet
    from oracle.sfno_backend import OracleBackend

    cfg = dict(SFNO_LAYERNORM_GOLDEN_CASES["ln_eq"])
    net = SphericalFourierNeuralOperatorNet(**cfg, backend=OracleBackend())
    seen = []
    orig = N.DistributedLayerNorm.forward

    def spy(self, x, gelu=False):
        seen.append((self is net.blocks[0].norm0, gelu))
        return orig(self, x, gelu=gelu)

    monkeypatch.setattr(N.DistributedLayerNorm, "forward", spy)
    net(torch.randn(1, cfg["inp_chans"], *cfg["inp_shape"]))
    assert (True, True) in seen and (False, False) in seen
    assert all(g for is0, g in seen if is0)


def test_compat_patch_points_makani_names_at_the_class(monkeypatch):
    from makani_b200 import compat

    class Theirs(nn.Module):
        pass

    mods = {}
    for name in ("makani", "makani.mpu", "makani.mpu.layer_norm", "makani.models", "makani.models.networks", "makani.models.networks.sfnonet",
                 "makani.models.networks.snonet"):
        mods[name] = types.ModuleType(name)
        monkeypatch.setitem(sys.modules, name, mods[name])
    for name in ("makani.mpu.layer_norm", "makani.models.networks.sfnonet", "makani.models.networks.snonet"):
        mods[name].DistributedLayerNorm = Theirs
    compat.patch_makani_layer_norm()
    for name in ("makani.mpu.layer_norm", "makani.models.networks.sfnonet", "makani.models.networks.snonet"):
        assert mods[name].DistributedLayerNorm is N.DistributedLayerNorm, name


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc is not available")
def test_layer_norm_kernels_do_not_spill():
    csrc = os.path.join(ROOT, "makani_b200", "csrc")
    log = os.path.join(ROOT, "makani_b200", "build", "norm.o.log")
    sources = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh"))]
    if os.path.exists(log) and os.path.getmtime(log) >= max(os.path.getmtime(s) for s in sources):
        report = open(log).read()
    else:
        from makani_b200 import build as _build

        nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
        with tempfile.TemporaryDirectory() as tmp:
            r = subprocess.run([nvcc] + _build.FLAGS + ["-c", os.path.join(csrc, "norm.cu"), "-o", os.path.join(tmp, "norm.o")],
                               capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        report = r.stdout + r.stderr
    pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?Function properties for \1\n\s+(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    kernels = {m.group(1): (int(m.group(3)), int(m.group(4))) for m in pat.finditer(report) if "ln_" in m.group(1)}
    # forward and backward for (float, float), (bf16, bf16), (bf16, float), staged and not; the parameter-gradient finalize
    assert sum("ln_forward_kernel" in k for k in kernels) == 6 and sum("ln_backward_kernel" in k for k in kernels) == 6, kernels
    assert sum("ln_param_grad_kernel" in k for k in kernels) == 1, kernels
    spilling = {k: v for k, v in kernels.items() if v[0] or v[1]}
    assert not spilling, spilling

"""The channel layer norm on the GPU (csrc/norm.cu through makani_b200.norm.DistributedLayerNorm):

* y, dx, dgamma and dbeta against transpose + F.layer_norm (+ F.gelu) in fp64 autograd of the exact operands, per element, over C in {1, 3, 45, 384,
  1024} (C = 1024 takes the unstaged kernels: its tile does not fit in shared memory), odd H x W and 721 x 1440 at C = 384; float32, bfloat16, and
  bfloat16 under autocast (fp32 out); GELU on and off, with and without affine and bias; inputs offset by 1e3 from zero.  Bound per element:
  (1e-5 + 16 u |mu| r) times the larger of 1, |ref| and the size of the terms that make it up, u = 2^-24 (the offset enters once, through the fp32 mu;
  a variance that cancelled would be off by far more), plus one bf16 ulp of a bf16 output.  dgamma / dbeta: the same factor times the sum of the
  absolute values of their terms;
* the output dtype equals makani's layer's with and without autocast;
* two runs are bit-identical (y, dx, dgamma, dbeta);
* the forward and backward launch only the new kernels;
* makani's own SFNO with layer_norm (tests/golden/sfno_layernorm_golden.npz) on the CUDA path, fp32 and TF32."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from makani_b200 import norm as N
from test_gpu_engine import DEV, launched_kernels

pytestmark = pytest.mark.gpu

TOL, U = 1e-5, 2.0 ** -24
EPS = 1e-6
# B, C, H, W
SHAPES = [(2, 1, 7, 13), (2, 3, 33, 65), (2, 45, 17, 31), (1, 384, 24, 48), (2, 1024, 9, 19)]
# id, dtype of x, autocast (y / dy fp32)
DTYPES = [("f32", torch.float32, False), ("bf16", torch.bfloat16, False), ("bf16-autocast", torch.bfloat16, True)]
# id, affine, bias, gelu
MODES = [("gelu", True, True, True), ("plain", True, True, False), ("no-affine", False, False, True), ("no-bias", True, False, False)]


def _bf16_ulp(ref):
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _module(C, affine, bias, gen):
    m = N.DistributedLayerNorm(C, eps=EPS, elementwise_affine=affine, bias=bias).to(DEV)
    with torch.no_grad():
        if affine:
            m.norm.weight.copy_(1.0 + 0.3 * torch.randn(C, device=DEV, generator=gen))
        if bias:
            m.norm.bias.copy_(0.2 * torch.randn(C, device=DEV, generator=gen))
    return m


def _run(m, x, dy, gelu, autocast):
    xi = x.clone().requires_grad_(True)
    m.zero_grad()
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = m(xi, gelu=gelu)
    y.backward(dy)
    return y.detach(), xi.grad, m.norm.weight.grad if m.norm.weight is not None else None, m.norm.bias.grad if m.norm.bias is not None else None


def _check(name, got, ref, factor, scale, bf16_out):
    got, ref = got.double(), ref.double()
    bound = factor * torch.maximum(ref.abs().clamp_min(1.0), scale)
    if bf16_out:
        bound = bound + _bf16_ulp(ref)
    worst = ((got - ref).abs() / bound).max().item()
    print(f"{name}: worst err / bound {worst:.3f}")
    assert torch.isfinite(got).all() and worst <= 1.0, (name, worst)


def _against_fp64(B, C, H, W, dtype, autocast, affine, bias, gelu, offset):
    gen = torch.Generator(device=DEV).manual_seed(C + H + W)
    m = _module(C, affine, bias, gen)
    x = (offset + torch.randn(B, C, H, W, device=DEV, generator=gen, dtype=torch.float64)).to(dtype)
    out_dtype = torch.float32 if autocast else dtype
    dy = torch.randn(B, C, H, W, device=DEV, generator=gen).to(out_dtype)
    y, dx, dw, db = _run(m, x, dy, gelu, autocast)
    assert y.dtype == out_dtype and dx.dtype == dtype and y.shape == x.shape

    # fp64 reference: makani's formula on the exact operands
    x64 = x.double().requires_grad_(True)
    w64 = m.norm.weight.detach().double().requires_grad_(True) if affine else None
    b64 = m.norm.bias.detach().double().requires_grad_(True) if bias else None
    z = F.layer_norm(x64.transpose(1, 3), (C,), w64, b64, EPS).transpose(1, 3)
    yr = F.gelu(z) if gelu else z
    yr.backward(dy.double())
    with torch.no_grad():
        mu = x64.mean(dim=1, keepdim=True)
        r = 1.0 / torch.sqrt(((x64 - mu) ** 2).mean(dim=1, keepdim=True) + EPS)
        xh = (x64 - mu) * r
        gam = w64.view(1, C, 1, 1) if affine else torch.ones(1, C, 1, 1, dtype=torch.float64, device=DEV)
        bet = b64.view(1, C, 1, 1) if bias else 0.0
        zz = xh * gam + bet
        g = dy.double() * (0.5 * (1.0 + torch.erf(zz / 2 ** 0.5)) + zz * torch.exp(-0.5 * zz * zz) / (2 * torch.pi) ** 0.5) if gelu else dy.double()
        factor = TOL + 16 * U * (mu.abs() * r)                         # per point
        m1, m2 = (gam * g).mean(dim=1, keepdim=True), (gam * g * xh).mean(dim=1, keepdim=True)
        _check("y", y, yr.detach(), factor, (gam * xh).abs() + abs(bet) if bias else (gam * xh).abs(), out_dtype == torch.bfloat16)
        _check("dx", dx, x64.grad, factor, r * ((gam * g).abs() + m1.abs() + xh.abs() * m2.abs()), dtype == torch.bfloat16)
        fmax = factor.max()
        if affine:
            _check("dgamma", dw, w64.grad, fmax, (g * xh).abs().sum(dim=(0, 2, 3)) + g.abs().sum(dim=(0, 2, 3)), False)
        if bias:
            _check("dbeta", db, b64.grad, fmax, g.abs().sum(dim=(0, 2, 3)), False)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dt", DTYPES, ids=[d[0] for d in DTYPES])
@pytest.mark.parametrize("mode", MODES, ids=[m[0] for m in MODES])
@pytest.mark.parametrize("offset", [0.0, 1e3], ids=["centred", "offset1e3"])
def test_against_fp64_layer_norm(shape, dt, mode, offset):
    _, dtype, autocast = dt
    _, affine, bias, gelu = mode
    _against_fp64(*shape, dtype, autocast, affine, bias, gelu, offset)


@pytest.mark.parametrize("dt", DTYPES, ids=[d[0] for d in DTYPES])
@pytest.mark.parametrize("mode,offset", [("gelu", 0.0), ("no-bias", 1e3)])
def test_against_fp64_layer_norm_721x1440(dt, mode, offset):
    _, dtype, autocast = dt
    _, affine, bias, gelu = next(m for m in MODES if m[0] == mode)
    _against_fp64(1, 384, 721, 1440, dtype, autocast, affine, bias, gelu, offset)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("autocast", [False, True])
def test_output_dtype_matches_makani(dtype, autocast):
    """makani's layer on CUDA refuses a bf16 input with its fp32 parameters outside autocast ("expected scalar type BFloat16"); the kernels take
    it and return bf16, as makani's formula does on the CPU"""
    m = N.DistributedLayerNorm(8).to(DEV)
    x = torch.randn(2, 8, 5, 6, device=DEV).to(dtype)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        y = m(x)
        yg = m(x, gelu=True)
        if dtype == torch.bfloat16 and not autocast:
            with pytest.raises(RuntimeError):
                torch.transpose(m.norm(torch.transpose(x, 1, 3)), 1, 3)
            yr = torch.transpose(m.norm.to(torch.bfloat16)(torch.transpose(x, 1, 3)), 1, 3).contiguous()
        else:
            yr = torch.transpose(m.norm(torch.transpose(x, 1, 3)), 1, 3).contiguous()
    assert y.dtype == yr.dtype == yg.dtype, (y.dtype, yr.dtype)
    assert y.is_contiguous()
    assert torch.allclose(y.double(), yr.double(), rtol=1e-2 if y.dtype == torch.bfloat16 else 1e-5, atol=1e-2 if y.dtype == torch.bfloat16 else 1e-5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_two_runs_are_bit_identical(dtype):
    gen = torch.Generator(device=DEV).manual_seed(1)
    m = _module(384, True, True, gen)
    x = (3.0 + torch.randn(1, 384, 240, 480, device=DEV, generator=gen)).to(dtype)
    dy = torch.randn(1, 384, 240, 480, device=DEV, generator=gen).to(dtype)
    a = _run(m, x, dy, True, False)
    b = _run(m, x, dy, True, False)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_launches_only_the_new_kernels():
    gen = torch.Generator(device=DEV).manual_seed(2)
    m = _module(64, True, True, gen)
    x = torch.randn(1, 64, 240, 480, device=DEV, requires_grad=True)
    dy = torch.randn_like(x)
    m(x, gelu=True).backward(dy)

    def run():
        x.grad = None
        m.zero_grad()
        m(x, gelu=True).backward(dy)

    want = ["ln_forward_kernel<float, float, true>", "ln_backward_kernel<float, float, true>", "ln_param_grad_kernel"]
    names = launched_kernels(run, done=lambda n: all(any(w in s for s in n) for w in want))
    assert all(any(w in s for s in names) for w in want), names
    assert all("ln_" in s for s in names), names
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    every = {e.name for e in prof.events()}
    assert not any("layer_norm" in s.lower() and "b200sht" not in s for s in every), every


@pytest.fixture
def torch_tf32():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("name", ["ln_eq", "ln_lg"])
@pytest.mark.parametrize("precision,rtol,grtol", [("fp32", 2e-4, 5e-4), ("tf32", 1e-2, 3e-2)])
def test_sfno_layer_norm_matches_reference_network(name, precision, rtol, grtol, torch_tf32):
    """makani's own SFNO with layer_norm (tests/golden/sfno_layernorm_golden.npz) on the CUDA path: fp32 at the tolerances of test_gpu_sfno.py; TF32
    looser, because a norm over 8 channels per point divides by the spread of 8 samples and so amplifies the TF32 rounding of the filter output far
    more than an instance norm over H x W points does (ln_eq: y rel. L2 4.0e-3 on an H100)"""
    from makani_b200.sfno import SphericalFourierNeuralOperatorNet
    from test_gpu_parity import close
    from test_sfno_cpu import golden_state_dict

    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_sfno_layernorm_golden import GRAD_KEYS, SFNO_LAYERNORM_GOLDEN_CASES

    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = (precision == "tf32")
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "sfno_layernorm_golden.npz"))
    net = SphericalFourierNeuralOperatorNet(**SFNO_LAYERNORM_GOLDEN_CASES[name], precision=precision)
    net.load_state_dict(golden_state_dict(g, name), strict=True)
    net = net.to(DEV)
    x = torch.from_numpy(g[f"{name}/x"]).to(DEV).requires_grad_(True)

    names = launched_kernels(lambda: net(x), done=lambda n: any("ln_forward_kernel" in s for s in n))
    assert any("ln_forward_kernel" in s for s in names), names      # the norms run on the new kernels
    y = net(x)
    close(y, torch.from_numpy(g[f"{name}/y"]), rtol, f"SFNO-LN[{name},{precision}] y")
    (y * torch.from_numpy(g[f"{name}/g"]).to(DEV)).sum().backward()
    close(x.grad, torch.from_numpy(g[f"{name}/dx"]), grtol, f"SFNO-LN[{name},{precision}] dx")
    params = dict(net.named_parameters())
    for k in GRAD_KEYS:
        ref = torch.from_numpy(g[f"{name}/grad/{k}"])
        got = params[k].grad
        got = torch.view_as_real(got) if got.is_complex() else got
        close(got, ref, grtol, f"SFNO-LN[{name},{precision}] d{k}")

"""Global attention on an H100: the kernels of csrc/attention_global.cu through the C ABI against fp64 evaluations of their exact fp32
operands, per element, at tile-boundary sizes; bit-identical reruns; AttentionS2 against the fp64 oracle (tests/attention_global_oracle.py)
for the forward and every input and parameter gradient; one sampled-row check at a 361 x 720 output grid."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import attention_global_oracle as GO  # noqa: E402
from makani_b200 import _lib  # noqa: E402
from makani_b200 import attention as A  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
# unit roundoff of the operands the tensor cores read: TF32 (10-bit mantissa, rounded to nearest) and the 3 x TF32 split
U = {_lib.PREC_TF32: 2.0 ** -11, _lib.PREC_FP32X3: 2.0 ** -24}
C_BOUND = 16.0


def _case(B, H, nq, nk, dqk, dv, masked, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, H, nq, dqk, device=DEV, generator=g)
    k = torch.randn(B, H, nk, dqk, device=DEV, generator=g)
    v = torch.randn(B, H, dv, nk, device=DEV, generator=g)
    do = torch.randn(B, H, nq, dv, device=DEV, generator=g)
    bias = torch.log(torch.rand(nk, device=DEV, generator=g) * 0.01 + 1e-4)
    if masked:
        bias[: min(40, nk - 1)] = -torch.inf   # the whole first key block and part of the second drop out
        bias[45::7] = -torch.inf
    return q, k, v, do, bias


def _reference(q, k, v, do, bias, scale):
    """fp64 o, lse, dq, dk, dv of the exact fp32 operands, and the sums of absolute terms that bound each element's error"""
    q, k, v, do, b = (t.double() for t in (q, k, v, do, bias))
    lg = scale * q @ k.transpose(-1, -2) + b
    lse = torch.logsumexp(lg, -1)
    p = torch.exp(lg - lse[..., None])
    o = p @ v.transpose(-1, -2)
    dp = do @ v
    D = (do * o).sum(-1)
    ds = p * (dp - D[..., None])
    dq, dk, dv = scale * ds @ k, scale * ds.transpose(-1, -2) @ q, do.transpose(-1, -2) @ p
    lab = 1.0 + scale * q.abs() @ k.abs().transpose(-1, -2)                       # 1 + |logit terms|
    ao = (p * lab) @ v.abs().transpose(-1, -2) + (p * lab).sum(-1, keepdim=True) * o.abs()
    alse = (p * lab).sum(-1) + lse.abs()
    adp = do.abs() @ v.abs()
    ads = p * (lab * (dp.abs() + D.abs()[..., None]) + adp + (do * o).abs().sum(-1)[..., None]) + ds.abs()
    adq, adk = scale * ads @ k.abs(), scale * ads.transpose(-1, -2) @ q.abs()
    adv = do.abs().transpose(-1, -2) @ (p * lab)
    return (o, lse, dq, dk, dv), (ao, alse, adq, adk, adv)


def _run(q, k, v, do, bias, scale, prec):
    o, lse = A.global_attention_forward(q, k, v, bias, scale, prec)
    dq, dk, dv = A.global_attention_backward(q, k, v, bias, o, lse, do, scale, prec)
    torch.cuda.synchronize()
    return o, lse, dq, dk, dv


SIZES = [(1, 2, 100, 77, 8, 8, True), (2, 1, 65, 33, 32, 32, False), (1, 3, 130, 97, 64, 24, True), (1, 1, 64, 161, 128, 128, True),
         (1, 2, 31, 200, 16, 104, False), (1, 1, 1, 5, 40, 8, False)]


@pytest.mark.parametrize("prec", [_lib.PREC_TF32, _lib.PREC_FP32X3], ids=["tf32", "fp32x3"])
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s[:6])) + ("m" if s[6] else ""))
def test_kernels_per_element_against_fp64_of_their_operands(size, prec):
    B, H, nq, nk, dqk, dv, masked = size
    q, k, v, do, bias = _case(B, H, nq, nk, dqk, dv, masked, seed=nq * 7 + nk)
    scale = 1.0 / np.sqrt(dqk)
    got = _run(q, k, v, do, bias, scale, prec)
    ref, terms = _reference(q, k, v, do, bias, scale)
    n = max(dqk, dv)
    tol = C_BOUND * (n * U[prec] + (max(nq, nk) + n) * 2.0 ** -24)
    worst = {}
    for name, g, r, t in zip(("o", "lse", "dq", "dk", "dv"), got, ref, terms):
        assert torch.isfinite(g).all(), name
        ratio = ((g.double() - r).abs() / (tol * t + 1e-300)).max().item()
        worst[name] = ratio
        assert ratio <= 1.0, (name, ratio)
    if masked:
        assert (got[3][:, :, bias.isinf()] == 0).all() and (got[4][..., bias.isinf()] == 0).all()
    print(f"\n{size} prec {prec}: worst error / bound", {k_: f"{v_:.3g}" for k_, v_ in worst.items()})


@pytest.mark.parametrize("prec", [_lib.PREC_TF32, _lib.PREC_FP32X3], ids=["tf32", "fp32x3"])
def test_two_runs_are_bit_identical(prec):
    q, k, v, do, bias = _case(2, 2, 700, 1100, 64, 64, True, seed=5)
    a = _run(q, k, v, do, bias, 0.125, prec)
    b = _run(q, k, v, do, bias, 0.125, prec)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _module_case(in_shape, out_shape, C, heads, ck, cv, grid_in, dtype, seed):
    torch.manual_seed(seed)
    m = A.AttentionS2(C, heads, in_shape, out_shape, grid_in=grid_in, k_channels=ck, out_channels=cv).to(DEV)
    with torch.no_grad():
        for n, p_ in m.named_parameters():
            if n.endswith("_bias"):
                p_.normal_(0.0, 0.2)
    query = torch.randn(2, C, *out_shape, device=DEV).to(dtype)
    kv = torch.randn(2, C, *in_shape, device=DEV).to(dtype)
    return m, query, kv


def _rel(a, b):
    return ((a.double() - b).norm() / b.norm()).item()


MODULE_CASES = [((9, 18), (9, 18), 16, 2, None, None, "equiangular"), ((12, 24), (7, 14), 24, 3, 48, 24, "legendre-gauss"),
                ((17, 32), (33, 64), 32, 1, 64, 128, "equiangular")]


@pytest.mark.parametrize("tf32", [False, True], ids=["fp32", "tf32"])
@pytest.mark.parametrize("case", MODULE_CASES, ids=lambda c: f"{c[0]}->{c[1]}")
def test_module_against_the_oracle(case, tf32):
    in_shape, out_shape, C, heads, ck, cv, grid_in = case
    m, query, kv = _module_case(in_shape, out_shape, C, heads, ck, cv, grid_in, torch.float32, seed=1)
    same = in_shape == out_shape
    key = value = None if same else kv
    x_in = [query] if same else [query, kv]
    for x in x_in:
        x.requires_grad_(True)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        y = m(query, key, value)
        gy = torch.randn_like(y)
        grads = torch.autograd.grad(y, x_in + list(m.parameters()), gy)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    params = {n: p_.detach().double().requires_grad_(True) for n, p_ in m.named_parameters()}
    xr = [x.detach().double().requires_grad_(True) for x in x_in]
    yr = GO.module_forward(params, xr[0], xr[0] if same else xr[1], xr[0] if same else xr[1], grid_in, heads, m.scale)
    gr = torch.autograd.grad(yr, xr + list(params.values()), gy.double())
    tol = 2e-3 if tf32 else 1e-5
    assert y.dtype == torch.float32 and _rel(y, yr) <= tol, _rel(y, yr)
    names = ["query"] + ([] if same else ["key/value"]) + list(params)
    ref = dict(zip(names, gr))
    for n, g, r in zip(names, grads, gr):
        if n == "k_bias":   # exactly zero: a per-query constant logit shift leaves the softmax unchanged
            assert (g.double().norm() / ref["k_weights"].norm()).item() <= tol
        else:
            assert _rel(g, r) <= tol, (n, _rel(g, r))


def test_module_bf16_inputs():
    m, query, kv = _module_case((10, 20), (5, 10), 16, 2, None, None, "legendre-gauss", torch.bfloat16, seed=2)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        y = m(query, kv, kv)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    params = {n: p_.detach().double() for n, p_ in m.named_parameters()}
    yr = GO.module_forward(params, query.double(), kv.double(), kv.double(), "legendre-gauss", 2, m.scale)
    assert y.dtype == torch.float32 and _rel(y, yr) <= 1e-5


def test_sampled_rows_at_361x720():
    in_shape, out_shape, C, heads = (181, 360), (361, 720), 64, 4
    torch.manual_seed(3)
    m = A.AttentionS2(C, heads, in_shape, out_shape).to(DEV)
    query = torch.randn(1, C, *out_shape, device=DEV)
    kv = torch.randn(1, C, *in_shape, device=DEV)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            y = m(query, kv, kv).view(1, C, -1)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    rows = torch.cat([torch.arange(0, 720), torch.randint(720, 361 * 720, (256,), generator=torch.Generator().manual_seed(0)),
                      torch.arange(360 * 720, 361 * 720)]).to(DEV)
    params = {n: p_.detach().double() for n, p_ in m.named_parameters()}
    yr = GO.module_forward(params, query.double(), kv.double(), kv.double(), "equiangular", heads, m.scale, rows=rows)
    assert _rel(y[:, :, rows], yr) <= 1e-5, _rel(y[:, :, rows], yr)

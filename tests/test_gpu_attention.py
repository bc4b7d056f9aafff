"""Neighbourhood attention on an H100: the three kernels of csrc/attention.cu through the C ABI against the fp64 oracle (tests/attention_oracle.py)
on the same fp32 operands, determinism, the module against the oracle (fp32, TF32, bf16 inputs) and FCN3's processor shape on sampled rows."""
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

pytestmark = pytest.mark.gpu

import attention_oracle as AO  # noqa: E402
from makani_b200 import _lib  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.quadrature import _grid_np  # noqa: E402
from makani_b200.sht import _ptr, _stream  # noqa: E402
from test_gpu_parity import close  # noqa: E402

DEV = torch.device("cuda", 0)
RTOL = 1e-5

# (name, in_shape, out_shape, grid_in, grid_out, cutoff in input spacings or None for pi, B, heads, ek, ev, logit magnitude)
# s = 1 and 2; pole rows that span whole rings (equiangular grids, cutoffs of several spacings) and whole rings wider than one staged chunk
# (9 x 520); nlon_out 260 (three longitude tiles, the last ragged); head dims 3, 8, 32, 64 with ek != ev (scalar path at 3); the global limit.
CASES = [
    ("eq17x32-h1-e3x8", (17, 32), (17, 32), "equiangular", "equiangular", 2.5, 1, 1, 3, 8, 3.0),
    ("eq33x64-lg17x32-s2-h4-e8x32", (33, 64), (17, 32), "equiangular", "legendre-gauss", 3.0, 2, 4, 8, 32, 3.0),
    ("lg16x32-h1-e64x32", (16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 2.0, 2, 1, 64, 32, 3.0),
    ("eq21x40-eq21x20-s2-h4-e32x64", (21, 40), (21, 20), "equiangular", "equiangular", 4.0, 1, 4, 32, 64, 3.0),
    ("eq9x520-eq9x260-s2-h1-e64x8-rings", (9, 520), (9, 260), "equiangular", "equiangular", 1.5, 1, 1, 64, 8, 3.0),
    ("lg12x24-h4-e3x64-logits30", (12, 24), (12, 24), "legendre-gauss", "legendre-gauss", 2.5, 2, 4, 3, 64, 30.0),
    ("eq33x64-h4-e32x8-logits30", (33, 64), (33, 64), "equiangular", "equiangular", 3.0, 1, 4, 32, 8, 30.0),
    ("global-eq9x16-lg7x8-h4-e8x3", (9, 16), (7, 8), "equiangular", "legendre-gauss", None, 2, 4, 8, 3, 3.0),
    ("global-lg8x16-h1-e32x64", (8, 16), (8, 16), "legendre-gauss", "legendre-gauss", None, 1, 1, 32, 64, 30.0),
]


def _cutoff(ish, units):
    return math.pi if units is None else units * math.pi / (ish[0] - 1)


def _omega(ish, grid):
    return 2.0 * np.pi * _grid_np(ish[0], grid)[1] / ish[1]


def _operands(ish, osh, B, H, ek, ev, mag, seed):
    """q, k with logits of magnitude about `mag` (scale 1 / sqrt(ek)), v and dy; fp32 on the device"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    sd = math.sqrt(mag)
    q = sd * torch.randn(B, osh[0] * osh[1], H * ek, generator=g, device=DEV)
    k = sd * torch.randn(B, ish[0] * ish[1], H * ek, generator=g, device=DEV)
    v = torch.randn(B, ish[0] * ish[1], H * ev, generator=g, device=DEV)
    dy = torch.randn(B, osh[0] * osh[1], H * ev, generator=g, device=DEV)
    return q, k, v, dy


def _raw(plan, q, k, v, dy, H, scale):
    """the two C-ABI calls on exact shapes (outputs allocated per call)"""
    B = q.shape[0]
    ek, ev = q.shape[2] // H, v.shape[2] // H
    y = torch.full((B, q.shape[1], v.shape[2]), float("nan"), device=DEV)
    lse = torch.full((B, H, q.shape[1]), float("nan"), device=DEV)
    _lib.call("b200sht_attention_forward", plan.handle, _ptr(q), _ptr(k), _ptr(v), _ptr(y), _ptr(lse), B, H, ek, ev, scale, _stream(DEV))
    dq, dk, dv = (torch.full_like(x, float("nan")) for x in (q, k, v))
    D = torch.full_like(lse, float("nan"))
    _lib.call("b200sht_attention_backward", plan.handle, _ptr(q), _ptr(k), _ptr(v), _ptr(y), _ptr(lse), _ptr(dy), _ptr(dq), _ptr(dk), _ptr(dv),
              _ptr(D), B, H, ek, ev, scale, _stream(DEV))
    torch.cuda.synchronize()
    return y, lse, dq, dk, dv, D


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_kernels_against_fp64_oracle(case):
    name, ish, osh, gi, go, units, B, H, ek, ev, mag = case
    nb = A.get_neighbourhood(ish, osh, gi, go, _cutoff(ish, units))
    plan = A.get_plan((ish, osh, gi, go, _cutoff(ish, units)), DEV)
    scale = 1.0 / math.sqrt(ek)
    q, k, v, dy = _operands(ish, osh, B, H, ek, ev, mag, seed=sum(map(ord, name)))
    y, lse, dq, dk, dv, D = _raw(plan, q, k, v, dy, H, scale)
    qr, kr, vr = (x.double().requires_grad_(True) for x in (q, k, v))
    yr, lr = AO.attention(qr, kr, vr, nb.row_ptr, nb.col, _omega(ish, gi), ish[1], osh[1], H, scale)
    yr.backward(dy.double())
    close(y, yr, RTOL, f"{name} y")
    close(lse, lr, RTOL, f"{name} lse")
    close(D, (dy.double() * yr.detach()).view(B, -1, H, ev).sum(-1).transpose(1, 2), RTOL, f"{name} D")
    close(dq, qr.grad, RTOL, f"{name} dq")
    close(dk, kr.grad, RTOL, f"{name} dk")
    close(dv, vr.grad, RTOL, f"{name} dv")


@pytest.mark.parametrize("case", [CASES[1], CASES[4]], ids=[CASES[1][0], CASES[4][0]])
def test_kernels_deterministic(case):
    name, ish, osh, gi, go, units, B, H, ek, ev, mag = case
    plan = A.get_plan((ish, osh, gi, go, _cutoff(ish, units)), DEV)
    q, k, v, dy = _operands(ish, osh, B, H, ek, ev, mag, seed=5)
    a, b = _raw(plan, q, k, v, dy, H, 0.3), _raw(plan, q, k, v, dy, H, 0.3)
    for x, z in zip(a, b):
        assert torch.equal(x, z)


def test_unsupported_head_dim_is_an_error():
    plan = A.get_plan(((17, 32), (17, 32), "equiangular", "equiangular", 0.5), DEV)
    q = torch.zeros(1, 17 * 32, 65, device=DEV)
    with pytest.raises(_lib.B200ShtError, match="exceed 64"):
        _raw(plan, q, q, q, q, 1, 1.0)


MODULE_CASES = [
    # in_channels, in_shape, out_shape, grid_in, grid_out, heads, k_channels, out_channels, bias, cutoff units, separate key / value
    (12, (17, 32), (17, 32), "equiangular", "equiangular", 4, None, None, True, 2.5, False),
    (6, (33, 64), (17, 32), "equiangular", "legendre-gauss", 2, 16, 10, True, 3.0, True),
    (8, (16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 1, 12, 20, False, 2.0, True),
]


def _module_pair(case, seed):
    cin, ish, osh, gi, go, H, ck, cv, bias, units, _ = case
    torch.manual_seed(seed)
    mod = A.NeighborhoodAttentionS2(cin, ish, osh, gi, go, num_heads=H, bias=bias, theta_cutoff=_cutoff(ish, units), k_channels=ck,
                                    out_channels=cv).to(DEV)
    if bias:
        with torch.no_grad():
            for n in ("q_bias", "k_bias", "v_bias", "proj_bias"):
                getattr(mod, n).normal_()
    params = {n: p.detach().double().requires_grad_(True) for n, p in mod.named_parameters()}
    nb = A.get_neighbourhood(*mod._key)
    return mod, params, nb


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("case", MODULE_CASES)
def test_module_against_oracle(case, tf32):
    cin, ish, osh, gi, go, H, ck, cv, bias, units, separate = case
    mod, params, nb = _module_pair(case, 21)
    g = torch.Generator(device=DEV).manual_seed(4)
    query = torch.randn(2, cin, *osh, generator=g, device=DEV)
    key = torch.randn(2, cin, *ish, generator=g, device=DEV) if separate else None
    value = torch.randn(2, cin, *ish, generator=g, device=DEV) if separate else None
    gy = torch.randn(2, mod.out_channels, *osh, generator=g, device=DEV)
    ins = [x.clone().requires_grad_(True) for x in (query, key, value) if x is not None]
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        out = mod(*ins)
        out.backward(gy)
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    refs = [x.double().requires_grad_(True) for x in (query, key, value) if x is not None]
    qk = refs + [refs[0]] * (3 - len(refs))
    ref = AO.module_forward(params, *qk, nb.row_ptr, nb.col, _omega(ish, gi), H, mod.scale)
    ref.backward(gy.double())
    assert out.dtype == torch.float32 and out.shape == ref.shape
    rtol = 2e-3 if tf32 else RTOL
    close(out, ref, rtol, "out")
    for n, (a, b) in enumerate(zip(ins, refs)):
        close(a.grad, b.grad, rtol, f"d input {n}")
    for n, p in mod.named_parameters():
        if n == "k_bias":
            # exactly zero: a key bias adds <q, b> to every logit of a query, and the softmax is invariant to that.  Both sides are rounding
            # noise (fp64 ~1e-14), so hold the library's to the bound of the key weights' gradient, the same sum weighted by the inputs.
            assert p.grad.abs().max().item() <= rtol * params["k_weights"].grad.abs().max().item(), p.grad.abs().max().item()
            continue
        close(p.grad, params[n].grad, rtol, f"d {n}")


def test_module_bf16_inputs():
    case = MODULE_CASES[1]
    cin, ish, osh = case[0], case[1], case[2]
    mod, params, nb = _module_pair(case, 5)
    g = torch.Generator(device=DEV).manual_seed(6)
    xs = [torch.randn(1, cin, *shape, generator=g, device=DEV).to(torch.bfloat16) for shape in (osh, ish, ish)]
    ins = [x.clone().requires_grad_(True) for x in xs]
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        out = mod(*ins)
        out.sum().backward()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    assert out.dtype == torch.float32 and all(x.grad.dtype == torch.bfloat16 for x in ins)
    ref = AO.module_forward(params, *[x.double() for x in xs], nb.row_ptr, nb.col, _omega(ish, case[3]), case[5], mod.scale)
    close(out, ref, RTOL, "bf16 out")


def test_fcn3_processor_shape_on_sampled_rows():
    """360 x 720 Legendre-Gauss, C = 256, 8 heads, theta_cutoff = 4 pi / 359: the module's output against the oracle on both pole rows and a
    seeded sample of the others"""
    ish = osh = (360, 720)
    torch.manual_seed(8)
    cutoff = 4 * math.pi / 359
    mod = A.NeighborhoodAttentionS2(256, ish, osh, "legendre-gauss", "legendre-gauss", num_heads=8, theta_cutoff=cutoff).to(DEV)
    with torch.no_grad():
        for n in ("q_bias", "k_bias", "v_bias", "proj_bias"):
            getattr(mod, n).normal_()
    nb = A.get_neighbourhood(*mod._key)
    rows = [0, 359] + sorted(np.random.default_rng(359).choice(np.arange(1, 359), 6, replace=False).tolist())
    x = torch.randn(1, 256, *ish, generator=torch.Generator(device=DEV).manual_seed(9), device=DEV)
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            out = mod(x)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    params = {n: p.detach().double() for n, p in mod.named_parameters()}
    with torch.no_grad():
        ref = AO.module_forward(params, x.double(), x.double(), x.double(), nb.row_ptr, nb.col, _omega(ish, "legendre-gauss"), 8, mod.scale,
                                rows=rows)
    close(out[:, :, rows], ref, RTOL, f"processor rows {rows}")

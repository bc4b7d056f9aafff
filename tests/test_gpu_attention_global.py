"""Global attention on an H100: the kernels of csrc/attention_global.cu through the C ABI, per element, against fp64 evaluations of the
operands the tensor cores read; bit-identical reruns; AttentionS2 against the fp64 oracle (tests/attention_global_oracle.py) for the
forward and every input and parameter gradient; one sampled-row check at a 361 x 720 output grid.

The per-element reference.  The prep kernel writes every operand of the first GEMMs (q, k, v, dO) rounded to TF32 with cvt.rna, and with
3 x TF32 also lo = rna(x - hi); the tensor core multiplies those values exactly and drops only the lo * lo product.  The reference takes
the same operands (engine_ref.tf32_rna reproduces the rounding bit for bit): a product of two split operands is
(a_hi + a_lo)(b_hi + b_lo) - a_lo b_lo, and at TF32 lo = 0.  It then evaluates o, lse, D = rowsum(dO o) (the row dot reads the fp32 dO),
dS = P (dP - D), dq, dk and dv in fp64 with exact softmax weights P, and products P V, dS K, dS^T Q, P^T dO against hi + lo.

The bound.  What the kernels still round is
  * P and dS, written into their TF32 product tiles: unit u_P = 2^-11 at TF32; at 3 x TF32 the hi + lo pair carries x to 2^-22 and the
    dropped lo * lo product is another 2^-22 |a||b|, so u_P = 2^-21;
  * the fp32 sums (tensor-core accumulation and the running FMAs), expf, the scale / bias FMA, logf and 1 / l: K 2^-24 relative to the
    magnitudes, K the element's fp32 sum length.
Each output element then satisfies |got - ref| <= C (kappa u_P + K 2^-24) sum|terms|, where kappa counts the product-tile roundings on its
path and K its sum lengths:
    o    kappa 1 (P)                         K = nk + dqk
    lse  kappa 0 (l sums unrounded P)        K = nk + dqk
    dq   kappa 2 (dS; o's P through D)       K = nk + dqk + dv
    dk   kappa 2 (dS; o's P through D)       K = nq + nk + dqk + dv   (lse and D come from sums over keys)
    dv   kappa 1 (P)                         K = nq + nk + dqk + dv
sum|terms| carries the logit sensitivities: lab = 1 + scale |q||k| + |b| + |lse| bounds the rounding of each logit and of its exp
argument, and a weight's relative error enters o as P lab |v| plus the shift of 1 / l, lse as P lab, dS as P lab (|dP| + |D|), D as the
error of o through |dO|.  A weight that underflows fp32 (an absolute 2^-126 at most) is a relative 2^-24 error of a weight of 2^-102, so
the magnitudes carry every nonzero P raised by 2^-102.  C is calibrated on an H100 (largest need in DESIGN.md section 4.10); every case
prints each output's worst ratio and the smallest C it would pass with (run with -s).

The case table runs every attention_global_kernel<KIND, DC, SPLIT> instantiation: each row names the DC it launches, runs the forward,
dK / dV and dQ kernels at TF32 and 3 x TF32, and asserts through the profiler that exactly those three instantiations ran (its union is
checked against the built set without a GPU in tests/test_attention_global_cpu.py).  Per DC there are rows whose streamed ring wraps at
least three times, with a partial last streamed block, a partial last resident tile at grid.x >= 3, BH >= 2 and dqk != dv (the smaller
operand's top chunks are TMA zero fill).  The logits column drives the online softmax to its edges: random; large (|scale q.k| near 100,
where an unshifted expf overflows); ascending (every key block's maximum exceeds all before it, so every block rescales); descending
(later blocks underflow to weight 0).  The mask column drops the whole first block and more, the whole last partial block, or every key
but one: there P = 1 and l = 1, so o is that key's operand exactly."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import attention_global_oracle as GO  # noqa: E402
from engine_ref import tf32_rna  # noqa: E402
from makani_b200 import _lib  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from test_gpu_engine import launched_kernels  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
TF32, X3 = _lib.PREC_TF32, _lib.PREC_FP32X3
U_P = {TF32: 2.0 ** -11, X3: 2.0 ** -21}
KAPPA = {"o": 1, "lse": 0, "dq": 2, "dk": 2, "dv": 1}
C_BOUND = 1.0
P_FLOOR = 2.0 ** -102

# (B, H, nq, nk, dqk, dv, logits, mask, DC launched = ceil(max(dqk, dv) / 32))
CASES = [
    # tile-boundary sizes, random logits
    (1, 2, 100, 77, 8, 8, "random", "first", 1), (2, 1, 65, 33, 32, 32, "random", "none", 1),
    (1, 3, 130, 97, 64, 24, "random", "first", 2), (1, 1, 64, 161, 128, 128, "random", "first", 4),
    (1, 2, 31, 200, 16, 104, "random", "none", 4), (1, 1, 1, 5, 40, 8, "random", "none", 2),
    (2, 2, 700, 1100, 64, 64, "random", "first", 2),
    # per DC: rings that wrap three times and more, partial last blocks and tiles, grid.x >= 3, BH >= 2, dqk != dv
    (2, 1, 231, 421, 8, 24, "random", "none", 1), (1, 2, 231, 421, 32, 16, "ascending", "last", 1),
    (2, 1, 231, 421, 24, 8, "large", "first", 1), (1, 2, 231, 421, 16, 32, "descending", "none", 1),
    (1, 2, 231, 421, 64, 40, "random", "first", 2), (2, 1, 231, 421, 48, 56, "large", "none", 2),
    (1, 2, 231, 421, 40, 64, "ascending", "none", 2), (2, 1, 231, 421, 56, 48, "descending", "last", 2),
    (1, 2, 231, 421, 96, 72, "random", "first", 3), (2, 1, 231, 421, 72, 96, "ascending", "none", 3),
    (1, 2, 231, 421, 88, 8, "descending", "last", 3), (2, 1, 231, 421, 8, 88, "large", "none", 3),
    (1, 2, 231, 421, 128, 104, "random", "first", 4), (2, 1, 231, 421, 104, 128, "ascending", "last", 4),
    (1, 2, 231, 421, 120, 16, "large", "none", 4), (2, 1, 231, 421, 16, 120, "descending", "first", 4),
    # exact multiples, single rows and keys, key counts around one block, every key but one
    (2, 1, 128, 64, 96, 72, "random", "none", 3), (1, 2, 128, 64, 24, 16, "random", "none", 1),
    (1, 2, 1, 421, 96, 72, "random", "one", 3), (2, 1, 77, 1, 72, 96, "random", "none", 3),
    (1, 2, 70, 31, 96, 80, "random", "none", 3), (1, 2, 70, 32, 8, 16, "random", "none", 1),
    (1, 2, 70, 33, 112, 64, "random", "none", 4),
    (2, 1, 231, 421, 80, 96, "random", "one", 3), (1, 2, 150, 300, 8, 8, "large", "one", 1),
    (2, 1, 231, 421, 128, 40, "random", "one", 4), (1, 2, 200, 97, 48, 64, "ascending", "last", 2),
]


def _id(c):
    """the parent's ids for its rows (B x H x nq x nk x dqk x dv, m when the first block is dropped), the logits and mask otherwise"""
    s = "x".join(map(str, c[:6])) + ("m" if c[7] == "first" else "")
    return s + ("" if c[6] == "random" else "-" + c[6]) + ("" if c[7] in ("none", "first") else "-" + c[7])


def _case(B, H, nq, nk, dqk, dv, logits, mask, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, H, nq, dqk, device=DEV, generator=g)
    k = torch.randn(B, H, nk, dqk, device=DEV, generator=g)
    v = torch.randn(B, H, dv, nk, device=DEV, generator=g)
    do = torch.randn(B, H, nq, dv, device=DEV, generator=g)
    bias = torch.log(torch.rand(nk, device=DEV, generator=g) * 0.01 + 1e-4)
    j = torch.arange(nk, device=DEV, dtype=torch.float32)
    if logits == "large":        # scale q.k ~ N(0, 60^2): |logits| around 100, past 88.7 in most rows
        q = q * 60.0
    elif logits == "ascending":  # 2 per 32-key block against a q.k spread of ~0.1: each block's maximum is the largest so far
        q, bias = q * 0.1, 2.0 * torch.div(j, 32, rounding_mode="floor")
    elif logits == "descending":  # exp(-0.5 j): keys past ~210 weigh below fp32's smallest subnormal
        q, bias = q * 0.1, -0.5 * j
    if mask == "first":
        bias[: min(40, nk - 1)] = -torch.inf   # the whole first key block and part of the second drop out
        bias[45::7] = -torch.inf
    elif mask == "last":
        bias[(nk - 1) // 32 * 32:] = -torch.inf   # the whole last, partial block
    elif mask == "one":
        bias[torch.arange(nk, device=DEV) != nk // 2] = -torch.inf
    return q, k, v, do, bias


def _split(x, prec):
    """(hi, lo) in fp64: what the prep kernel writes for fp32 operand x (lo = 0 at TF32)"""
    hi = tf32_rna(x)
    lo = tf32_rna(x - hi) if prec == X3 else torch.zeros_like(hi)
    return hi.double(), lo.double()


def _mm(a, b):
    """a @ b of split operands as the tensor core forms it: every product but lo * lo"""
    return (a[0] + a[1]) @ (b[0] + b[1]) - a[1] @ b[1]


def _t(a):
    return tuple(x.transpose(-1, -2) for x in a)


def _reference(q, k, v, do, bias, scale, prec):
    """fp64 o, lse, dq, dk, dv of the operands the kernels read, the sums of absolute terms that bound each element's error, and P"""
    Q, K, V, dO = (_split(t, prec) for t in (q, k, v, do))
    Qe, Ke, Ve, dOe = (x[0] + x[1] for x in (Q, K, V, dO))
    b = bias.double()
    s = scale * _mm(Q, _t(K)) + b
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    o = p @ Ve.transpose(-1, -2)
    dp = _mm(dO, V)
    D = (do.double() * o).sum(-1)
    ds = p * (dp - D[..., None])
    dq, dk, dv = scale * ds @ Ke, scale * ds.transpose(-1, -2) @ Qe, dOe.transpose(-1, -2) @ p
    pm = p + P_FLOOR * (p > 0)
    lab = 1.0 + scale * Qe.abs() @ Ke.abs().transpose(-1, -2) + torch.where(b.isfinite(), b.abs(), 0.0) + lse.abs()[..., None]
    pl = pm * lab
    ao = pl @ Ve.abs().transpose(-1, -2) + pl.sum(-1, keepdim=True) * o.abs()
    alse = pl.sum(-1) + lse.abs()
    adp = dOe.abs() @ Ve.abs()
    aD = (do.double().abs() * (ao + o.abs())).sum(-1)
    ads = pl * (dp.abs() + D.abs()[..., None]) + pm * (adp + aD[..., None]) + ds.abs()
    adq, adk = scale * ads @ Ke.abs(), scale * ads.transpose(-1, -2) @ Qe.abs()
    adv = dOe.abs().transpose(-1, -2) @ pl
    return (o, lse, dq, dk, dv), (ao, alse, adq, adk, adv), p


def _run(q, k, v, do, bias, scale, prec):
    o, lse = A.global_attention_forward(q, k, v, bias, scale, prec)
    dq, dk, dv = A.global_attention_backward(q, k, v, bias, o, lse, do, scale, prec)
    torch.cuda.synchronize()
    return o, lse, dq, dk, dv


# the profiler reports void b200sht::attention_global_kernel<0, 3, true>(b200sht::AgParams); cu++filt may print (int)0, (bool)1
AG_KERNEL = re.compile(r"attention_global_kernel<(?:\(int\))?(\d), (?:\(int\))?(\d), (?:\(bool\))?(0|1|false|true)>")


def ag_kernels(names):
    return {(int(m[1]), int(m[2]), m[3] in ("1", "true")) for m in map(AG_KERNEL.search, names) if m}


def case_kernels(case, prec):
    """the (KIND, DC, SPLIT) instantiations one forward + backward of `case` launches"""
    return {(kind, case[-1], prec == X3) for kind in range(3)}


def _edges(case, p, lse, bias):
    """the logits and masks do what their names say (p, lse: the reference's)"""
    nk, logits, mask = case[3], case[6], case[7]
    lg = p.log()
    if logits == "large":                                 # some row's largest logit is past 88.7, where an unshifted expf overflows
        assert (lg.amax(-1) + lse > 88.7).any()
    lg = lg - lg.amax(-1, keepdim=True)                   # logits less the row's largest; -inf where masked
    if logits in ("ascending", "descending"):
        live = [i for i in range(0, nk, 32) if bias[i: i + 32].isfinite().any()]   # the blocks with a key left
        bmax = torch.stack([lg[..., i: i + 32].amax(-1) for i in live], -1)
        if logits == "ascending":
            assert len(live) >= 3 and (bmax[..., 1:] > bmax[..., :-1]).all()
        else:                                             # the last live block's every weight rounds to 0 in fp32
            assert (bmax[..., -1] < np.log(2.0 ** -150)).all()
    if mask == "one":
        assert int(bias.isfinite().sum()) == 1


@pytest.mark.parametrize("prec", [TF32, X3], ids=["tf32", "fp32x3"])
@pytest.mark.parametrize("case", CASES, ids=_id)
def test_kernels_per_element_against_fp64_of_their_operands(case, prec):
    B, H, nq, nk, dqk, dv, logits, mask, dc = case
    q, k, v, do, bias = _case(B, H, nq, nk, dqk, dv, logits, mask, seed=nq * 7 + nk)
    scale = 1.0 / np.sqrt(dqk)
    got = _run(q, k, v, do, bias, scale, prec)
    ref, terms, p = _reference(q, k, v, do, bias, scale, prec)
    _edges(case, p, ref[1], bias)
    lengths = {"o": nk + dqk, "lse": nk + dqk, "dq": nk + dqk + dv, "dk": nq + nk + dqk + dv, "dv": nq + nk + dqk + dv}
    worst, need = {}, {}
    for name, g, r, t in zip(("o", "lse", "dq", "dk", "dv"), got, ref, terms):
        assert torch.isfinite(g).all(), name
        unit = KAPPA[name] * U_P[prec] + lengths[name] * 2.0 ** -24
        err = (g.double() - r).abs()
        rel = torch.where(err == 0, torch.zeros_like(err), err / (unit * t))
        need[name] = rel.max().item()
        worst[name] = need[name] / C_BOUND
    print(f"\n[attention_global] {_id(case)} {'tf32' if prec == TF32 else 'fp32x3'}: worst ratio / needs C >=",
          {n: f"{worst[n]:.3g} / {need[n]:.3g}" for n in worst}, f"(C = {C_BOUND})")
    bad = {n: r for n, r in worst.items() if r > 1.0}
    assert not bad, bad
    if mask != "none":
        assert (got[3][:, :, bias.isinf()] == 0).all() and (got[4][..., bias.isinf()] == 0).all()
    if mask == "one":   # P = 1, l = 1: o is the key's operand, hi + lo summed in the tensor core's fp32 accumulator
        hi, lo = (x[..., nk // 2] for x in _split(v, prec))
        want = (hi + lo).float()[:, :, None, :].expand_as(got[0])
        if prec == TF32:
            assert torch.equal(got[0], want)
        else:
            assert ((got[0] - want).abs() <= 2.0 ** -23 * want.abs()).all()
    again = _run(q, k, v, do, bias, scale, prec)
    for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), got, again):
        assert torch.equal(x, y), f"rerun differs: {name}"
    want = case_kernels(case, prec)
    names = launched_kernels(lambda: _run(q, k, v, do, bias, scale, prec), lambda n: ag_kernels(n) == want)
    assert ag_kernels(names) == want, f"expected {sorted(want)}, launched {names}"
    print(f"[attention_global] {_id(case)} launched (KIND, DC, SPLIT) {sorted(ag_kernels(names))}")


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
                ((17, 32), (33, 64), 32, 1, 64, 128, "equiangular"), ((10, 20), (6, 12), 16, 2, 160, 192, "legendre-gauss")]


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

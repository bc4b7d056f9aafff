"""Neighbourhood attention on an H100: the three kernels of csrc/attention.cu through the C ABI, determinism, the module against the oracle
(fp32, TF32, bf16 inputs) and FCN3's processor shape on sampled rows.

Every kernel case is checked twice.  Against the contract oracle (tests/attention_oracle.py) on the same fp32 operands, with
`test_gpu_parity.close` (normwise, rtol 1e-5): that pins the end-to-end semantics, forward and autograd backward.  And element by element
against the fp64 references of tests/attention_ref.py on the kernels' exact operands (the scaled query fl(scale q), the plan's fp32 weights,
and for the backward the forward kernel's own fp32 y and lse): |got - ref| <= C_ATTN 2^-24 mag, with the first-order rounding bound derived in
that module.  Every output is written inside a NaN sentinel buffer whose padding must stay untouched, and every case asserts through the
profiler which attn_query_kernel / attn_kv_kernel instantiations it launched."""
import math
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

pytestmark = pytest.mark.gpu

import attention_oracle as AO  # noqa: E402
import attention_ref as AR  # noqa: E402
from makani_b200 import _lib  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.quadrature import _grid_np  # noqa: E402
from makani_b200.sht import _ptr, _stream  # noqa: E402
from test_gpu_engine import launched_kernels  # noqa: E402
from test_gpu_parity import close  # noqa: E402

DEV = torch.device("cuda", 0)
RTOL = 1e-5
# C of the per-element bound |got - ref| <= C 2^-24 mag of tests/attention_ref.py, calibrated on an H100 (DESIGN.md sections 4.9 and 5)
C_ATTN = 1.0

# (name, in_shape, out_shape, grid_in, grid_out, cutoff in input spacings or None for pi, B, heads, ek, ev, logits, storage offset in floats of
# every operand and output, (EM, VEC) the row must launch).  logits: the magnitude of random logits, or "ascending" / "descending" for logits
# monotone in the input latitude (see _operands).
# s = 1, 2, 3 and 4; pole rows that span whole rings (equiangular grids, cutoffs of several spacings) and whole rings wider than one staged chunk
# (9 x 520); nlon_out 260 (three longitude tiles, the last ragged) and 450 -> 150 (ragged last tiles on both sides: 150 = 128 + 22 output
# longitudes for the query-side kernels, 450 = 7 * 64 + 2 input longitudes for the key/value kernel); single-point neighbourhoods (alpha = 1,
# dl pure cancellation); logits that force a running-max rescale at every band row or at none, and logits about 100, where exp(l) alone
# overflows fp32; the global limit.  Together the rows launch every (EM, VEC) pair of csrc/attention.cu: the scalar path with odd head dims and
# with multiples of 4 at a 4-byte storage offset (vec_ok routes unaligned operands there).
CASES = [
    ("eq17x32-h1-e3x8", (17, 32), (17, 32), "equiangular", "equiangular", 2.5, 1, 1, 3, 8, 3.0, 0, (8, False)),
    ("eq33x64-lg17x32-s2-h4-e8x32", (33, 64), (17, 32), "equiangular", "legendre-gauss", 3.0, 2, 4, 8, 32, 3.0, 0, (32, True)),
    ("lg16x32-h1-e64x32", (16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 2.0, 2, 1, 64, 32, 3.0, 0, (64, True)),
    ("eq21x40-eq21x20-s2-h4-e32x64", (21, 40), (21, 20), "equiangular", "equiangular", 4.0, 1, 4, 32, 64, 3.0, 0, (64, True)),
    ("eq9x520-eq9x260-s2-h1-e64x8-rings", (9, 520), (9, 260), "equiangular", "equiangular", 1.5, 1, 1, 64, 8, 3.0, 0, (64, True)),
    ("lg12x24-h4-e3x64-logits30", (12, 24), (12, 24), "legendre-gauss", "legendre-gauss", 2.5, 2, 4, 3, 64, 30.0, 0, (64, False)),
    ("eq33x64-h4-e32x8-logits30", (33, 64), (33, 64), "equiangular", "equiangular", 3.0, 1, 4, 32, 8, 30.0, 0, (32, True)),
    ("global-eq9x16-lg7x8-h4-e8x3", (9, 16), (7, 8), "equiangular", "legendre-gauss", None, 2, 4, 8, 3, 3.0, 0, (8, False)),
    ("global-lg8x16-h1-e32x64", (8, 16), (8, 16), "legendre-gauss", "legendre-gauss", None, 1, 1, 32, 64, 30.0, 0, (64, True)),
    ("lg16x96-lg16x32-s3-h2-e4x4", (16, 96), (16, 32), "legendre-gauss", "legendre-gauss", 2.5, 1, 2, 4, 4, 3.0, 0, (4, True)),
    ("eq17x128-eq17x32-s4-h1-e8x4", (17, 128), (17, 32), "equiangular", "equiangular", 2.5, 2, 1, 8, 4, 3.0, 0, (8, True)),
    ("eq9x450-eq9x150-s3-h2-e16x16-ragged", (9, 450), (9, 150), "equiangular", "equiangular", 1.5, 1, 2, 16, 16, 3.0, 0, (16, True)),
    ("lg16x32-h3-e12x16-single-point", (16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 0.05, 1, 3, 12, 16, 3.0, 0, (16, True)),
    ("eq17x32-h2-e3x3-ascending", (17, 32), (17, 32), "equiangular", "equiangular", 2.5, 1, 2, 3, 3, "ascending", 0, (4, False)),
    ("lg12x24-eq13x24-h1-e15x16-descending", (12, 24), (13, 24), "legendre-gauss", "equiangular", 3.0, 2, 1, 15, 16, "descending", 0,
     (16, False)),
    ("eq33x64-h2-e30x29-logits100", (33, 64), (33, 64), "equiangular", "equiangular", 2.0, 1, 2, 30, 29, 100.0, 0, (32, False)),
    ("eq17x32-lg16x32-h2-e16x12-offset4B", (17, 32), (16, 32), "equiangular", "legendre-gauss", 2.5, 1, 2, 16, 12, 3.0, 1, (16, False)),
    ("lg16x64-lg16x32-s2-h1-e32x32-offset4B", (16, 64), (16, 32), "legendre-gauss", "legendre-gauss", 2.0, 2, 1, 32, 32, 3.0, 1, (32, False)),
    ("eq21x40-h2-e64x48-offset4B-logits30", (21, 40), (21, 40), "equiangular", "equiangular", 2.0, 1, 2, 64, 48, 30.0, 1, (64, False)),
]


def em_vec(ek, ev, off):
    """(EM, VEC) that csrc/attention.cu dispatches to (head_em, vec_ok) for head dims ek, ev and operands at a storage offset of `off` floats
    from 16-byte-aligned allocations"""
    e = max(ek, ev)
    return next(m for m in (4, 8, 16, 32, 64) if e <= m), ek % 4 == 0 and ev % 4 == 0 and off % 4 == 0


def attn_kernels(em, vec):
    """the three instantiations one forward + backward launches: (kernel, EM, VEC, QUERY or None)"""
    return {("attn_query_kernel", em, vec, False), ("attn_query_kernel", em, vec, True), ("attn_kv_kernel", em, vec, None)}


# the profiler reports void b200sht::attn_query_kernel<16, true, false>(...); cu++filt prints (int)16, (bool)1, (bool)0
ATTN_KERNEL = re.compile(r"(attn_query_kernel|attn_kv_kernel)<(?:\(int\))?(\d+), (?:\(bool\))?(0|1|false|true)(?:, (?:\(bool\))?(0|1|false|true))?>")


def _launched_attn(names):
    return {(m[1], int(m[2]), m[3] in ("1", "true"), None if m[4] is None else m[4] in ("1", "true")) for m in map(ATTN_KERNEL.search, names) if m}


def _cutoff(ish, units):
    return math.pi if units is None else units * math.pi / (ish[0] - 1)


def _omega(ish, grid):
    return 2.0 * np.pi * _grid_np(ish[0], grid)[1] / ish[1]


def _operands(ish, osh, B, H, ek, ev, logits, seed):
    """q, k, v and dy, fp32 on the device.  A number `logits`: random q, k with logits of about that magnitude (scale 1 / sqrt(ek)).
    "ascending" / "descending": every q and k of a head on one direction d, q = a sqrt(ek) d with a in [0.5, 1.5) per point and k = g(i) d, so
    l = a g(i) with g monotone in the input latitude i, from -6 to 6 or back.  The kernels walk t's band by ascending i: ascending logits
    force a running-max rescale at every band row, descending ones none after the first point."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if isinstance(logits, str):
        d = torch.randn(H, ek, generator=g, device=DEV)
        d = d / d.norm(dim=1, keepdim=True)
        a = 0.5 + torch.rand(B, osh[0] * osh[1], H, 1, generator=g, device=DEV)
        q = (a * math.sqrt(ek) * d).reshape(B, -1, H * ek)
        lat = torch.linspace(-6.0, 6.0, ish[0], device=DEV) * (1 if logits == "ascending" else -1)
        k = (lat.repeat_interleave(ish[1]).view(1, -1, 1, 1) * d).expand(B, -1, -1, -1).reshape(B, -1, H * ek).contiguous()
    else:
        sd = math.sqrt(logits)
        q = sd * torch.randn(B, osh[0] * osh[1], H * ek, generator=g, device=DEV)
        k = sd * torch.randn(B, ish[0] * ish[1], H * ek, generator=g, device=DEV)
    v = torch.randn(B, ish[0] * ish[1], H * ev, generator=g, device=DEV)
    dy = torch.randn(B, osh[0] * osh[1], H * ev, generator=g, device=DEV)
    return q, k, v, dy


PAD = 1024   # floats of NaN on each side of every output


def _at_offset(x, off):
    """x copied to `off` floats past a 16-byte-aligned allocation (the C ABI takes any fp32 pointer)"""
    if not off:
        return x
    buf = torch.empty(x.numel() + off, device=DEV)
    buf[off:].copy_(x.reshape(-1))
    return buf[off:].view(x.shape)


def _sentinel(shape, off):
    """(buffer, view): the view starts `off` floats past PAD NaNs and is followed by PAD NaNs"""
    n = int(np.prod(shape))
    buf = torch.full((PAD + off + n + PAD,), float("nan"), device=DEV)
    return buf, buf[PAD + off : PAD + off + n].view(shape)


def _untouched(buf, x):
    o = x.storage_offset()
    return bool(torch.isnan(buf[:o]).all() and torch.isnan(buf[o + x.numel() :]).all())


def _run(plan, q, k, v, dy, H, scale, off=0):
    """the two C-ABI calls on exact shapes, every output inside a NaN sentinel buffer at storage offset `off`:
    ((y, lse, dq, dk, dv, D), their buffers)"""
    B = q.shape[0]
    ek, ev = q.shape[2] // H, v.shape[2] // H
    bufs, outs = zip(*(_sentinel(shape, off) for shape in (
        (B, q.shape[1], v.shape[2]), (B, H, q.shape[1]), q.shape, k.shape, v.shape, (B, H, q.shape[1]))))
    y, lse, dq, dk, dv, D = outs
    _lib.call("b200sht_attention_forward", plan.handle, _ptr(q), _ptr(k), _ptr(v), _ptr(y), _ptr(lse), B, H, ek, ev, scale, _stream(DEV))
    _lib.call("b200sht_attention_backward", plan.handle, _ptr(q), _ptr(k), _ptr(v), _ptr(y), _ptr(lse), _ptr(dy), _ptr(dq), _ptr(dk), _ptr(dv),
              _ptr(D), B, H, ek, ev, scale, _stream(DEV))
    torch.cuda.synchronize()
    return outs, bufs


def _raw(plan, q, k, v, dy, H, scale):
    return _run(plan, q, k, v, dy, H, scale)[0]


def _plan_omega(nb, nlat_in, nlon_in):
    """the plan's fp32 quadrature weight of every input latitude (0 where no output row reaches it)"""
    om = np.zeros(nlat_in)
    om[np.asarray(nb.col) // nlon_in] = nb.val
    return om.astype(np.float32).astype(np.float64)


NEEDS = {}


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_kernels_against_fp64_oracle(case):
    name, ish, osh, gi, go, units, B, H, ek, ev, logits, off, (em, vec) = case
    assert em_vec(ek, ev, off) == (em, vec), f"{name}: the row says {(em, vec)}, the dispatch picks {em_vec(ek, ev, off)}"
    nb = A.get_neighbourhood(ish, osh, gi, go, _cutoff(ish, units))
    plan = A.get_plan((ish, osh, gi, go, _cutoff(ish, units)), DEV)
    single = bool((np.diff(nb.row_ptr) == 1).all())
    assert single == name.endswith("single-point"), f"{name}: neighbourhood sizes {np.unique(np.diff(nb.row_ptr))}"
    scale = 1.0 / math.sqrt(ek)
    q, k, v, dy = (_at_offset(x, off) for x in _operands(ish, osh, B, H, ek, ev, logits, seed=sum(map(ord, name))))
    (y, lse, dq, dk, dv, D), bufs = _run(plan, q, k, v, dy, H, scale, off)
    for what, buf, x in zip(("y", "lse", "dq", "dk", "dv", "D"), bufs, (y, lse, dq, dk, dv, D)):
        assert _untouched(buf, x), f"{name}: a kernel wrote outside {what}"
        assert not torch.isnan(x).any(), f"{name}: {what} has unwritten (NaN) elements"
    want = attn_kernels(em, vec)
    names = launched_kernels(lambda: _run(plan, q, k, v, dy, H, scale, off), lambda n: _launched_attn(n) == want)
    assert _launched_attn(names) == want, f"{name}: expected {sorted(want, key=str)}, launched {names}"

    # the contract oracle on the same fp32 operands (normwise).  The softmax's sensitivity to its logits grows with their size, so the rtol
    # grows with the logit magnitude beyond the 30 the 1e-5 was measured at.  With single-point neighbourhoods the exact dq and dk are zero
    # (the softmax of one logit is 1 whatever the logit): the per-element bound below holds them to their rounding instead.
    rtol = RTOL * max(1.0, logits / 30.0) if not isinstance(logits, str) else RTOL
    qr, kr, vr = (x.double().requires_grad_(True) for x in (q, k, v))
    yr, lr = AO.attention(qr, kr, vr, nb.row_ptr, nb.col, _omega(ish, gi), ish[1], osh[1], H, scale)
    yr.backward(dy.double())
    close(y, yr, rtol, f"{name} y")
    close(lse, lr, rtol, f"{name} lse")
    close(D, (dy.double() * yr.detach()).view(B, -1, H, ev).sum(-1).transpose(1, 2), rtol, f"{name} D")
    if not single:
        close(dq, qr.grad, rtol, f"{name} dq")
        close(dk, kr.grad, rtol, f"{name} dk")
    close(dv, vr.grad, rtol, f"{name} dv")

    # per element against fp64 on the kernels' exact operands
    s32 = torch.tensor(scale, dtype=torch.float32, device=DEV)
    qt = (q * s32).double()
    om = _plan_omega(nb, ish[0], ish[1])
    (yx, my), (lx, ml) = AR.forward(qt, k.double(), v.double(), nb.row_ptr, nb.col, om, ish[1], osh[1], H)
    bw = AR.backward(qt, k.double(), v.double(), y.double(), lse.double(), dy.double(), nb.row_ptr, nb.col, om, ish[1], osh[1], H, s32.item())
    needs = {"y": AR.need(y, yx, my), "lse": AR.need(lse, lx, ml)}
    for what, got in (("D", D), ("dq", dq), ("dk", dk), ("dv", dv)):
        needs[what] = AR.need(got, *bw[what])
    NEEDS[name] = needs
    print(f"\n[attention] {name}: ran {' '.join(sorted(names))}")
    print(f"[attention] {name}: needs C >= " + ", ".join(f"{w} {c:.3g}" for w, c in needs.items()) + f" (C = {C_ATTN})")
    bad = {w: c for w, c in needs.items() if not c <= C_ATTN}
    assert not bad, f"{name}: outside the per-element bound: needs C = {bad}"


@pytest.mark.parametrize("case", [CASES[1], CASES[4]], ids=[CASES[1][0], CASES[4][0]])
def test_kernels_deterministic(case):
    name, ish, osh, gi, go, units, B, H, ek, ev, mag = case[:11]
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

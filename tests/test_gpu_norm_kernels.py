"""The pointwise kernels of the SFNO block (csrc/norm.cu) through the C ABI, against fp64 references of their exact operands
(tests/engine_ref.py): instance norm (+ GELU) forward and backward, including the `stats` and `sums` buffers, and bias + GELU.

Statistics: |mean - mean64| <= 1e-6 sigma64 + 2^-24 |mean64| (the stored mean is one fp32 rounding) and |rstd / rstd64 - 1| <= 1e-6,
whatever the row holds: an offset far larger than its spread, an outlier at x[row, 0] (the pivot the statistics are taken about) or
elsewhere, a constant row.  y and dx are checked against fp64 of the kernel's own stored statistics and sums, per element in units of
2^-24 times the magnitudes of their terms (`C_POINTWISE`; GELU adds erff / __expf, bf16 one output rounding).  The sums are held to
c K 2^-24 sum |term| with K the length of the per-thread chain plus the tree.  Every output is surrounded by NaN sentinels.  Every
check prints the smallest constant it would pass with (run with -s)."""
import math

import pytest
import torch

import engine_ref as E
from makani_b200 import _lib
from makani_b200.sht import _ptr, _stream
from test_gpu_engine import DEV, call

pytestmark = pytest.mark.gpu
EPS = 1e-6
STAT_TOL = 1e-6
# per-element constant of y / dx in units of 2^-24 x (magnitudes of the terms), calibrated on an H100 (DESIGN.md section 5)
C_POINTWISE = 16.0
R_BF16 = 2.0 ** -8
PAD = 64            # sentinel elements on each side of every output
SENT = {torch.float32: (torch.int32, 0x7FC05EED), torch.bfloat16: (torch.int16, 0x7FC5)}

# id, dtype, B, C, n, element offset of x (1: not 16-byte aligned, no vector path)
SHAPES = [
    ("one-split-n1000", torch.float32, 2, 3, 1000, 0),
    ("splits-n8320", torch.float32, 1, 4, 8320, 0),
    ("64-splits-721x1440", torch.float32, 1, 1, 721 * 1440, 0),
    ("scalar-n4097", torch.float32, 2, 3, 4097, 0),
    ("bf16-splits-n8320", torch.bfloat16, 1, 4, 8320, 0),
    ("bf16-scalar-n8196", torch.bfloat16, 2, 3, 8196, 0),
    ("misaligned-x", torch.float32, 1, 4, 8320, 1),
    ("rows65535-n16", torch.float32, 5, 13107, 16, 0),
]
DATA = ["normal", "offset1e3-std1e-2", "pivot-outlier-30sigma", "pivot-outlier-1000sigma", "mid-outlier-1000sigma", "constant"]


def _dt(dtype):
    return _lib.BF16 if dtype == torch.bfloat16 else _lib.F32


def _data(kind, rows, n, gen):
    x = torch.randn(rows, n, dtype=torch.float64, device=DEV, generator=gen)
    if kind == "offset1e3-std1e-2":
        x = 1e3 + 1e-2 * x
    elif kind.endswith("sigma"):
        x[:, 0 if kind.startswith("pivot") else n // 2 + 1] = float(kind.split("-")[-1][:-5])
    elif kind == "constant":
        x[:] = 0.75
    return x


def _padded(dtype, numel, offset=0):
    """a sentinel-filled buffer and the view of `numel` elements PAD + offset into it"""
    it, bits = SENT[dtype]
    buf = torch.full((numel + 2 * PAD + offset,), bits, dtype=it, device=DEV).view(dtype)
    return buf, buf[PAD + offset: PAD + offset + numel]


def _untouched(buf, numel, offset=0):
    it, bits = SENT[buf.dtype]
    raw = buf.view(it)
    return bool((raw[: PAD + offset] == bits).all() and (raw[PAD + offset + numel:] == bits).all())


def _report(tag, what, got, ref, mag, K=1, r=0.0, c=C_POINTWISE, extra=0.0):
    ratio = E.bound_ratio(got, ref, mag, K, r=r, c=c, extra=extra)
    need = E.needed_c(got, ref, mag, K, r=r, extra=extra)
    print(f"[pointwise] {tag} {what}: worst ratio {ratio:.3e}, needs c >= {need:.3e} (c = {c})")
    assert ratio <= 1.0, f"{tag} {what}: exceeds the bound by {ratio:.3g}x"


def _chain(rows, n):
    """K of a row sum: the longest per-thread chain, the 256-thread tree and the fp64 sum over the splits"""
    splits = int(_lib.load().b200sht_pointwise_workspace_floats(1, rows, n)) // (2 * rows)
    return math.ceil(n / (256 * splits)) + 8 + splits


@pytest.mark.parametrize("gelu", [False, True], ids=["norm", "norm+gelu"])
@pytest.mark.parametrize("kind", DATA)
@pytest.mark.parametrize("case,dtype,B,C,n,off", SHAPES, ids=[s[0] for s in SHAPES])
def test_instance_norm(case, dtype, B, C, n, off, kind, gelu):
    gen = torch.Generator(device=DEV).manual_seed(8642)
    rows = B * C
    tag = f"{case} {kind} {'gelu' if gelu else 'plain'}"
    st = _stream(DEV)
    x64 = _data(kind, rows, n, gen)
    xbuf, xs = _padded(dtype, rows * n, off)
    xs.copy_(x64.reshape(-1).to(dtype))
    xd = xs.view(rows, n).double()                                   # the exact stored operand
    gamma = (torch.randn(C, device=DEV, generator=gen) * 0.5 + 1.0)
    beta = torch.randn(C, device=DEV, generator=gen) * 0.3
    ws = torch.full((int(_lib.load().b200sht_pointwise_workspace_floats(B, C, n)),), float("nan"), device=DEV)
    ybuf, ys = _padded(dtype, rows * n)
    sbuf, stats = _padded(torch.float32, rows * 2)
    call("b200sht_instance_norm_forward", _ptr(xs), _ptr(ys), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(ws), _dt(dtype), B, C, n, EPS, int(gelu), st)
    assert _untouched(ybuf, rows * n) and _untouched(sbuf, rows * 2), f"{tag}: a write outside y / stats"

    # statistics
    mean64, var64 = E.norm_stats_ref(xd)
    rstd64 = 1.0 / torch.sqrt(var64 + EPS)
    mk, rk = stats.view(rows, 2)[:, 0].double(), stats.view(rows, 2)[:, 1].double()
    em = ((mk - mean64).abs() / (STAT_TOL * var64.sqrt() + E.U32 * mean64.abs())).max().item()
    er = ((rk / rstd64 - 1.0).abs() / STAT_TOL).max().item()
    print(f"[pointwise] {tag} stats: mean error {em:.3e}, rstd error {er:.3e} (x the bounds)")
    assert em <= 1.0 and er <= 1.0, f"{tag}: statistics off by {em:.3g}x (mean) / {er:.3g}x (rstd) of the bound"
    if kind == "constant":
        assert (rk == torch.tensor(1.0 / math.sqrt(EPS), dtype=torch.float32).double()).all()

    # y from the kernel's stats: z = fma((x - mean) rstd, gamma, beta), one rounding per step
    g64, b64 = gamma.double()[None, :, None], beta.double()[None, :, None]
    xh = ((xd - mk[:, None]) * rk[:, None]).view(B, C, n)
    z = xh * g64 + b64
    magz = xh.abs() * g64.abs() + b64.abs()
    if gelu:
        yref, magy = E.gelu_ref(z), E.gelu_grad_ref(z).abs() * magz + z.abs()
    else:
        yref, magy = z, magz
    _report(tag, "y", ys.view(B, C, n), yref, magy, r=R_BF16 if dtype == torch.bfloat16 else 0.0)
    if kind == "constant" and not gelu:
        assert (ys.view(B, C, n) == beta.to(dtype)[None, :, None]).all(), f"{tag}: a constant row must give y = beta"

    # backward, from the same stats
    dy64 = torch.randn(rows, n, dtype=torch.float64, device=DEV, generator=gen)
    dybuf, dys = _padded(dtype, rows * n)
    dys.copy_(dy64.reshape(-1).to(dtype))
    dyd = dys.view(B, C, n).double()
    dxbuf, dxs = _padded(dtype, rows * n)
    subuf, sums = _padded(torch.float32, rows * 2)
    ws.fill_(float("nan"))
    call("b200sht_instance_norm_backward", _ptr(xs), _ptr(dys), _ptr(dxs), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(sums), _ptr(ws), _dt(dtype),
         B, C, n, int(gelu), st)
    assert _untouched(dxbuf, rows * n) and _untouched(subuf, rows * 2), f"{tag}: a write outside dx / sums"
    gp = E.gelu_grad_ref(z) if gelu else torch.ones_like(z)
    g = dyd * gp
    magg = dyd.abs() * (gp.abs() + (1.0 if gelu else 0.0))     # erff / __expf in gelu'
    S1, S2 = g.sum(-1).reshape(-1), (g * xh).sum(-1).reshape(-1)
    M1, M2 = magg.sum(-1).reshape(-1), (magg * xh.abs()).sum(-1).reshape(-1)
    sk = sums.view(rows, 2).double()
    K = _chain(rows, n)
    _report(tag, "sum g", sk[:, 0], S1, M1, K=K, c=E.C_ACC, extra=4 * E.U32)
    _report(tag, "sum g xhat", sk[:, 1], S2, M2, K=K, c=E.C_ACC, extra=4 * E.U32)
    # dx = rstd gamma (g - S1 / n - xhat S2 / n) with the kernel's sums
    s1n, s2n = (sk[:, 0] / n).view(B, C, 1), (sk[:, 1] / n).view(B, C, 1)
    gs = rk.view(B, C, 1) * g64
    dxref = gs * (g - s1n - xh * s2n)
    magdx = gs.abs() * (magg + s1n.abs() + xh.abs() * s2n.abs())
    _report(tag, "dx", dxs.view(B, C, n), dxref, magdx, r=R_BF16 if dtype == torch.bfloat16 else 0.0)


@pytest.mark.parametrize("case,dtype,B,C,n,off", SHAPES, ids=[s[0] for s in SHAPES])
def test_bias_gelu(case, dtype, B, C, n, off):
    gen = torch.Generator(device=DEV).manual_seed(1357)
    rows = B * C
    st = _stream(DEV)
    xbuf, xs = _padded(dtype, rows * n, off)
    xs.copy_((torch.randn(rows * n, device=DEV, generator=gen) * 1.5).to(dtype))
    xd = xs.view(B, C, n).double()
    bias = torch.randn(C, device=DEV, generator=gen)
    bd = bias.double()[None, :, None]
    ybuf, ys = _padded(dtype, rows * n)
    call("b200sht_bias_gelu_forward", _ptr(xs), _ptr(bias), _ptr(ys), _dt(dtype), B, C, n, st)
    assert _untouched(ybuf, rows * n), f"{case}: a write outside y"
    z = xd + bd
    r = R_BF16 if dtype == torch.bfloat16 else 0.0
    _report(case, "bias+gelu y", ys.view(B, C, n), E.gelu_ref(z), E.gelu_grad_ref(z).abs() * (xd.abs() + bd.abs()) + z.abs(), r=r)

    dybuf, dys = _padded(dtype, rows * n)
    dys.copy_(torch.randn(rows * n, device=DEV, generator=gen).to(dtype))
    dyd = dys.view(B, C, n).double()
    dxbuf, dxs = _padded(dtype, rows * n)
    rbuf, rs = _padded(torch.float32, rows * 2)
    ws = torch.full((int(_lib.load().b200sht_pointwise_workspace_floats(B, C, n)),), float("nan"), device=DEV)
    call("b200sht_bias_gelu_backward", _ptr(xs), _ptr(bias), _ptr(dys), _ptr(dxs), _ptr(rs), _ptr(ws), _dt(dtype), B, C, n, st)
    assert _untouched(dxbuf, rows * n) and _untouched(rbuf, rows * 2), f"{case}: a write outside dx / row sums"
    gp = E.gelu_grad_ref(z)
    gpp = (torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)) * (2.0 - z * z)
    dxref = dyd * gp
    mag = dyd.abs() * (gp.abs() + gpp.abs() * (xd.abs() + bd.abs()) + 1.0)
    _report(case, "bias+gelu dx", dxs.view(B, C, n), dxref, mag, r=r)
    # row sums of the stored fp32 dx (before any bf16 rounding): sum dx over the row
    K = _chain(rows, n)
    _report(case, "bias+gelu row sums", rs.view(rows, 2)[:, 0].double(), dxref.reshape(rows, n).sum(-1), mag.reshape(rows, n).sum(-1), K=K, c=E.C_ACC,
            extra=C_POINTWISE * E.U32)

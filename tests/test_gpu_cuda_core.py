"""The CUDA-core kernels outside the tensor-core engine through the C ABI, against fp64 references of their exact operands
(tests/engine_ref.py): the per-mode channel mixes (csrc/mix.cu, every precision), ComplexReLU (csrc/act.cu) and the pointwise kernels
of the SFNO block (csrc/norm.cu: instance norm (+ GELU), bias + GELU).

Same conventions as tests/test_gpu_engine.py: inputs the kernels must not read hold NaN, outputs start as a NaN sentinel, stored entries
must lie in a per-element bound in units of 2^-24 times the magnitudes of their terms, padding holds exact zeros, everything else stays
untouched.  Every check prints its worst bound ratio and the smallest constant it would pass with (run with -s)."""
import math

import pytest
import torch

import engine_ref as E
from makani_b200 import _lib
from makani_b200.sht import _ptr, _stream
from test_gpu_engine import DEV, FP32, TF32, call, check, check_spec, sentinel, untouched

pytestmark = pytest.mark.gpu


def _spec_input(L, M, B, C, dense, gen):
    cp = (C + 3) // 4 * 4
    s = torch.randn(L, M, 2, B, cp, device=DEV, generator=gen)
    s[..., C:] = 0
    s[E.zero_mask(L, M, 0, dense, device=DEV)] = 0
    s[~E.stored_mask(L, M, 0, dense, device=DEV)] = float("nan")
    return s


# ---------------------------------------------------------------------------------------------- per-mode channel mixes
PERMODE_CODES = {"diagonal": _lib.OP_DIAGONAL, "sep_diagonal": _lib.OP_SEP_DIAGONAL, "sep_dhconv": _lib.OP_SEP_DHCONV}
# id, L, M, B, G, Ci, Co, dense   (separable operators: only the rows with Ci == Co)
PERMODE_CASES = [
    ("G1-B1-C5", 33, 33, 1, 1, 5, 5, False),
    ("G2-B3-Ci6-Co10", 40, 41, 3, 2, 6, 10, False),
    ("G2-B3-C6", 40, 41, 3, 2, 6, 6, False),
    ("G1-B8-Ci8-Co7-dense", 33, 33, 8, 1, 8, 7, True),
    ("G1-B8-C7-dense", 33, 33, 8, 1, 7, 7, True),
    ("headline-240x241-C16", 240, 241, 1, 1, 16, 16, False),
]
PERMODE_PARAMS = [pytest.param(*c, op, prec, id=f"{c[0]}-{op}-{pn}") for c in PERMODE_CASES for op in PERMODE_CODES
                  for prec, pn in ((FP32, "fp32"), (TF32, "tf32")) if op == "diagonal" or c[5] == c[6]]


@pytest.mark.parametrize("case,L,M,B,G,Ci,Co,dense,op,prec", PERMODE_PARAMS)
def test_permode_mix(case, L, M, B, G, Ci, Co, dense, op, prec):
    """forward, dgrad and wgrad of OP_DIAGONAL / OP_SEP_DIAGONAL / OP_SEP_DHCONV: every precision runs the same fp32 kernels on the native
    weight, so fp32 operands and K 2^-24 sum |a||b| (C_FMA) with no output rounding; the channel padding of y and gx must be exact zeros"""
    code = PERMODE_CODES[op] | (_lib.DENSE_FLAG if dense else 0)
    st = _stream(DEV)
    gen = torch.Generator(device=DEV).manual_seed(2468)
    Cig, Cog = Ci // G, Co // G
    cpi, cpo = (Ci + 3) // 4 * 4, (Co + 3) // 4 * 4
    shape = {"diagonal": (G, Cig, Cog, L, M), "sep_diagonal": (G, Cig, L, M), "sep_dhconv": (G, Cig, L)}[op]
    w = torch.randn(*shape, dtype=torch.complex64, device=DEV, generator=gen)
    x = _spec_input(L, M, B, Ci, dense, gen)
    gy = _spec_input(L, M, B, Co, dense, gen)
    tag = case

    y = sentinel(L * M * 2 * B * cpo)
    call("b200sht_mix_forward", L, M, code, _ptr(x), _ptr(w), None, _ptr(y), B, G, Ci, Co, prec, st)
    ref, mag, K = E.permode_forward_ref(op, x, w, G, Ci, Co, dense)
    check_spec(tag, "forward", y.view(L, M, 2, B, cpo), ref, mag, K, Co, dense=dense, c=E.C_FMA)

    gx = sentinel(L * M * 2 * B * cpi)
    gw = torch.view_as_complex(sentinel(2 * w.numel()).view(*shape, 2))
    call("b200sht_mix_backward", L, M, code, _ptr(x), _ptr(w), _ptr(gy), _ptr(gx), _ptr(gw), None, B, G, Ci, Co, prec, st)
    ref, mag, K = E.permode_dgrad_ref(op, gy, w, G, Ci, Co, dense)
    check_spec(tag, "dgrad", gx.view(L, M, 2, B, cpi), ref, mag, K, Ci, dense=dense, c=E.C_FMA)
    ref, mag, K = E.permode_wgrad_ref(op, x, gy, G, Ci, Co, dense)
    check(tag, "wgrad", gw, ref, mag, K, c=E.C_FMA)   # unstored (l, m): reference and bound 0 -> exact zeros


# --------------------------------------------------------------------------------------------------------- ComplexReLU
RELU_CODES = {"real": 0, "cartesian": 1, "modulus": 2, "halfplane": 3}
# modulus: y = (|z| + b) z / |z| and its gradient through sqrtf, one division and |z| + b, whose rounding is relative to |z| + |b|:
# |got - ref| <= c 2^-24 (1 + |b| / |z|) |x| (forward) and (|gr| + |gi|) (1 + |b| / |z|) (gradient).  Calibrated on an H100 (DESIGN.md section 5).
C_RELU_MOD = 8.0
# id, L, M, B, C, dense
RELU_CASES = [("B2-C5-cppad", 33, 33, 2, 5, False), ("B3-C8-dense", 17, 17, 3, 8, True), ("attention-240x241-B1-C16", 240, 241, 1, 16, False)]


def _relu_input(L, M, B, C, dense, gen):
    """standard-normal spec with the branch points of every mode: z = 0, points on both axes, and signed zeros"""
    x = _spec_input(L, M, B, C, dense, gen)
    st = E.stored_mask(L, M, 0, dense, device=DEV)[:, :, None, None].expand(L, M, B, C)
    u = torch.rand(L, M, B, C, device=DEV, generator=gen)
    re, im = x[:, :, 0, :, :C], x[:, :, 1, :, :C]
    pick = lambda lo, hi: st & (u >= lo) & (u < hi)
    re[pick(0.00, 0.04)] = 0.0; im[pick(0.00, 0.04)] = 0.0              # z = 0
    re[pick(0.04, 0.08)] = 0.0                                          # imaginary axis: angle +-pi/2
    im[pick(0.08, 0.12)] = 0.0                                          # real axis: angle 0 or pi
    re[pick(0.12, 0.14)] = -0.0; im[pick(0.12, 0.14)] = 0.0             # -0 + 0i: angle pi
    re[pick(0.14, 0.16)] = 0.0; im[pick(0.14, 0.16)] = -0.0             # 0 - 0i
    re[pick(0.16, 0.18)] = -0.0                                         # -0 on the imaginary axis
    im[pick(0.18, 0.20)] = -0.0                                         # -0 on the real axis: angle -0 or -pi
    return x


def _relu_bias(kind, C, gen):
    if kind == "none":
        return None
    if kind == "scalar":
        return torch.tensor([0.25], device=DEV)
    return torch.randn(C, device=DEV, generator=gen) * 0.75     # |z| + b on both sides of 0


def _exact_check(tag, what, got, ref, mask):
    """real / cartesian / halfplane: ref is x, gy, or slope times one of them: one rounding of slope * x at most"""
    err = (got - ref).abs()
    ratio = float((err / (E.U32 * ref.abs())).nan_to_num(0.0, posinf=math.inf)[mask].max()) if mask.any() else 0.0
    print(f"[relu] {tag} {what}: worst error {ratio:.3e} x 2^-24 |ref| (bound 1)")
    assert torch.isfinite(got[mask]).all() and ratio <= 1.0, f"{tag} {what}: error {ratio:.3g} x 2^-24 |ref|"


@pytest.mark.parametrize("bias_kind", ["channel", "scalar", "none"])
@pytest.mark.parametrize("mode", E.RELU_MODES)
@pytest.mark.parametrize("case,L,M,B,C,dense", RELU_CASES, ids=[c[0] for c in RELU_CASES])
def test_complex_relu(case, L, M, B, C, dense, mode, bias_kind):
    """forward and backward of every mode through the module's autograd function (a scalar bias is expanded to [C] and its gradient is the
    sum of the per-channel ones), against autograd of oracle.complex_relu in complex128 on the exact fp32 inputs"""
    from makani_b200.spectral_convolution import _ComplexReLUPacked

    gen = torch.Generator(device=DEV).manual_seed(97531)
    slope = float(torch.tensor(0.1, dtype=torch.float32))   # the fp32 slope the kernel multiplies by
    cp = (C + 3) // 4 * 4
    x = _relu_input(L, M, B, C, dense, gen)
    gy = _spec_input(L, M, B, C, dense, gen)
    bias = _relu_bias(bias_kind, C, gen)
    tag = f"{case} {mode} bias={bias_kind}"
    code = RELU_CODES[mode] | (_lib.DENSE_FLAG if dense else 0)
    st_mask = E.stored_mask(L, M, 0, dense, device=DEV)

    xin = x.clone().requires_grad_(True)
    b = bias.clone().requires_grad_(True) if bias is not None else None
    y = _ComplexReLUPacked.apply(xin, b, code, slope, L, M, B, C)
    y.backward(gy)
    yref, gref, gbref = E.complex_relu_ref(mode, x, bias, slope, gy, C, dense)
    yv, gv = y.detach().view(L, M, 2, B, cp), xin.grad.view(L, M, 2, B, cp)
    for what, got in (("forward", yv), ("backward", gv)):
        assert (got[st_mask][..., C:] == 0).all(), f"{tag} {what}: channel padding must hold exact zeros"
    got_y, got_g = E.spec_to_complex(yv, C, dense), E.spec_to_complex(gv, C, dense)
    z = E.spec_to_complex(x, C, dense)
    keep = st_mask[:, :, None, None].expand(L, M, B, C)
    if mode != "modulus":
        if mode == "halfplane":   # off the axes, angle - b within fp32 reach of a branch boundary: either side is right
            ang = torch.angle(z) - ((bias.double().reshape(-1) if bias.numel() > 1 else bias.double()) if bias is not None else 0.0)
            near = (ang.abs() < 1e-5) | ((ang - math.pi / 2).abs() < 1e-5)
            keep = keep & ~(near & (z.real != 0) & (z.imag != 0))
        for what, got, ref in (("forward", got_y, yref), ("backward", got_g, gref)):
            _exact_check(tag, what + " re", got.real, ref.real, keep)
            _exact_check(tag, what + " im", got.imag, ref.imag, keep)
        if bias is not None:
            assert (b.grad == 0).all(), f"{tag}: only the modulus mode has a bias gradient"
        return
    bc = (bias.double().reshape(-1) if bias.numel() > 1 else bias.double()) if bias is not None else torch.zeros((), dtype=torch.float64, device=DEV)
    za = z.abs()
    keep = keep & ((za + bc).abs() > 1e-5 * (za + bc.abs()))   # |z| + b within fp32 reach of 0: the gradient jumps there
    amp = torch.where(za > 0, 1.0 + bc.abs() / za, torch.zeros((), dtype=torch.float64, device=DEV))
    magy = amp * (z.real.abs() + z.imag.abs())
    magg = amp * (E.spec_to_complex(gy, C, dense).real.abs() + E.spec_to_complex(gy, C, dense).imag.abs())
    for what, got, ref, mag in (("forward", got_y, yref, magy), ("backward", got_g, gref, magg)):
        ratio = E.bound_ratio(got[keep], ref[keep], mag[keep], 1, c=C_RELU_MOD)
        need = E.needed_c(got[keep], ref[keep], mag[keep], 1)
        print(f"[relu] {tag} {what}: worst ratio {ratio:.3e}, needs c >= {need:.3e} (c = {C_RELU_MOD})")
        assert ratio <= 1.0, f"{tag} {what}: exceeds the bound by {ratio:.3g}x"
    if bias is not None:
        # one term (gr xr + gi xi) / |z| per stored (l, m, b) with |z| > 0 and |z| + b > 0: n 2^-24 sum |term| (n terms per channel)
        g = E.spec_to_complex(gy, C, dense)
        act = (za > 0) & (za + bc > 0)
        term = torch.where(act, (g.real * z.real).abs() + (g.imag * z.imag).abs(), torch.zeros((), dtype=torch.float64, device=DEV)) / za.clamp_min(1e-300)
        n = float(st_mask.sum().item() * B)
        mag = term.sum((0, 1, 2))
        if bias.numel() == 1:
            mag = mag.sum().reshape(1)
            n *= C
        ratio = E.bound_ratio(b.grad, gbref, mag, n, c=1.0)
        need = E.needed_c(b.grad, gbref, mag, n)
        print(f"[relu] {tag} bias-grad: worst ratio {ratio:.3e}, needs c >= {need:.3e} (c = 1, K = {n:.0f})")
        assert ratio <= 1.0, f"{tag} bias-grad: exceeds n 2^-24 sum |term| by {ratio:.3g}x"


def test_complex_relu_bias_grad_is_bit_identical_run_to_run():
    """the modulus bias gradient is a fixed-order reduction: the same bits on every call"""
    L, M, B, C = 240, 241, 4, 8
    gen = torch.Generator(device=DEV).manual_seed(11)
    x = _relu_input(L, M, B, C, False, gen)
    gy = _spec_input(L, M, B, C, False, gen)
    bias = torch.randn(C, device=DEV, generator=gen) * 0.75
    st = _stream(DEV)
    gx = torch.empty_like(x)
    outs = []
    for _ in range(5):
        gb = sentinel(C)
        call("b200sht_complex_relu_backward", L, M, 2, _ptr(x), _ptr(bias), 0.1, _ptr(gy), _ptr(gx), _ptr(gb), B, C, st)
        outs.append(gb.view(torch.int32).clone())
    assert all(torch.equal(o, outs[0]) for o in outs[1:]), "the bias gradient changed between identical calls"

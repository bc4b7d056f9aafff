"""fp64 references of the tensor-core engine's contractions (csrc/umma.cu) in the library's packed layouts, and the error bound the
engine is held to.  Plain PyTorch: the helpers run on the CPU (tests/test_engine_ref_cpu.py) or on the device in float64
(tests/test_gpu_engine.py).

Packed layouts (include/b200sht.h):
    latspec  [mmax8][2][B][C][kp]      analysis input / synthesis output (plane p, image b * C + c; rows k >= nlat are padding)
    spec     [L][M][2][B][cp]          only l >= lstart(m0 + m) stored; lstart(m0 + m) <= l < m0 + m hold exact zeros
    weight   [Lw][G][Cig][2][cop]      packed dense mix weight (Lw = 1 for OP_SHARED)

Every reference returns (ref, mag): the exact result of the contraction of the operands it is given, and the sum of |a_k| |b_k| over
the same terms.  For complex terms |x| |w| bounds |xr wr| + |xi wi| (and |xr wi| + |xi wr|).  With TF32 operands every product is exact
in fp32, so what the engine may add to the reference is its fp32 accumulation and, where the epilogue rounds, one cvt.rna:

    |got - ref| <= r |ref| + (1 + r) gamma(K) mag + floor,    gamma(K) = c K 2^-24,    r = 2^-11 where the output is rounded to TF32, else 0

(`bound_ratio`).  `C_ACC` is c, calibrated on an H100 (DESIGN.md section 5).  `floor` covers underflow: a term whose operand or product
lies below the smallest normal fp32, 2^-126, may be flushed to zero, so each term may lose up to 2^-126 max(1, |b|) (`underflow_floor`).
The Legendre table reaches such values at high orders near the poles; where it does, the reference and its sum of magnitudes are
themselves of that size.
"""
import torch

TRI = 32                 # kTriBlock of csrc/common.cuh
U32 = 2.0 ** -24         # unit roundoff of fp32
R_TF32 = 2.0 ** -11      # unit roundoff of TF32: bound of one cvt.rna.tf32.f32 of the output
# c of gamma(K) = c K 2^-24, calibrated on an H100 80GB HBM3 at 700 W (DESIGN.md section 5): tests/test_gpu_engine.py prints, per check, the
# smallest c it would pass with.  The largest was 0.26 for the tensor-core engine and 0.25 for the fp32 CUDA-core mix kernels
# (round-to-nearest FMA chains) that serve the shapes the engine cannot address: about 2x headroom.
C_ACC = 0.5
FLT_MIN = 2.0 ** -126
# 3 x TF32 (PREC_FP32X3): per term the omitted lo.lo product (<= 2^-21 |a||b|) and the TF32 rounding of the two residuals
# (<= 2^-21 + 2^-22): 2^-20 |a||b| in all.  Derived, not calibrated.
SPLIT_TERM = 2.0 ** -20
# c for the fp32 CUDA-core kernels whose chains can be as short as one or two products (the SIMT Legendre stages at the last orders, the
# per-mode mixes): the first-order worst case of a K-term fp32 FMA chain, |err| <= K 2^-24 sum |a||b|.  Derived, not calibrated.
C_FMA = 1.0


# ------------------------------------------------------------------------------------------------- TF32 conversions
def tf32_rna(t):
    """cvt.rna.tf32.f32: round to the nearest TF32 value, ties away from zero (finite values; inf and NaN pass through)."""
    t = t.contiguous()
    bits = t.view(torch.int32)
    r = ((bits + 0x1000) & ~0x1FFF).view(torch.float32)
    return torch.where(torch.isfinite(t), r, t)


def tf32_trunc(t):
    """what the TF32 MMA reads from an fp32 register: the 13 low mantissa bits dropped."""
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def rand_tf32(*shape, device="cpu", generator=None):
    """standard-normal values that are TF32-representable (exact operands of the tensor cores)"""
    return tf32_rna(torch.randn(*shape, device=device, generator=generator))


# ----------------------------------------------------------------------------------------------- storage convention
def lstart(m):
    return (m // TRI) * TRI


def stored_mask(L, M, m0=0, dense=False, device="cpu"):
    """bool [L][M]: entries of a packed spec that are stored (l >= 32 floor((m0 + m) / 32)); `dense`: all of them"""
    l = torch.arange(L, device=device)[:, None]
    m = torch.arange(M, device=device)[None, :]
    if dense:
        return torch.ones(L, M, dtype=torch.bool, device=device)
    return l >= lstart(m0 + m)


def zero_mask(L, M, m0=0, dense=False, device="cpu"):
    """bool [L][M]: stored entries that hold exact zeros by convention (lstart(m0 + m) <= l < m0 + m); none when dense"""
    l = torch.arange(L, device=device)[:, None]
    m = torch.arange(M, device=device)[None, :]
    if dense:
        return torch.zeros(L, M, dtype=torch.bool, device=device)
    return stored_mask(L, M, m0, False, device) & (l < m0 + m)


def vector_zero_mask(L, M, m0=0, device="cpu"):
    """bool [2L][M]: stored entries of a stacked vector spec (rows D_l, then Q_l at L + l; include/b200sht.h) that hold exact zeros.  The
    Legendre stages see 2L rows, stored from lstart(m0 + m) (stored_mask(2L, M, m0)), so the whole Q half is stored; D and Q are both
    zero for l < m0 + m, which in the Q half reaches below lstart(m0 + m)."""
    l = torch.arange(2 * L, device=device)[:, None] % L
    m = torch.arange(M, device=device)[None, :]
    return stored_mask(2 * L, M, m0, False, device) & (l < m0 + m)


def to_tiled(Z, M2=None):
    """standard latspec [mmax][2][R][kp] -> the tiled layout [R][kp/8][2][M2][8][8] (orders zero-padded to 8 * M2) that
    b200sht_legendre_synthesis_tiled writes and b200sht_fft_synthesis(scale_mode | 2) reads (include/b200sht.h)"""
    mmax, _, R, kp = Z.shape
    M2 = M2 or (mmax + 7) // 8
    Zp = torch.zeros(8 * M2, 2, R, kp, device=Z.device, dtype=Z.dtype)
    Zp[:mmax] = Z
    # (m2, c, p, r, kt, k8) -> (r, kt, p, m2, c, k8)
    return Zp.view(M2, 8, 2, R, kp // 8, 8).permute(3, 4, 2, 0, 1, 5).contiguous().reshape(-1)


# ------------------------------------------------------------------------------------------------------- Legendre
def legendre_analysis_ref(T, X, nlat, cp, m0=0):
    """spec[l][m][n] = sum_k T[m][l][k] X[m][n][k] over k < nlat.
    T [M][L][>= nlat] (the table as the engine reads it), X [M][2][B][C][>= nlat] (latspec; rows >= nlat are not read).
    Returns (ref, mag) as float64 [L][M][2][B][cp], zero outside the stored region and in the channel padding."""
    M, L = T.shape[:2]
    _, _, B, C, _ = X.shape
    a = T[..., :nlat].double()
    b = X[..., :nlat].double().reshape(M, 2 * B * C, nlat).transpose(1, 2)
    out = []
    for f in (a, a.abs()):
        s = torch.bmm(f, b if f is a else b.abs())                       # [M][L][2 B C]
        s = s.view(M, L, 2, B, C).permute(1, 0, 2, 3, 4)
        full = torch.zeros(L, M, 2, B, cp, dtype=torch.float64, device=T.device)
        full[..., :C] = s
        full[~stored_mask(L, M, m0, device=T.device)] = 0
        out.append(full)
    return out[0], out[1]


def legendre_synthesis_ref(T, spec, C, m0=0):
    """Z[m][n][k] = sum_{l >= lstart(m0 + m)} T[m][l][k] spec[l][m][n].
    T [M][L][kp], spec [L][M][2][B][cp] (unstored entries are ignored, whatever they hold).
    Returns (ref, mag, K): float64 [M][2][B][C][kp] and the reduction length per order, [M][1][1][1][1]."""
    M, L, kp = T.shape
    B = spec.shape[3]
    st = stored_mask(L, M, m0, device=T.device)
    s = torch.where(st[:, :, None, None, None], spec.double(), torch.zeros((), dtype=torch.float64, device=T.device))
    s = s[..., :C].permute(1, 0, 2, 3, 4).reshape(M, L, 2 * B * C)           # [M][L][n]
    a = T.double()
    ref = torch.bmm(s.transpose(1, 2), a).view(M, 2, B, C, kp)
    mag = torch.bmm(s.abs().transpose(1, 2), a.abs()).view(M, 2, B, C, kp)
    K = st.sum(0).to(torch.float64).view(M, 1, 1, 1, 1)
    return ref, mag, K


# ------------------------------------------------------------------------------------------------------------ mix
def spec_to_complex(spec, C, dense=False):
    """packed spec [L][M][2][B][cp] -> complex128 [L][M][B][C], unstored rows (m >= mend(l)) set to zero"""
    L, M = spec.shape[:2]
    z = torch.complex(spec[:, :, 0, :, :C].double(), spec[:, :, 1, :, :C].double())
    keep = stored_mask(L, M, 0, dense, device=spec.device)[:, :, None, None]
    return torch.where(keep, z, torch.zeros((), dtype=z.dtype, device=z.device))


def _planes(z):
    """(real, imaginary) of a complex tensor; a real tensor (a magnitude bound) goes to both planes"""
    return (z.real, z.imag) if torch.is_complex(z) else (z, z)


def complex_to_spec(z, cp):
    """complex [L][M][B][C] -> packed float64 [L][M][2][B][cp] (zero channel padding)"""
    L, M, B, C = z.shape
    out = torch.zeros(L, M, 2, B, cp, dtype=torch.float64, device=z.device)
    out[:, :, 0, :, :C], out[:, :, 1, :, :C] = _planes(z)
    return out


def weight_to_complex(wp, G, Cig, Cog):
    """packed weight [Lw][G][Cig][2][cop] (flat or shaped) -> complex128 [Lw][G][Cig][Cog]"""
    cop = (Cog + 3) // 4 * 4
    w = wp.reshape(-1, G, Cig, 2, cop).double()
    return torch.complex(w[..., 0, :Cog], w[..., 1, :Cog])


def complex_to_weight(w, cop):
    """complex [Lw][G][Cig][Cog] -> packed float64 [Lw][G][Cig][2][cop]"""
    Lw, G, Cig, Cog = w.shape
    out = torch.zeros(Lw, G, Cig, 2, cop, dtype=torch.float64, device=w.device)
    out[..., 0, :Cog], out[..., 1, :Cog] = _planes(w)
    return out


def _pair(eq, a, b):
    """(einsum(eq, a, b), einsum(eq, |a|, |b|)) in complex128 / float64"""
    return torch.einsum(eq, a, b), torch.einsum(eq, a.abs(), b.abs())


def mix_forward_ref(x, w, G, Ci, Co, cbias=None, dense=False):
    """y[l][m][b][g Cog + o] = sum_i x[l][m][b][g Cig + i] w[l][g][i][o] (+ cbias[g Cog + o]) on the stored rows.
    x packed spec [L][M][2][B][cpi], w packed weight [Lw][G][Cig][2][cop], cbias complex [Co] or None.
    Returns (ref, mag, K) with ref / mag packed float64 [L][M][2][B][cpo] (zero in unstored rows and the padding)."""
    L, M, _, B, _ = x.shape
    Cig, Cog = Ci // G, Co // G
    xc = spec_to_complex(x, Ci, dense).view(L, M, B, G, Cig)
    wc = weight_to_complex(w, G, Cig, Cog).expand(L, G, Cig, Cog)
    y, mag = _pair("lmbgi,lgio->lmbgo", xc, wc)
    y, mag = y.reshape(L, M, B, Co), mag.reshape(L, M, B, Co)
    if cbias is not None:
        cb = cbias.to(torch.complex128).reshape(Co)
        y = y + cb
        mag = mag + cb.abs()
    keep = stored_mask(L, M, 0, dense, device=x.device)[:, :, None, None]
    y = torch.where(keep, y, torch.zeros((), dtype=y.dtype, device=y.device))
    mag = torch.where(keep, mag, torch.zeros((), dtype=mag.dtype, device=mag.device))
    cpo = (Co + 3) // 4 * 4
    return complex_to_spec(y, cpo), complex_to_spec(mag, cpo), 2 * Cig


def mix_dgrad_ref(gy, w, G, Ci, Co, dense=False):
    """gx[l][m][b][g Cig + i] = sum_o gy[l][m][b][g Cog + o] conj(w[l][g][i][o]): the PyTorch complex gradient of mix_forward.
    Returns (ref, mag, K) packed float64 [L][M][2][B][cpi]."""
    L, M, _, B, _ = gy.shape
    Cig, Cog = Ci // G, Co // G
    gc = spec_to_complex(gy, Co, dense).view(L, M, B, G, Cog)
    wc = weight_to_complex(w, G, Cig, Cog).expand(L, G, Cig, Cog)
    gx, mag = _pair("lmbgo,lgio->lmbgi", gc, wc.conj())
    cpi = (Ci + 3) // 4 * 4
    return complex_to_spec(gx.reshape(L, M, B, Ci), cpi), complex_to_spec(mag.reshape(L, M, B, Ci), cpi), 2 * Cog


def mix_wgrad_ref(x, gy, G, Ci, Co, shared=False, dense=False):
    """gw[l][g][i][o] = sum over the stored rows (m, b) of conj(x[.][g Cig + i]) gy[.][g Cog + o]; `shared`: also summed over l.
    Returns (ref, mag, K): packed float64 [Lw][G][Cig][2][cop] and the reduction length (rows, x 2 for the complex product) per l,
    [Lw][1][1][1][1]."""
    L, M, _, B, _ = x.shape
    Cig, Cog = Ci // G, Co // G
    xc = spec_to_complex(x, Ci, dense).view(L, M, B, G, Cig)
    gc = spec_to_complex(gy, Co, dense).view(L, M, B, G, Cog)
    eq = "lmbgi,lmbgo->gio" if shared else "lmbgi,lmbgo->lgio"
    gw, mag = _pair(eq, xc.conj(), gc)
    rows = stored_mask(L, M, 0, dense, device=x.device).sum(1).double() * B
    if shared:
        gw, mag, rows = gw[None], mag[None], rows.sum().view(1)
    cop = (Cog + 3) // 4 * 4
    return complex_to_weight(gw, cop), complex_to_weight(mag, cop), 2 * rows.view(-1, 1, 1, 1, 1)


def mix_cbias_grad_ref(gy, Co, dense=False):
    """gcbias[o] = sum over the stored rows (l, m, b) of gy[.][o] (complex128 [Co]); returns (ref, mag, K)"""
    L, M, _, B, _ = gy.shape
    gc = spec_to_complex(gy, Co, dense)
    rows = float(stored_mask(L, M, 0, dense).sum().item() * B)
    return gc.sum((0, 1, 2)), gc.abs().sum((0, 1, 2)), rows


# ---------------------------------------------------------------------------------------------------------- bound
def underflow_floor(K, b):
    """what flushing terms below 2^-126 to zero can cost a K-term sum whose second operands are `b`"""
    return K * FLT_MIN * max(1.0, float(b[torch.isfinite(b)].abs().max().item()))


def bound_ratio(got, ref, mag, K, r=0.0, c=C_ACC, extra=0.0, floor=0.0):
    """worst |got - ref| / (r |ref| + (1 + r) (c K 2^-24 + extra) mag + floor) over the elements (<= 1: inside the bound).
    An element whose bound is 0 (exact zeros expected) and that is not exactly equal gives inf; so does a non-finite got.
    Complex tensors are compared by real and imaginary part, each against the bound of its magnitudes."""
    if torch.is_complex(got) or torch.is_complex(ref):
        got, ref = torch.view_as_real(got.to(torch.complex128)), torch.view_as_real(ref.to(torch.complex128))
        mag = mag.double()[..., None]
    got = got.double()
    if not torch.isfinite(got).all():
        return float("inf")
    err = (got - ref).abs()
    tol = r * ref.abs() + (1.0 + r) * (c * K * U32 + extra) * mag + floor
    ratio = torch.where(err == 0, torch.zeros_like(err), err / tol)
    return float(ratio.max().item()) if ratio.numel() else 0.0


def needed_c(got, ref, mag, K, r=0.0, extra=0.0, floor=0.0):
    """the smallest c for which bound_ratio(..., c) <= 1 holds (elements with mag = 0 aside): the calibration statistic"""
    if torch.is_complex(got) or torch.is_complex(ref):
        got, ref = torch.view_as_real(got.to(torch.complex128)), torch.view_as_real(ref.to(torch.complex128))
        mag = mag.double()[..., None]
    err = (got.double() - ref).abs() - r * ref.abs() - (1.0 + r) * extra * mag - floor
    den = (1.0 + r) * K * U32 * mag
    c = torch.where(den > 0, err.clamp_min(0) / den, torch.zeros_like(err))
    return float(c.max().item()) if c.numel() else 0.0


# --------------------------------------------------------------------------------------------- per-mode channel mixes
# Native complex weights of the per-mode operators (csrc/mix.cu, mix_permode_kernel):
#   OP_DIAGONAL [G][Cig][Cog][L][M],   OP_SEP_DIAGONAL [G][Cig][L][M],   OP_SEP_DHCONV [G][Cig][L]   (separable: Ci == Co)
# K counts real products per output element, as the mix references above: 2 per complex product.
PERMODE_OPS = ("diagonal", "sep_diagonal", "sep_dhconv")


def _permode_apply(op, z, w, G, Cig, Cog, conj_w, dgrad):
    """sum over the input channel of z * w (or conj(w)) per (l, m), for z complex [L][M][B][Cin] and the native weight"""
    L, M, B, _ = z.shape
    wc = w.to(torch.complex128)
    if conj_w:
        wc = wc.conj()
    if op == "diagonal":
        zg = z.view(L, M, B, G, Cog if dgrad else Cig)
        eq = "lmbgo,giolm->lmbgi" if dgrad else "lmbgi,giolm->lmbgo"
        out, mag = _pair(eq, zg, wc)
        return out.reshape(L, M, B, -1), mag.reshape(L, M, B, -1), 2 * (Cog if dgrad else Cig)
    wf = wc.reshape(G * Cig, L, -1).permute(1, 2, 0)[:, :, None, :]      # [L][M or 1][1][C]
    return z * wf, z.abs() * wf.abs(), 2


def permode_forward_ref(op, x, w, G, Ci, Co, dense=False):
    """y[l][m][b][g Cog + o] = sum_i x[l][m][b][g Cig + i] w(g, i, o, l, m) on the stored rows.  x packed spec [L][M][2][B][cpi], w native.
    Returns (ref, mag, K): packed float64 [L][M][2][B][cpo] (zero in unstored rows and the padding)."""
    L, M = x.shape[:2]
    y, mag, K = _permode_apply(op, spec_to_complex(x, Ci, dense), w, G, Ci // G, Co // G, False, False)
    cpo = (Co + 3) // 4 * 4
    return complex_to_spec(y, cpo), complex_to_spec(mag, cpo), K


def permode_dgrad_ref(op, gy, w, G, Ci, Co, dense=False):
    """gx[l][m][b][g Cig + i] = sum_o gy[l][m][b][g Cog + o] conj(w(g, i, o, l, m)): the PyTorch complex gradient of permode_forward.
    Returns (ref, mag, K) packed float64 [L][M][2][B][cpi]."""
    gx, mag, K = _permode_apply(op, spec_to_complex(gy, Co, dense), w, G, Ci // G, Co // G, True, True)
    cpi = (Ci + 3) // 4 * 4
    return complex_to_spec(gx, cpi), complex_to_spec(mag, cpi), K


def permode_wgrad_ref(op, x, gy, G, Ci, Co, dense=False):
    """gw(g, i, o, l, m) = sum over b of conj(x[l][m][b][g Cig + i]) gy[l][m][b][g Cog + o] on the stored rows (OP_SEP_DHCONV: also
    summed over the stored m of l).  Returns (ref, mag, K): complex128 / float64 in the native layout and K (OP_SEP_DHCONV: [L][1])."""
    L, M, _, B, _ = x.shape
    Cig, Cog = Ci // G, Co // G
    xc = spec_to_complex(x, Ci, dense).conj()
    gc = spec_to_complex(gy, Co, dense)
    if op == "diagonal":
        gw, mag = _pair("lmbgi,lmbgo->giolm", xc.view(L, M, B, G, Cig), gc.view(L, M, B, G, Cog))
        return gw, mag, 2.0 * B
    if op == "sep_diagonal":
        gw, mag = _pair("lmbc,lmbc->clm", xc, gc)
        return gw.reshape(G, Cig, L, M), mag.reshape(G, Cig, L, M), 2.0 * B
    gw, mag = _pair("lmbc,lmbc->cl", xc, gc)
    rows = stored_mask(L, M, 0, dense, device=x.device).sum(1).double() * B
    return gw.reshape(G, Cig, L), mag.reshape(G, Cig, L), 2 * rows.view(L, 1)


# -------------------------------------------------------------------------------------------------------- ComplexReLU
RELU_MODES = ("real", "cartesian", "modulus", "halfplane")


def complex_relu_ref(mode, x, bias, slope, gy, C, dense=False):
    """ComplexReLU (oracle.complex_relu) of a packed spec x [L][M][2][B][cp] and its PyTorch complex gradient for the output gradient gy, by
    autograd in complex128 on the exact fp32 inputs.  bias: float [C], a 1-element tensor (one bias for every channel) or None (0).
    Modulus at z = 0 gives y = 0 and no gradient (the oracle's (|z| + b) z / |z| is 0 / 0 there).
    Returns complex128 [L][M][B][C] y, gx and the bias gradient (shape of `bias`; None without one)."""
    from oracle import makani_oracle as O

    z = spec_to_complex(x, C, dense).requires_grad_(True)
    g = spec_to_complex(gy, C, dense)
    b = bias.double().requires_grad_(True) if bias is not None else None
    bb = (b.reshape(-1) if b.numel() > 1 else b.reshape(())) if b is not None else 0.0
    zero = (z.detach() == 0) if mode == "modulus" else torch.zeros(z.shape, dtype=torch.bool, device=z.device)
    zs = torch.where(zero, torch.ones((), dtype=z.dtype), z)     # keep 0 / 0 out of the graph
    y = torch.where(zero, torch.zeros((), dtype=z.dtype), O.complex_relu(zs, mode, bb, slope))
    inputs = [z] + ([b] if b is not None and mode == "modulus" else [])
    grads = torch.autograd.grad(y, inputs, grad_outputs=g)
    gb = grads[1] if len(grads) > 1 else (torch.zeros_like(b) if b is not None else None)
    return y.detach(), grads[0], gb


# ------------------------------------------------------------------------------------------------------ instance norm
def norm_stats_ref(x):
    """fp64 mean and 1 / sqrt(var + eps) factor pieces of rows x [rows][n] (any float dtype): (mean, var) float64 [rows]"""
    xd = x.double()
    mean = xd.mean(1)
    return mean, ((xd - mean[:, None]) ** 2).mean(1)


def gelu_ref(z):
    return 0.5 * z * (1.0 + torch.erf(z / 2.0 ** 0.5))


def gelu_grad_ref(z):
    return 0.5 * (1.0 + torch.erf(z / 2.0 ** 0.5)) + z * torch.exp(-0.5 * z * z) / (2.0 * torch.pi) ** 0.5

"""fp64 references of the tensor-core longitude DFT (csrc/dft.cu) in its own factorisation (csrc/dft_math.cuh), and the error
bounds the kernels are held to.  Plain PyTorch: CPU (tests/test_dft_ref_cpu.py) or the device in float64 (tests/test_gpu_dft.py).

Factorisation, N = nlon = 8 N2:  longitude j = N2 j1 + j2,  order m = c + 8 m2,
    exp(2 pi i m j / N) = exp(2 pi i c j1 / 8) * tw(c, j2) * E[m2][j2],   tw(c, j2) = exp(2 pi i c j2 / N),  E = exp(2 pi i m2 j2 / N2).
Only the columns j2 <= N2 / 2 of E enter the GEMMs; the partner column N2 - j2 uses conj(E) and the partner twiddle
exp(i pi c / 4) conj(tw(c, j2)).  With `rounded` tables the references use the values the plan stores (dft_tables_kernel):
E = cvt.rna.tf32((float) cos / sin) with the analysis column N2 / 2 halved (that column is its own partner and is counted twice),
tw = (float) cos / sin.  Unrounded tables make both references plain rfft / irfft.

Every reference returns (ref, mag) as tests/engine_ref.py does: the result and the sum of the magnitudes of the terms along the
whole chain (butterflies, twiddles, GEMM), which bounds what fp32 arithmetic may add:  c K 2^-24 mag  (engine_ref.bound_ratio).

Synthesis (b200sht_fft_synthesis, scale_mode | 2): with TF32 latspec values every GEMM product is exact, so the kernel may differ
from the rounded-table reference only by fp32 accumulation and butterflies (+ one bf16 rounding of a bf16 output).

Analysis (b200sht_fft_analysis, scale_mode | 2): the producers scale the GEMM operands Ye, Yo by (1 + 2^-10 / 3) and the tensor cores
truncate them to TF32; the epilogue stores trunc_tf32(X sc (1 + 2^-10 / 3)).  A truncation of v (1 + f) errs by v f - delta with
0 <= delta < ulp <= 2^-10 |v (1 + f)|, i.e. by at most (1 + 1/3) 2^-10 |v| per operand (TRUNC_TERM) and by at most
2^-10 (1 + f) - f < R_OUT relative on the stored value; its mean over a binade is ~0, so the gain of the output stays 1.
`analysis_ref` also returns tmag = sum_j2 |E| (|Ye| + |Yo|) scaled as the output, the magnitude the operand truncation acts on.
"""
import math

import torch

import engine_ref as E

TRUNC_COMP = 1.0 + 2.0 ** -10 / 3.0       # kTruncComp of csrc/dft.cu
TRUNC_TERM = (1.0 + 1.0 / 3.0) * 2.0 ** -10   # worst error of one compensated truncation, relative to the operand
R_OUT = 2.0 ** -10 * (1.0 + TRUNC_COMP - 1.0) - (TRUNC_COMP - 1.0)   # worst relative error of the stored compensated truncation
R_BF16 = 2.0 ** -8                        # one round-to-nearest of a bf16 output (8 significant bits)
# c of c K 2^-24 mag with K = M2 + 8 (GEMM length + butterfly depth), calibrated on an H100 80GB HBM3 at a 400 W power limit (DESIGN.md section 5):
# tests/test_gpu_dft.py prints the smallest c each check passes with; the largest was 0.11 (synthesis): about 2x headroom
C_DFT = 0.25


def gemm_len(mmax):
    return (mmax + 7) // 8 + 8


def tables(nlon, mmax, rounded=True):
    """(Ec, Es, Ea_c, Ea_s, tw): E restricted to j2 <= N2 / 2 as float64 [M2][half + 1] (synthesis, then the analysis copy with
    the column N2 / 2 halved) and the twiddles complex128 [8][N2]"""
    N2 = nlon // 8
    half, M2 = N2 // 2, (mmax + 7) // 8
    m2 = torch.arange(M2, dtype=torch.int64)[:, None]
    j2 = torch.arange(half + 1, dtype=torch.int64)[None, :]
    ang = 2.0 * math.pi * ((m2 * j2) % N2).double() / N2
    ec, es = torch.cos(ang), torch.sin(ang)
    c = torch.arange(8, dtype=torch.float64)[:, None]
    ta = 2.0 * math.pi * (c * torch.arange(N2, dtype=torch.float64)[None, :]) / nlon
    twr, twi = torch.cos(ta), torch.sin(ta)
    if rounded:
        ec, es = E.tf32_rna(ec.float()).double(), E.tf32_rna(es.float()).double()
        twr, twi = twr.float().double(), twi.float().double()
    eac, eas = ec.clone(), es.clone()
    if N2 % 2 == 0:
        eac[:, half] *= 0.5
        eas[:, half] *= 0.5
    return ec, es, eac, eas, torch.complex(twr, twi)


def _col_twiddles(tw, N2):
    """twiddle of every column j = 0 .. N2 - 1 as the kernels use it: tw(c, j) for j <= N2 / 2, the partner twiddle
    exp(i pi c / 4) conj(tw(c, N2 - j)) above"""
    half = N2 // 2
    rot = torch.exp(1j * math.pi / 4 * torch.arange(8, dtype=torch.float64))[:, None]
    out = tw.clone()
    j = torch.arange(half + 1, N2)
    out[:, j] = rot * tw[:, N2 - j].conj()
    return out


def _omega(sign):
    """[j1][c] exp(sign 2 pi i c j1 / 8)"""
    k = torch.arange(8, dtype=torch.float64)
    return torch.exp(sign * 2j * math.pi * k[:, None] * k[None, :] / 8)


def _order_scale(mode, nlon, mmax, rowscale, nlat):
    """[nlat][mmax] output factor of the analysis: rowscale[k] (mode 0) or 1 / 2 (mode 1)"""
    if mode == 0:
        return rowscale.double().reshape(nlat, 1).expand(nlat, mmax)
    ms = torch.full((mmax,), 2.0, dtype=torch.float64)
    ms[0] = 1.0
    if mmax - 1 == nlon // 2:
        ms[-1] = 1.0
    return ms.expand(nlat, mmax)


def synthesis_ref(Z, nlon, mode, rowscale=None, bias=None, C=1, rounded=True):
    """y[r][k][j] from the standard latspec Z [mmax][2][R][K rows]: mode 0  2 Re sum_m Z_m e^{i m phi_j} - Re Z_0 - Re Z_nyq (-1)^j
    (= irfft(norm="forward")), mode 1  rowscale[k] Re sum_m Z_m e^{i m phi_j}; both + bias[r % C].
    Returns (ref, mag) float64 [R][K][nlon]."""
    mmax, _, R, K = Z.shape
    N2, M2 = nlon // 8, (mmax + 7) // 8
    half = N2 // 2
    ec, es, _, _, tw = tables(nlon, mmax, rounded)
    zp = torch.zeros(8 * M2, 2, R, K, dtype=torch.float64)
    zp[:mmax] = Z.double().cpu()
    zr = zp[:, 0].view(M2, 8, R, K).permute(2, 3, 1, 0)   # [R][K][c][m2]
    zi = zp[:, 1].view(M2, 8, R, K).permute(2, 3, 1, 0)
    s1, s2, s3, s4 = zr @ ec, zi @ es, zr @ es, zi @ ec      # [R][K][8][half + 1]
    a1, a2, a3, a4 = zr.abs() @ ec.abs(), zi.abs() @ es.abs(), zr.abs() @ es.abs(), zi.abs() @ ec.abs()
    V = torch.zeros(R, K, 8, N2, dtype=torch.complex128)
    Vm = torch.zeros(R, K, 8, N2, dtype=torch.float64)       # |Vr| + |Vi| magnitude
    V[..., : half + 1] = torch.complex(s1 - s2, s3 + s4)
    Vm[..., : half + 1] = a1 + a2 + a3 + a4
    jp = torch.arange(half + 1, N2)
    V[..., jp] = torch.complex(s1 + s2, s4 - s3)[..., N2 - jp]
    Vm[..., jp] = (a1 + a2 + a3 + a4)[..., N2 - jp]
    U = V * _col_twiddles(tw, N2)                            # class 0: twiddle 1
    Um = Vm * 2.0
    x = torch.einsum("rkcj,ac->rkaj", U, _omega(1.0)).real   # [R][K][j1][j2]
    xm = Um.sum(2, keepdim=True).expand(R, K, 8, N2)
    x, xm = x.reshape(R, K, nlon), xm.reshape(R, K, nlon)
    b = bias.double().cpu().repeat(R // C)[:, None, None] if bias is not None else torch.zeros((), dtype=torch.float64)
    if mode == 0:
        alt = torch.where(torch.arange(nlon) % 2 == 0, 1.0, -1.0).double()
        z0 = zp[0, 0][:, :, None]
        zn = zp[nlon // 2, 0][:, :, None] * alt if mmax == nlon // 2 + 1 else torch.zeros((), dtype=torch.float64)
        ref = 2.0 * x - z0 - zn + b
        mag = 2.0 * xm + z0.abs() + zn.abs() + b.abs()
    else:
        rs = rowscale.double().cpu()[None, :K, None]
        ref, mag = rs * x + b, rs.abs() * xm + b.abs()
    return ref, mag


def analysis_ref(x, mmax, mode, rowscale=None, rounded=True):
    """X[r][k][m] from rows x [R][nlat][nlon] (the values the kernel reads): mode 0  rowscale[k] sum_j x_j e^{-i m phi_j},
    mode 1  (1 or 2) sum_j x_j e^{-i m phi_j} (= 2 pi rfft(norm="forward") up to the caller's row scale).
    Returns (ref complex128 [R][nlat][mmax], mag, tmag float64 [R][nlat][mmax])."""
    R, nlat, nlon = x.shape
    N2, M2 = nlon // 8, (mmax + 7) // 8
    half = N2 // 2
    _, _, ec, es, tw = tables(nlon, mmax, rounded)
    xd = x.double().cpu().view(R, nlat, 8, N2)               # [r][k][j1][j2]
    Y = torch.einsum("rkaj,ac->rkcj", xd.to(torch.complex128), _omega(-1.0)) * _col_twiddles(tw, N2).conj()
    Ym = xd.abs().sum(2, keepdim=True).expand(R, nlat, 8, N2) * 4.0   # |Re| + |Im| after the radix-8 stage and the twiddle
    j = torch.arange(half + 1)
    P = torch.zeros(R, nlat, 8, half + 1, dtype=torch.complex128)   # partner column N2 - j2; column N2 / 2 is its own partner
    Pm = torch.zeros(R, nlat, 8, half + 1, dtype=torch.float64)
    P[..., 1:] = Y[..., N2 - j[1:]]
    Pm[..., 1:] = Ym[..., N2 - j[1:]]
    if N2 % 2 == 0:   # the kernel reads column N2 / 2 again and turns it with the partner twiddle
        rot = torch.exp(1j * math.pi / 4 * torch.arange(8, dtype=torch.float64))[:, None]
        yh = torch.einsum("rka,ac->rkc", xd[..., half].to(torch.complex128), _omega(-1.0))
        P[..., half] = yh * (rot[:, 0] * tw[:, half].conj()).conj()
    A = Y[..., : half + 1]
    Ye, Yo = A + P, A - P
    Yem = Ym[..., : half + 1] + Pm
    Xre = Ye.real @ ec.T + Yo.imag @ es.T                     # [r][k][c][m2]
    Xim = Ye.imag @ ec.T - Yo.real @ es.T
    mag = Yem @ (ec.abs() + es.abs()).T
    tmag = (Ye.real.abs() + Ye.imag.abs()) @ ec.abs().T + (Yo.real.abs() + Yo.imag.abs()) @ es.abs().T
    to_m = lambda t: t.permute(0, 1, 3, 2).reshape(R, nlat, 8 * M2)[..., :mmax]
    sc = _order_scale(mode, nlon, mmax, rowscale, nlat)[None]
    return torch.complex(to_m(Xre), to_m(Xim)) * sc, to_m(mag) * sc.abs(), to_m(tmag) * sc.abs()


def analysis_floor(ref, tmag):
    """the operand-truncation term of the analysis bound, per real / imaginary part ([..., 2] as bound_ratio views a complex ref)"""
    return (1.0 + R_OUT) * TRUNC_TERM * tmag.double()[..., None]


def simulate_analysis(x, mmax, mode, rowscale=None):
    """what the analysis kernel computes, up to fp32 accumulation: the fp64 factorisation with the rounded tables, the GEMM operands
    scaled by (1 + 2^-10 / 3) and truncated to TF32, the output scaled by (1 + 2^-10 / 3) and truncated (the stored TF32 value)"""
    R, nlat, nlon = x.shape
    N2, M2 = nlon // 8, (mmax + 7) // 8
    half = N2 // 2
    _, _, ec, es, tw = tables(nlon, mmax, True)
    xd = x.double().cpu().view(R, nlat, 8, N2)
    Y = torch.einsum("rkaj,ac->rkcj", xd.to(torch.complex128), _omega(-1.0)) * _col_twiddles(tw, N2).conj()
    j = torch.arange(half + 1)
    P = torch.zeros(R, nlat, 8, half + 1, dtype=torch.complex128)
    P[..., 1:] = Y[..., N2 - j[1:]]
    if N2 % 2 == 0:
        rot = torch.exp(1j * math.pi / 4 * torch.arange(8, dtype=torch.float64))[:, None]
        yh = torch.einsum("rka,ac->rkc", xd[..., half].to(torch.complex128), _omega(-1.0))
        P[..., half] = yh * (rot[:, 0] * tw[:, half].conj()).conj()
    A = Y[..., : half + 1]
    op = lambda t: E.tf32_trunc((t * TRUNC_COMP).float()).double()
    Ye, Yo = A + P, A - P
    yer, yei, yor, yoi = op(Ye.real), op(Ye.imag), op(Yo.real), op(Yo.imag)
    Xre = yer @ ec.T + yoi @ es.T
    Xim = yei @ ec.T - yor @ es.T
    to_m = lambda t: t.permute(0, 1, 3, 2).reshape(R, nlat, 8 * M2)[..., :mmax]
    sc = _order_scale(mode, nlon, mmax, rowscale, nlat)[None]
    out = lambda t: E.tf32_trunc((t * sc * TRUNC_COMP).float()).double()
    return torch.complex(out(to_m(Xre)), out(to_m(Xim)))


def gain(got, ref):
    """least-squares slope of got against ref (real and imaginary parts together)"""
    g, r = torch.view_as_real(got.to(torch.complex128)) if torch.is_complex(got) else got.double(), \
        torch.view_as_real(ref.to(torch.complex128)) if torch.is_complex(ref) else ref.double()
    return float((g * r).sum() / (r * r).sum())


def rel_l2(got, ref):
    d = (got.to(ref.dtype) - ref).abs().pow(2).sum().sqrt()
    return float(d / ref.abs().pow(2).sum().sqrt().clamp_min(1e-300))

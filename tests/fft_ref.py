"""fp64 references of the CUDA-core longitude FFT (csrc/fft.cu) and the bound it is held to.  Plain PyTorch: CPU
(tests/test_fft_ref_cpu.py) or the device in float64 (tests/test_gpu_fft.py).

Operations (include/b200sht.h, b200sht_fft_analysis / _synthesis without the TF32 bit):
    analysis   X[k][m] = s(k, m) rfft(x[k])[m],  m < mmax;  s = rs[k] (mode 0, the plan's fp32 row scale) or 1 at m = 0 and Nyquist, 2
               otherwise (mode 1)
    synthesis  y[k] = irfft(Z[k], norm="forward") + bias (mode 0);  rs[k] irfft(Z'[k], norm="forward") (mode 1, Z' = Z with the orders
               0 < m < N/2 halved), + bias.  The imaginary parts of the DC and Nyquist orders are not read.

Every reference returns (ref, mag): the exact result of the operands it is given and, per output element, the sum of |term| along the
transform scaled as the output: sum_j |x_j| for the analysis, sum_m f_m (|Re Z_m| + |Im Z_m|) (+ |bias|) for the synthesis, f_m the
weight of order m in the real sum.  Each real and imaginary part is held to

    |got - ref| <= r |ref| + (1 + r) c K 2^-24 mag      (engine_ref.bound_ratio),   K = stages of the plan + 3 (split, scale, bias)

with r = 2^-11 for an analysis output rounded to TF32, 2^-8 for a bf16 synthesis output, 0 otherwise, and c = C_FFT.

`paired` selects which terms the magnitude sums.  The compile-time kernels transform each real row as its own half-length complex FFT
(rows never mix): `paired=False`, the element's own row.  The run-time kernels pack rows 2i and 2i + 1 into one complex sequence
z = a + i b, so the rounding error of one row lands in its partner's spectrum: `paired=True`, the magnitude of the row pair.  That is a
property of the two-for-one algorithm, not slack: a row of scale 2^-20 paired with a row of scale 1 comes out about 10 % off relative to
its own size (tests/test_fft_ref_cpu.py shows it on the kernels' own host arithmetic).
"""
import math

import numpy as np
import torch

R_TF32 = 2.0 ** -11      # one cvt.rna.tf32.f32 of the analysis output (scale_mode | 2)
R_BF16 = 2.0 ** -8       # one round-to-nearest of a bf16 synthesis output
# c of c K 2^-24 mag, calibrated on an H100 80GB HBM3 at a 700 W power limit (DESIGN.md section 5): tests/test_gpu_fft.py prints the
# smallest c each check passes with; the largest was 0.70 (run-time analysis, nlon 15 at B*C = 65535): 2x headroom
C_FFT = 1.4


def row_scale(w, nlon, kp=None):
    """the plan's fp32 row scale, as b200sht_plan_create_ex computes it: float(quad_w[k] 2.0 pi / nlon), zero in the padding up to kp"""
    w = torch.tensor(np.array(w, dtype=np.float64))
    rs = (w * 2.0 * math.pi / nlon).float()
    if kp is not None and kp > rs.numel():
        rs = torch.cat([rs, torch.zeros(kp - rs.numel())])
    return rs


def mode_scale(nlon, mmax):
    """float64 [mmax]: the mode-1 analysis factor, 1 at m = 0 and at Nyquist (2 m == nlon), 2 otherwise"""
    m = torch.arange(mmax)
    return torch.where((m == 0) | (2 * m == nlon), 1.0, 2.0).double()


def fft_len(nstages):
    """K of the bound for a plan of `nstages` stages (b200sht_debug_fft_plan)"""
    return nstages + 3


def pair_sum(a):
    """a [..., K, n] -> the sum of rows 2i and 2i + 1 along dim -2, at both rows (an odd last row pairs with a zero row)"""
    K = a.shape[-2]
    if K % 2:
        a = torch.cat([a, torch.zeros_like(a[..., :1, :])], -2)
    s = a.unflatten(-2, (-1, 2)).sum(-2, keepdim=True)
    return s.expand(*s.shape[:-2], 2, s.shape[-1]).flatten(-3, -2)[..., :K, :]


def analysis_ref(x, mmax, mode, rs=None, paired=False):
    """x [R][nlat][nlon] (the values the kernel reads) -> (ref complex128 [R][nlat][mmax], mag float64 [R][nlat][mmax]).
    rs: the fp32 row scale (mode 0), at least nlat long."""
    xd = x.double()
    nlat, nlon = xd.shape[-2:]
    ref = torch.fft.rfft(xd, dim=-1)[..., :mmax]
    a = xd.abs().sum(-1, keepdim=True)
    if paired:
        a = pair_sum(a)
    if mode == 0:
        sc = rs[:nlat].to(device=xd.device, dtype=torch.float64)[:, None]
    else:
        sc = mode_scale(nlon, mmax).to(xd.device)
    return ref * sc, (a * sc.abs()).expand(ref.shape)


def synthesis_ref(Z, nlon, mode, rs=None, bias=None, C=1, paired=False):
    """Z [mmax][2][R][nlat] (the orders and rows the kernel reads) -> (ref, mag) float64 [R][nlat][nlon].
    rs: the fp32 row scale (mode 1); bias: [C] per channel (image r has channel r % C) or None."""
    mmax, _, R, nlat = Z.shape
    dev = Z.device
    m = torch.arange(mmax, device=dev)
    selfc = (m == 0) | (2 * m == nlon)
    zr = Z[:, 0].double().permute(1, 2, 0)                               # [R][nlat][mmax]
    zi = torch.where(selfc, 0.0, Z[:, 1].double().permute(1, 2, 0))
    w = torch.where(selfc, 1.0, 0.5).double() if mode == 1 else torch.ones(mmax, dtype=torch.float64, device=dev)
    full = torch.zeros(R, nlat, nlon // 2 + 1, dtype=torch.complex128, device=dev)
    full[..., :mmax] = torch.complex(zr, zi) * w
    ref = torch.fft.irfft(full, n=nlon, dim=-1, norm="forward")
    f = torch.where(selfc, 1.0, 2.0).double() * w
    a = ((zr.abs() + zi.abs()) * f).sum(-1, keepdim=True)
    if paired:
        a = pair_sum(a)
    if mode == 1:
        sc = rs[:nlat].to(device=dev, dtype=torch.float64)[:, None]
        ref, a = ref * sc, a * sc.abs()
    mag = a.expand(R, nlat, nlon)
    if bias is not None:
        b = bias.to(device=dev, dtype=torch.float64).repeat(R // C)[:, None, None]
        ref, mag = ref + b, mag + b.abs()
    return ref, mag

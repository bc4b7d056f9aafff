"""
CPU ORACLE for the vector spherical harmonic transforms  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

torch_harmonics.RealVectorSHT / InverseRealVectorSHT (norm "ortho") restated as the contract written out in include/b200sht.h, next to
the scalar restatement in oracle/makani_oracle.py, whose quadrature and Legendre recurrence it reuses.  pure PyTorch / numpy, fp32 or fp64.
Component 0 of a field is the colatitude (theta) component, 1 the longitude (phi) component; coefficient 0 is the spheroidal S, 1 the
toroidal T.  torch-harmonics' source is not available, so this restatement is pinned by identities that do not depend on it
(tests/test_vector_sht_cpu.py): the tables against scipy's spherical harmonics, the surface-gradient and -r x grad g identities, the round
trip; and the reference's own vector-loss test classes run against it (tests/reference_suites/run_reference_vector_tests.py).

Only `tests/` and `scripts/vsht_bench.py` (an informational GPU baseline) import this module; nothing under `makani_b200/` does.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from oracle.makani_oracle import legpoly, precompute_latitudes


def vector_legpoly(mmax: int, lmax: int, theta: np.ndarray, csphase: bool = True):
    """D[m,l,k] = dP_l^m(cos theta)/dtheta and Q[m,l,k] = m P_l^m(cos theta)/sin theta of the orthonormal table, fp64, each (mmax, lmax, K).

    D from the raising / lowering relation of the Condon-Shortley functions, dP_l^m/dtheta = (sqrt((l-m)(l+m+1)) P_l^(m+1)
    - sqrt((l+m)(l-m+1)) P_l^(m-1)) / 2 with P_l^(-1) = -P_l^1; Q = m P / sin theta, at the poles its limit (non-zero for m = 1 only).
    Without the Condon-Shortley phase both tables of order m are (-1)^m times these."""
    x, s = np.cos(theta), np.sin(theta)
    P = legpoly(mmax + 1, lmax, x, csphase=True)                       # (mmax + 1, lmax, K)
    l = np.arange(lmax, dtype=np.float64)[None, :, None]
    m = np.arange(mmax, dtype=np.float64)[:, None, None]
    Pm1 = np.concatenate([-P[1:2], P[: mmax - 1]], axis=0)
    up = np.sqrt(np.clip((l - m) * (l + m + 1), 0.0, None))
    dn = np.sqrt(np.clip((l + m) * (l - m + 1), 0.0, None))
    D = 0.5 * (up * P[1 : mmax + 1] - dn * Pm1)
    D = np.where(l >= m, D, 0.0)
    Q = np.zeros_like(D)
    pole = np.abs(s) < 1e-12
    Q[:, :, ~pole] = m * P[:mmax][:, :, ~pole] / s[~pole]
    if mmax > 1 and pole.any():
        # m = 1 at x = +-1: P_l^1 / sin theta -> -sqrt((2l+1) l (l+1) / (4 pi)) / 2 * (+-1)^(l+1)
        lv = np.arange(lmax, dtype=np.float64)
        lim = -0.5 * np.sqrt((2 * lv + 1) * lv * (lv + 1) / (4 * math.pi))
        for k in np.nonzero(pole)[0]:
            sgn = np.where(x[k] > 0, 1.0, (-1.0) ** (lv + 1))
            Q[1, :, k] = lim * sgn
    if not csphase:
        D[1::2] *= -1.0
        Q[1::2] *= -1.0
    return np.ascontiguousarray(D), np.ascontiguousarray(Q)


def _l_factor(lmax, dtype):
    l = torch.arange(lmax, dtype=dtype)
    f = torch.zeros(lmax, dtype=dtype)
    f[1:] = 1.0 / (l[1:] * (l[1:] + 1.0))
    return f


class RealVectorSHT(nn.Module):
    def __init__(self, nlat, nlon, lmax=None, mmax=None, grid="equiangular", norm="ortho", csphase=True, dtype=torch.float32):
        super().__init__()
        if norm != "ortho":
            raise NotImplementedError("only norm='ortho' is requested anywhere in makani")
        self.nlat, self.nlon, self.grid, self.norm, self.csphase = nlat, nlon, grid, norm, csphase
        self.lmax = lmax or nlat
        self.mmax = mmax or nlon // 2 + 1
        theta, w = precompute_latitudes(nlat, grid)
        D, Q = vector_legpoly(self.mmax, self.lmax, theta, csphase=csphase)
        self.register_buffer("dweights", torch.from_numpy(D * w[None, None, :]).to(dtype), persistent=False)
        self.register_buffer("qweights", torch.from_numpy(Q * w[None, None, :]).to(dtype), persistent=False)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        assert x.shape[-3] == 2 and x.shape[-2] == self.nlat and x.shape[-1] == self.nlon
        X = 2.0 * math.pi * torch.fft.rfft(x, dim=-1, norm="forward")[..., : self.mmax]
        Dw, Qw = self.dweights.to(X.dtype), self.qweights.to(X.dtype)
        xt, xp = X[..., 0, :, :], X[..., 1, :, :]
        c = lambda a, t: torch.einsum("...km,mlk->...lm", a, t)
        f = _l_factor(self.lmax, self.dweights.dtype).to(device=X.device, dtype=X.dtype)[:, None]
        S = (c(xt, Dw) - 1j * c(xp, Qw)) * f
        T = (-1j * c(xt, Qw) - c(xp, Dw)) * f
        return torch.stack([S, T], dim=-3)


class InverseRealVectorSHT(nn.Module):
    def __init__(self, nlat, nlon, lmax=None, mmax=None, grid="equiangular", norm="ortho", csphase=True, dtype=torch.float32):
        super().__init__()
        if norm != "ortho":
            raise NotImplementedError("only norm='ortho' is requested anywhere in makani")
        self.nlat, self.nlon, self.grid, self.norm, self.csphase = nlat, nlon, grid, norm, csphase
        self.lmax = lmax or nlat
        self.mmax = mmax or nlon // 2 + 1
        theta, _ = precompute_latitudes(nlat, grid)
        D, Q = vector_legpoly(self.mmax, self.lmax, theta, csphase=csphase)
        self.register_buffer("dpct", torch.from_numpy(D).to(dtype), persistent=False)
        self.register_buffer("qpct", torch.from_numpy(Q).to(dtype), persistent=False)

    def forward(self, c: torch.Tensor) -> torch.Tensor:
        assert c.shape[-3] == 2 and c.shape[-2] == self.lmax and c.shape[-1] == self.mmax
        D, Q = self.dpct.to(c.dtype), self.qpct.to(c.dtype)
        s, t = c[..., 0, :, :], c[..., 1, :, :]
        e = lambda a, tab: torch.einsum("...lm,mlk->...km", a, tab)
        out = []
        for Z in (e(s, D) + 1j * e(t, Q), 1j * e(s, Q) - e(t, D)):
            Z = Z.clone()
            Z[..., 0] = Z[..., 0].real
            if self.mmax > self.nlon // 2 and self.nlon % 2 == 0:
                Z[..., self.nlon // 2] = Z[..., self.nlon // 2].real
            out.append(torch.fft.irfft(Z, n=self.nlon, dim=-1, norm="forward"))
        return torch.stack(out, dim=-3)


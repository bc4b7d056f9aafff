"""
CPU ORACLE for the DISCO convolution  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

torch_harmonics.DiscreteContinuousConvS2 (basis_type "morlet") restated in fp64 as the contract written out in include/b200sht.h and DESIGN.md
section 5, written independently of the product builder in makani_b200/disco.py:
  - the geometry goes through Cartesian unit vectors rotated by R_y(-theta_t) (the YZY passive rotation), r = atan2(|v_xy|, v_z),
    bearing = atan2(v_y, v_x), where the product evaluates the spherical-trigonometry closed forms;
  - psi_hat is a dense torch tensor (K, nlat_out, nlat_in, nlon_in) built on the whole grid (no band search);
  - the contraction is roll-and-matmul over the output longitudes, the shape of torch-harmonics' own CPU path; the psi operand may be dense or a
    torch sparse COO tensor (scripts/disco_bench.py runs the sparse form on the GPU as the library baseline).
torch-harmonics' source is not available, so this restatement is pinned by identities that do not depend on it (tests/test_disco_cpu.py):
support against a haversine distance, normalisation sums, longitude equivariance, Funk-Hecke on the isotropic function, the adjoint identity;
and makani's own FCN3 encoder / processor blocks run on it (tests/reference_suites/run_reference_disco.py).

Only `tests/`, `scripts/disco_bench.py` and `__graft_entry__.smoke` import this module; nothing under `makani_b200/` does.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from oracle.makani_oracle import precompute_latitudes

CUTOFF_SLACK = 1e-3
NORM_EPS = 1e-9


def morlet(kernel_shape, rho, phi):
    """(K, ...) values of the morlet functions at normalised radius rho and bearing phi (torch fp64)"""
    n0, n1 = kernel_shape
    x, y = rho * torch.sin(phi), rho * torch.cos(phi)

    def h(j, u):
        f = math.pi * ((j + 1) // 2)
        return torch.sin(f * u) if j % 2 == 1 else torch.cos(f * u)

    win = torch.cos(0.5 * math.pi * rho).square()
    return torch.stack([win * h(k % n1, x) * h(k // n1, y) for k in range(n0 * n1)])


def dense_psi(kernel_shape, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff):
    """psi_hat (K, nlat_out, nlat_in, nlon_in) fp64 torch tensor"""
    if isinstance(kernel_shape, int):
        kernel_shape = (kernel_shape, kernel_shape)
    (hi, wi), (ho, wo) = in_shape, out_shape
    th_i, w_i = (torch.from_numpy(np.asarray(a)) for a in precompute_latitudes(hi, grid_in))
    th_o, _ = (torch.from_numpy(np.asarray(a)) for a in precompute_latitudes(ho, grid_out))
    ph = torch.arange(wi, dtype=torch.float64) * (2 * math.pi / wi)
    # input points as unit vectors (hi, wi, 3), rotated into the frame of each output point (ho, hi, wi, 3)
    v = torch.stack([torch.sin(th_i)[:, None] * torch.cos(ph)[None, :], torch.sin(th_i)[:, None] * torch.sin(ph)[None, :],
                     torch.cos(th_i)[:, None].expand(hi, wi)], dim=-1)
    a = -th_o
    rot = torch.zeros(ho, 3, 3, dtype=torch.float64)
    rot[:, 0, 0], rot[:, 0, 2], rot[:, 1, 1], rot[:, 2, 0], rot[:, 2, 2] = torch.cos(a), torch.sin(a), 1.0, -torch.sin(a), torch.cos(a)
    u = torch.einsum("tab,ijb->tija", rot, v)
    r = torch.atan2(torch.hypot(u[..., 0], u[..., 1]), u[..., 2])
    bearing = torch.remainder(torch.atan2(u[..., 1], u[..., 0]), 2 * math.pi)
    rc = (1 + CUTOFF_SLACK) * theta_cutoff
    mask = r <= rc
    psi = morlet(kernel_shape, (r / rc).clamp(max=1.0), bearing) * mask                          # (K, ho, hi, wi)
    q = (2 * math.pi / wi) * w_i[None, None, :, None]
    vsum = (psi.abs() * q).sum(dim=(2, 3))                                                         # (K, ho)
    if basis_norm_mode == "mean":
        d = vsum.mean(dim=1, keepdim=True).expand_as(vsum)
    elif basis_norm_mode == "individual":
        d = vsum
    elif basis_norm_mode == "support":
        d = (mask * q).sum(dim=(2, 3)).expand_as(vsum)
    elif basis_norm_mode == "none":
        d = torch.ones_like(vsum)
    else:
        raise NotImplementedError(basis_norm_mode)
    return psi * q / (d[:, :, None, None] + NORM_EPS), mask


def contraction(x, psi2d, K, nlat_out, nlon_out):
    """X[b,c,k,t,p] = sum_{i,j} psi[k,t,i,j] x[b,c,i,(j + pscale p) mod nlon_in]; psi2d (K * nlat_out, nlat_in * nlon_in), dense or sparse COO"""
    B, C, hi, wi = x.shape
    ps = wi // nlon_out
    xf = x.reshape(B * C, hi, wi)
    cols = []
    for p in range(nlon_out):
        xr = torch.roll(xf, -ps * p, dims=-1).reshape(B * C, hi * wi)
        cols.append(torch.mm(psi2d, xr.t()) if not psi2d.is_sparse else torch.sparse.mm(psi2d, xr.t()))
    X = torch.stack(cols, dim=-1)                                                                  # (K * nlat_out, B * C, nlon_out)
    return X.reshape(K, nlat_out, B, C, nlon_out).permute(2, 3, 0, 1, 4).contiguous()


def adjoint(dX, psi2d, nlat_in, nlon_in):
    """dx[b,c,i,j'] = sum_{k,t,p} psi[k,t,i,j' - pscale p] dX[b,c,k,t,p] (the transpose of `contraction`)"""
    B, C, K, ho, wo = dX.shape
    ps = nlon_in // wo
    g = dX.permute(2, 3, 0, 1, 4).reshape(K * ho, B * C, wo)
    dx = torch.zeros(B * C, nlat_in, nlon_in, dtype=dX.dtype, device=dX.device)
    for p in range(wo):
        z = (psi2d.t() @ g[:, :, p]).t().reshape(B * C, nlat_in, nlon_in)
        dx += torch.roll(z, ps * p, dims=-1)
    return dx.reshape(B, C, nlat_in, nlon_in)


class DiscreteContinuousConvS2(nn.Module):
    """oracle of torch_harmonics.DiscreteContinuousConvS2: same constructor and parameters (fp32, drawn as the product draws them), psi in fp64"""

    def __init__(self, in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type="piecewise linear", basis_norm_mode="mean",
                 groups=1, grid_in="equiangular", grid_out="equiangular", bias=True, theta_cutoff=None, dtype=torch.float32):
        super().__init__()
        if basis_type != "morlet":
            raise NotImplementedError(f"the oracle restates the morlet basis only, not {basis_type!r}")
        if theta_cutoff is None:
            raise ValueError("theta_cutoff is required")
        if isinstance(kernel_shape, int):
            kernel_shape = (kernel_shape, kernel_shape)
        self.nlat_in, self.nlon_in = in_shape
        self.nlat_out, self.nlon_out = out_shape
        self.kernel_size = kernel_shape[0] * kernel_shape[1]
        self.groups, self.groupsize = groups, in_channels // groups
        psi, _ = dense_psi(tuple(kernel_shape), basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff)
        # psi stays fp64 whatever the parameters' dtype (`.double()` on the module makes the whole layer fp64)
        self.register_buffer("psi", psi.reshape(self.kernel_size * self.nlat_out, -1), persistent=False)
        scale = math.sqrt(1.0 / self.groupsize / self.kernel_size)
        self.weight = nn.Parameter(scale * torch.randn(out_channels, self.groupsize, self.kernel_size, dtype=dtype))
        self.bias = nn.Parameter(torch.zeros(out_channels, dtype=dtype)) if bias else None

    def forward(self, x):
        B = x.shape[0]
        X = contraction(x.to(self.psi.dtype), self.psi, self.kernel_size, self.nlat_out, self.nlon_out).to(self.weight.dtype)
        G = self.groups
        W = self.weight.reshape(G, -1, self.groupsize * self.kernel_size)
        y = torch.matmul(W, X.reshape(B, G, self.groupsize * self.kernel_size, -1)).reshape(B, -1, self.nlat_out, self.nlon_out)
        if self.bias is not None:
            y = y + self.bias.reshape(1, -1, 1, 1)
        return y

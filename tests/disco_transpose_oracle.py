"""fp64 oracle of the transposed DISCO convolution (torch_harmonics.DiscreteContinuousConvTransposeS2, basis "morlet")  --  TEST
INFRASTRUCTURE, NOT PRODUCT CODE.

The contract of makani_b200.DiscreteContinuousConvTransposeS2 restated independently of the product builder (`precompute_psi(...,
transpose=True)`), in the same way as oracle/makani_disco_oracle.py restates the forward convolution:
  - the geometry is that of the forward convolution from the out grid to the in grid: each in-grid latitude t (theta_in[t], phi = 0) is a
    centre; the out-grid points go through Cartesian unit vectors rotated by R_y(-theta_in[t]), r = atan2(|v_xy|, v_z),
    bearing = atan2(v_y, v_x), over the whole out grid (no band search), one centre row at a time so that FCN3-sized grids fit;
  - torch-harmonics' transpose normalisation with the quadrature merged, in the 2 pi w / nlon convention:
        v[k, i] = sum_{t, j} |psi_k(t, i, j)| 2 pi w_in[t] / nlon_out,   a[i] = sum_{t, j in support} 2 pi w_in[t] / nlon_out,
        d[k, i] = mean_i v[k, .] | v[k, i] | a[i] | 1,                   psi_T = psi_k(t, i, j) (2 pi w_in[t] / nlon_in) / (d[k, i] + 1e-9);
  - the transposed contraction y[b, c, i, j'] = sum_{k, t, p} psi_T[k, t, i, (j' - s p) mod nlon_out] Y[b, c, k, t, p] by roll-and-matmul,
    with psi_T dense or torch sparse COO.
torch-harmonics' source is not available, so element-wise parity with it is not pinned; tests/test_disco_transpose_cpu.py pins this restatement
by the adjoint identity to the forward oracle, the constant field and longitude equivariance.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from oracle.makani_disco_oracle import CUTOFF_SLACK, NORM_EPS, morlet
from oracle.makani_oracle import precompute_latitudes


def psi_T_entries(kernel_shape, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff, device="cpu"):
    """psi_T as COO entries: (t, i, j) index tensors of the support points and values (K, n), fp64 on `device`"""
    if isinstance(kernel_shape, int):
        kernel_shape = (kernel_shape, kernel_shape)
    (hi, wi), (ho, wo) = in_shape, out_shape
    th_i, w_i = (torch.from_numpy(np.asarray(a)).to(device) for a in precompute_latitudes(hi, grid_in))
    th_o, _ = (torch.from_numpy(np.asarray(a)).to(device) for a in precompute_latitudes(ho, grid_out))
    ph = torch.arange(wo, dtype=torch.float64, device=device) * (2 * math.pi / wo)
    v = torch.stack([torch.sin(th_o)[:, None] * torch.cos(ph)[None, :], torch.sin(th_o)[:, None] * torch.sin(ph)[None, :],
                     torch.cos(th_o)[:, None].expand(ho, wo)], dim=-1)                             # out-grid points (ho, wo, 3)
    rc = (1 + CUTOFF_SLACK) * theta_cutoff
    ts, iis, jjs, raw = [], [], [], []
    for t in range(hi):
        a = -th_i[t]
        rot = torch.zeros(3, 3, dtype=torch.float64, device=device)
        rot[0, 0], rot[0, 2], rot[1, 1], rot[2, 0], rot[2, 2] = torch.cos(a), torch.sin(a), 1.0, -torch.sin(a), torch.cos(a)
        u = v @ rot.T
        r = torch.atan2(torch.hypot(u[..., 0], u[..., 1]), u[..., 2])
        bearing = torch.remainder(torch.atan2(u[..., 1], u[..., 0]), 2 * math.pi)
        i, j = torch.nonzero(r <= rc, as_tuple=True)
        ts.append(torch.full_like(i, t))
        iis.append(i)
        jjs.append(j)
        raw.append(morlet(kernel_shape, r[i, j] / rc, bearing[i, j]))
    t, i, j, raw = torch.cat(ts), torch.cat(iis), torch.cat(jjs), torch.cat(raw, dim=1)
    K = raw.shape[0]
    qc = (2 * math.pi / wo) * w_i[t]                                                                 # per entry
    vsum = torch.zeros(K, ho, dtype=torch.float64, device=device).index_add_(1, i, raw.abs() * qc)
    area = torch.zeros(ho, dtype=torch.float64, device=device).index_add_(0, i, qc)
    if basis_norm_mode == "mean":
        d = vsum.mean(dim=1, keepdim=True).expand_as(vsum)
    elif basis_norm_mode == "individual":
        d = vsum
    elif basis_norm_mode == "support":
        d = area[None, :].expand_as(vsum)
    elif basis_norm_mode == "none":
        d = torch.ones_like(vsum)
    else:
        raise NotImplementedError(basis_norm_mode)
    return t, i, j, raw * ((2 * math.pi / wi) * w_i[t]) / (d[:, i] + NORM_EPS)


def dense_psi_T(kernel_shape, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff):
    """psi_T (K, nlat_in, nlat_out, nlon_out) fp64 (small grids)"""
    t, i, j, val = psi_T_entries(kernel_shape, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff)
    K, (ho, wo) = val.shape[0], out_shape
    out = torch.zeros(K, in_shape[0], ho, wo, dtype=torch.float64)
    out[:, t, i, j] = val
    return out


def sparse_psi_T(kernel_shape, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff, device="cpu"):
    """psi_T as a coalesced torch sparse COO matrix (K * nlat_in, nlat_out * nlon_out) fp64 on `device`"""
    t, i, j, val = psi_T_entries(kernel_shape, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff, device)
    K, hi, (ho, wo) = val.shape[0], in_shape[0], out_shape
    k = torch.arange(K, device=val.device)[:, None].expand_as(val)
    idx = torch.stack([(k * hi + t).reshape(-1), (i * wo + j).expand_as(val).reshape(-1)])
    return torch.sparse_coo_tensor(idx, val.reshape(-1), (K * hi, ho * wo)).coalesce()


def transpose_contraction(Y, psi2d, nlat_out, nlon_out):
    """y[b,c,i,j'] = sum_{k,t,p} psi_T[k,t,i,(j' - s p) mod nlon_out] Y[b,c,k,t,p]; psi2d (K * nlat_in, nlat_out * nlon_out), dense or sparse"""
    B, C, K, hi, wi = Y.shape
    s = nlon_out // wi
    g = Y.permute(2, 3, 0, 1, 4).reshape(K * hi, B * C, wi)
    pt = psi2d.t()
    y = torch.zeros(B * C, nlat_out, nlon_out, dtype=Y.dtype, device=Y.device)
    for p in range(wi):
        y += torch.roll((pt @ g[:, :, p]).t().reshape(B * C, nlat_out, nlon_out), s * p, dims=-1)
    return y.reshape(B, C, nlat_out, nlon_out)


class DiscreteContinuousConvTransposeS2(nn.Module):
    """oracle of torch_harmonics.DiscreteContinuousConvTransposeS2: the product's constructor and parameter draw (fp32), psi_T in fp64;
    `sparse=True` holds psi_T as a sparse COO matrix built on `device` (FCN3-sized grids)"""

    def __init__(self, in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type="piecewise linear", basis_norm_mode="mean",
                 groups=1, grid_in="equiangular", grid_out="equiangular", bias=True, theta_cutoff=None, dtype=torch.float32, sparse=False,
                 device="cpu"):
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
        args = (tuple(kernel_shape), basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff)
        self.psi = sparse_psi_T(*args, device=device) if sparse else dense_psi_T(*args).reshape(self.kernel_size * self.nlat_in, -1)
        scale = math.sqrt(1.0 / self.groupsize / self.kernel_size)
        self.weight = nn.Parameter(scale * torch.randn(out_channels, self.groupsize, self.kernel_size, dtype=dtype))
        self.bias = nn.Parameter(torch.zeros(out_channels, dtype=dtype)) if bias else None

    def forward(self, x):
        B, G, K = x.shape[0], self.groups, self.kernel_size
        W = self.weight.reshape(G, -1, self.groupsize, K)                                           # (G, C_out/G, C_in/G, K)
        Y = torch.einsum("gock,bgcp->bgokp", W, x.reshape(B, G, self.groupsize, -1))
        Y = Y.reshape(B, -1, K, self.nlat_in, self.nlon_in)
        y = transpose_contraction(Y.to(torch.float64), self.psi, self.nlat_out, self.nlon_out).to(self.weight.dtype)
        if self.bias is not None:
            y = y + self.bias.reshape(1, -1, 1, 1)
        return y

"""DiscreteContinuousConvS2 -- drop-in for `torch_harmonics.DiscreteContinuousConvS2` as FCN3 builds it (makani/models/networks/fourcastnet3.py:117-252
encoders, :364-381 decoders, :511-543 the "local" processor blocks; snonet.py), with the filter contraction on the sm_90a kernels of csrc/disco.cu.

    DiscreteContinuousConvS2(in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type="piecewise linear", basis_norm_mode="mean",
                             groups=1, grid_in="equiangular", grid_out="equiangular", bias=True, theta_cutoff=None)
    forward: x (B, C_in, *in_shape) fp32 / bf16 on a CUDA device -> float32 (B, C_out, *out_shape)

The filter tensor psi_hat[k, t, i, j] is built here on the host in fp64 (`precompute_psi`, the contract restated in include/b200sht.h and DESIGN.md
section 5) and held by output latitude in CSR form.  The library's plan keeps it twice on the device, in fp32.  y = W X (+ bias) with
X = contraction(x) of shape (B, C_in, K, *out_shape) is a grouped GEMM on cuBLAS (torch.matmul; TF32 follows torch.backends.cuda.matmul.allow_tf32).
The backward recomputes X for the weight gradient rather than keeping it (X is K times the activation) and returns dx = adjoint(W^T dy).

DiscreteContinuousConvTransposeS2 (drop-in for `torch_harmonics.DiscreteContinuousConvTransposeS2`, same constructor) runs the same two kernels
the other way round on a plan of the swapped geometry: its forward is the adjoint kernel after the GEMM, its backward the forward kernel.

Only the "morlet" basis is implemented; "piecewise linear", "zernike", "harmonic" and the "nodal" norm mode raise NotImplementedError, and
theta_cutoff=None raises ValueError (every makani call site passes it).
"""
import math
import threading
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import B200ShtError
from .quadrature import _grid_np
from .sht import _dtype_code, _ptr, _stream

CUTOFF_SLACK = 1e-3      # support r <= (1 + CUTOFF_SLACK) theta_cutoff
NORM_EPS = 1e-9          # psi_hat = psi q / (d + NORM_EPS)
NORM_MODES = ("mean", "individual", "support", "none")
_UNIMPLEMENTED_BASES = ("piecewise linear", "zernike", "harmonic")


class MorletFilterBasis:
    """Morlet basis on the unit disk (`torch_harmonics.filter_basis` for basis_type="morlet"): kernel_shape (n0, n1), K = n0 n1;
    function k has n = k mod n1, m = k // n1 and psi_k(rho, phi) = cos^2(pi rho / 2) h_n(rho sin phi) h_m(rho cos phi)."""

    def __init__(self, kernel_shape):
        if isinstance(kernel_shape, int):
            kernel_shape = (kernel_shape, kernel_shape)
        if len(kernel_shape) != 2 or min(kernel_shape) < 1:
            raise ValueError(f"morlet kernel_shape must be (n0, n1) with n0, n1 >= 1, got {kernel_shape}")
        self.kernel_shape = tuple(int(s) for s in kernel_shape)

    @property
    def kernel_size(self):
        return self.kernel_shape[0] * self.kernel_shape[1]

    @staticmethod
    def _h(j, u):
        f = math.ceil(j / 2) * math.pi
        return np.sin(f * u) if j % 2 else np.cos(f * u)

    def __call__(self, rho, phi):
        """values (K, n) at normalised radii rho in [0, 1] and bearings phi"""
        n1 = self.kernel_shape[1]
        x, y = rho * np.sin(phi), rho * np.cos(phi)
        hann = np.cos(0.5 * np.pi * rho) ** 2
        return np.stack([hann * self._h(k % n1, x) * self._h(k // n1, y) for k in range(self.kernel_size)])


def get_filter_basis(kernel_shape, basis_type):
    """`torch_harmonics.filter_basis.get_filter_basis`: an object with `.kernel_size` (and `.kernel_shape`)."""
    if basis_type == "morlet":
        return MorletFilterBasis(kernel_shape)
    if basis_type in _UNIMPLEMENTED_BASES:
        raise NotImplementedError(f"DISCO filter basis {basis_type!r} is not implemented (only 'morlet' is)")
    raise ValueError(f"unknown DISCO filter basis {basis_type!r}")


# CSR by output latitude t: entries row_ptr[t] .. row_ptr[t + 1] - 1 hold (ker, col = i * nlon_in + j, val), sorted by (i, j, k)
DiscoPsi = namedtuple("DiscoPsi", "row_ptr ker col val nlat_in nlon_in nlat_out nlon_out kernel_size")


def support_search(in_shape, out_shape, grid_in, grid_out, theta_cutoff):
    """The support of every output latitude t (its point at longitude 0): a list of (i, j, r, bearing) arrays, one entry per input point with
    r <= (1 + CUTOFF_SLACK) theta_cutoff, in (i, j) order.  Shared by the DISCO filter tensor and the neighbourhood of NeighborhoodAttentionS2."""
    (nlat_in, nlon_in), (nlat_out, nlon_out) = in_shape, out_shape
    if nlon_in % nlon_out:
        raise ValueError(f"nlon_in {nlon_in} must be a multiple of nlon_out {nlon_out}")
    cost_in, _ = _grid_np(nlat_in, grid_in)
    cost_out, _ = _grid_np(nlat_out, grid_out)
    th_in, th_out = np.arccos(np.clip(cost_in, -1, 1)), np.arccos(np.clip(cost_out, -1, 1))
    phi = 2.0 * np.pi * np.arange(nlon_in) / nlon_in
    rc = (1.0 + CUTOFF_SLACK) * theta_cutoff
    out = []
    for t in range(nlat_out):
        rows = np.nonzero(np.abs(th_in - th_out[t]) <= rc)[0]   # r >= |theta_i - theta_t|
        ct, st = math.cos(th_out[t]), math.sin(th_out[t])
        ci, si = np.cos(th_in[rows])[:, None], np.sin(th_in[rows])[:, None]
        cp, sp = np.cos(phi)[None, :], np.sin(phi)[None, :]
        # the input point in the frame of the output point: (xr, yr, zr) = R_y(-theta_t) (sin th cos ph, sin th sin ph, cos th).
        # r = arccos(zr) evaluated as atan2(|(xr, yr)|, zr): the same angle, without arccos' loss of half the digits near r = 0
        xr, yr, zr = ct * si * cp - ci * st, sp * si, ct * ci + st * si * cp
        r = np.arctan2(np.hypot(xr, yr), zr)
        bearing = np.mod(np.arctan2(yr, xr), 2.0 * np.pi)
        ii, jj = np.nonzero(r <= rc)
        out.append((rows[ii], jj, r[ii, jj], bearing[ii, jj]))
    return out


def precompute_psi(kernel_shape, basis_type, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff, transpose=False):
    """psi_hat in fp64 as DiscoPsi.  Every grid point with r <= (1 + 1e-3) theta_cutoff is present for every k (zeros of the basis included).

    transpose=True gives psi_T of DiscreteContinuousConvTransposeS2 on this (swapped) geometry: the same support and basis values, with
    torch-harmonics' transpose normalisation.  Its sums run over the entries of each input row i, weighted by the quadrature of their centre
    row t: v[k, i] = sum |psi| 2 pi w_out[t] / nlon_in, the support a[i] = sum 2 pi w_out[t] / nlon_in, and
    psi_T = psi 2 pi w_out[t] / nlon_out / (d[k, i] + 1e-9)."""
    basis = get_filter_basis(kernel_shape, basis_type)
    if basis_norm_mode not in NORM_MODES:
        if basis_norm_mode == "nodal":
            raise NotImplementedError("DISCO basis_norm_mode 'nodal' is not implemented")
        raise ValueError(f"unknown basis_norm_mode {basis_norm_mode!r}")
    (nlat_in, nlon_in), (nlat_out, nlon_out) = in_shape, out_shape
    K = basis.kernel_size
    _, w_in = _grid_np(nlat_in, grid_in)
    _, w_out = _grid_np(nlat_out, grid_out)
    q = 2.0 * np.pi * w_in / nlon_in
    rc = (1.0 + CUTOFF_SLACK) * theta_cutoff
    # (i, j, psi (K, n)) of each output latitude
    per_t = [(i, j, basis(r / rc, bearing)) for i, j, r, bearing in support_search(in_shape, out_shape, grid_in, grid_out, theta_cutoff)]

    if transpose:
        qc = 2.0 * np.pi * w_out / nlon_in                                 # quadrature of the centre rows, in the sums of v and a
        v, s = np.zeros((K, nlat_in)), np.zeros(nlat_in)                   # (K, nlat_in), (nlat_in,)
        for t, (i, _, p) in enumerate(per_t):
            v += np.stack([np.bincount(i, np.abs(pk), nlat_in) for pk in p]) * qc[t]
            s += np.bincount(i, minlength=nlat_in) * qc[t]
    else:
        v = np.stack([np.sum(np.abs(p) * q[i], axis=1) for i, _, p in per_t], axis=1)   # (K, nlat_out)
        s = np.array([np.sum(q[i]) for i, _, _ in per_t])
    nrow = v.shape[1]
    if basis_norm_mode == "mean":
        d = np.repeat(v.mean(axis=1, keepdims=True), nrow, axis=1)
    elif basis_norm_mode == "individual":
        d = v
    elif basis_norm_mode == "support":
        d = np.repeat(s[None, :], K, axis=0)
    else:
        d = np.ones((K, nrow))

    row_ptr = np.zeros(nlat_out + 1, dtype=np.int64)
    ker, col, val = [], [], []
    for t, (i, j, p) in enumerate(per_t):
        n = len(i)
        if transpose:
            vals = p * (2.0 * np.pi * w_out[t] / nlon_out) / (d[:, i] + NORM_EPS)
        else:
            vals = p * q[i][None, :] / (d[:, t : t + 1] + NORM_EPS)      # (K, n), points already in (i, j) order
        ker.append(np.tile(np.arange(K, dtype=np.int32), n))
        col.append(np.repeat((i * nlon_in + j).astype(np.int32), K))
        val.append(vals.T.reshape(-1))
        row_ptr[t + 1] = row_ptr[t] + n * K
    cat = lambda a, dt: np.concatenate(a).astype(dt) if a else np.zeros(0, dt)   # noqa: E731
    return DiscoPsi(row_ptr, cat(ker, np.int32), cat(col, np.int32), cat(val, np.float64), nlat_in, nlon_in, nlat_out, nlon_out, K)


def psi_lat_out(psi):
    """output latitude of every entry of a DiscoPsi"""
    return np.repeat(np.arange(psi.nlat_out, dtype=np.int32), np.diff(psi.row_ptr))


def psi_dense(psi):
    """psi_hat as a dense fp64 array (K, nlat_out, nlat_in, nlon_in) (tests, small grids)"""
    out = np.zeros((psi.kernel_size, psi.nlat_out, psi.nlat_in * psi.nlon_in))
    out[psi.ker, psi_lat_out(psi), psi.col] = psi.val
    return out.reshape(psi.kernel_size, psi.nlat_out, psi.nlat_in, psi.nlon_in)


class DiscoPlan:
    """Owner of a b200sht_disco_plan (both device layouts of psi_hat in fp32)."""

    def __init__(self, psi, device):
        lib = _lib.load()
        self.device = torch.device(device)
        self.nlat_in, self.nlon_in, self.nlat_out, self.nlon_out, self.K = psi.nlat_in, psi.nlon_in, psi.nlat_out, psi.nlon_out, psi.kernel_size
        lat = np.ascontiguousarray(psi_lat_out(psi))
        ker, col = np.ascontiguousarray(psi.ker, np.int32), np.ascontiguousarray(psi.col, np.int32)
        val = np.ascontiguousarray(psi.val, np.float64)
        h = _lib.c_void_p()
        with torch.cuda.device(self.device):
            _lib.call("b200sht_disco_plan_create", _lib.ctypes.byref(h), self.nlat_in, self.nlon_in, self.nlat_out, self.nlon_out, self.K,
                      len(val), ker.ctypes.data, lat.ctypes.data, col.ctypes.data, val.ctypes.data, _stream(self.device))
        self.handle, self._lib = h, lib

    def query(self, what):
        return int(self._lib.b200sht_disco_plan_query(self.handle, what))

    def __del__(self):
        h = getattr(self, "handle", None)
        if h is not None and h.value and getattr(self, "_lib", None) is not None:
            self._lib.b200sht_disco_plan_destroy(h)
            self.handle = None

    def forward(self, x):
        """x (B, C, nlat_in, nlon_in) fp32 / bf16 contiguous -> X (B, C, K, nlat_out, nlon_out) fp32"""
        B, C = x.shape[0], x.shape[1]
        X = torch.empty((B, C, self.K, self.nlat_out, self.nlon_out), dtype=torch.float32, device=x.device)
        _lib.call("b200sht_disco_forward", self.handle, _ptr(x), _dtype_code(x.dtype), B, C, _ptr(X), _stream(x.device))
        return X

    def adjoint(self, dX, dtype=torch.float32):
        """dX (B, C, K, nlat_out, nlon_out) fp32 contiguous -> dx (B, C, nlat_in, nlon_in) of `dtype`"""
        B, C = dX.shape[0], dX.shape[1]
        dx = torch.empty((B, C, self.nlat_in, self.nlon_in), dtype=dtype, device=dX.device)
        _lib.call("b200sht_disco_adjoint", self.handle, _ptr(dX), _ptr(dx), _dtype_code(dtype), B, C, _stream(dX.device))
        return dx


_psi_cache, _plan_cache, _cache_lock = {}, {}, threading.Lock()


def _psi_key(kernel_shape, basis_type, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff, transpose=False):
    key = (tuple(kernel_shape), basis_type, basis_norm_mode, tuple(in_shape), tuple(out_shape), grid_in, grid_out, float(theta_cutoff))
    return key + (True,) if transpose else key


def get_psi(*key):
    """precompute_psi, cached per (kernel shape, basis, norm mode, geometry, cutoff[, transpose])"""
    with _cache_lock:
        if key not in _psi_cache:
            _psi_cache[key] = precompute_psi(*key)
        return _psi_cache[key]


def get_plan(key, device):
    """the device plan of get_psi(*key), cached per key and device"""
    device = torch.device(device)
    if device.type != "cuda":
        raise B200ShtError(f"the DISCO convolution runs on CUDA devices only (got {device}); makani_b200 has no CPU fallback")
    dkey = key + (device.index if device.index is not None else torch.cuda.current_device(),)
    with _cache_lock:
        plan = _plan_cache.get(dkey)
    if plan is None:
        plan = DiscoPlan(get_psi(*key), device)
        with _cache_lock:
            plan = _plan_cache.setdefault(dkey, plan)
    return plan


def _grouped(W, G):
    """(C_out, C_in/G, K) -> (G, C_out/G, C_in/G * K)"""
    return W.reshape(G, W.shape[0] // G, -1)


class _DiscoConv(torch.autograd.Function):
    """y = W_g X_g (+ bias), X = plan.forward(x).  Saves x and W only."""

    @staticmethod
    def forward(ctx, x, weight, bias, plan, groups):
        B = x.shape[0]
        X = plan.forward(x)
        Wg = _grouped(weight.to(torch.float32), groups)
        y = torch.matmul(Wg, X.view(B, groups, -1, plan.nlat_out * plan.nlon_out))      # (B, G, C_out/G, HW)
        y = y.view(B, weight.shape[0], plan.nlat_out, plan.nlon_out)
        if bias is not None:
            y = y + bias.to(torch.float32).view(1, -1, 1, 1)
        ctx.save_for_backward(x, weight)
        ctx.plan, ctx.groups, ctx.has_bias = plan, groups, bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        plan, G = ctx.plan, ctx.groups
        B, C = x.shape[0], x.shape[1]
        gy = gy.to(torch.float32).contiguous()
        gyg = gy.view(B, G, -1, plan.nlat_out * plan.nlon_out)
        Wg = _grouped(weight.to(torch.float32), G)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dX = torch.matmul(Wg.transpose(1, 2), gyg)                                      # (B, G, C_in/G * K, HW)
            dx = plan.adjoint(dX.view(B, C, plan.K, plan.nlat_out, plan.nlon_out), x.dtype)
        if ctx.needs_input_grad[1]:
            X = plan.forward(x).view(B, G, -1, plan.nlat_out * plan.nlon_out)
            dw = torch.matmul(gyg, X.transpose(2, 3)).sum(0).reshape(weight.shape).to(weight.dtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = gy.sum(dim=(0, 2, 3))
        return dx, dw, db, None, None


def _transposed_mix(W, G):
    """(C_out, C_in/G, K) -> (G, C_out/G * K, C_in/G): the channel mix of the transposed convolution, rows (o, k)"""
    Wg = _grouped(W, G)
    return Wg.view(G, Wg.shape[1], W.shape[1], W.shape[2]).transpose(2, 3).reshape(G, -1, W.shape[1])


class _DiscoConvTranspose(torch.autograd.Function):
    """y = adjoint(Y) (+ bias), Y = W_g^T-mix of x with K-fold rows (o, k).  Saves x and W only; the backward's gY = plan.forward(gy)."""

    @staticmethod
    def forward(ctx, x, weight, bias, plan, groups):
        B, C_out = x.shape[0], weight.shape[0]
        Y = torch.matmul(_transposed_mix(weight.to(torch.float32), groups),
                         x.to(torch.float32).view(B, groups, -1, plan.nlat_out * plan.nlon_out))   # (B, G, C_out/G * K, HW_in)
        y = plan.adjoint(Y.view(B, C_out, plan.K, plan.nlat_out, plan.nlon_out))
        if bias is not None:
            y = y + bias.to(torch.float32).view(1, -1, 1, 1)
        ctx.save_for_backward(x, weight)
        ctx.plan, ctx.groups, ctx.has_bias = plan, groups, bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        plan, G = ctx.plan, ctx.groups
        B, C, HW = x.shape[0], x.shape[1], plan.nlat_out * plan.nlon_out
        gy = gy.to(torch.float32).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            gY = plan.forward(gy).view(B, G, -1, HW)                                             # (B, G, C_out/G * K, HW_in)
            Wt = _transposed_mix(weight.to(torch.float32), G)
        if ctx.needs_input_grad[0]:
            dx = torch.matmul(Wt.transpose(1, 2), gY).view(x.shape).to(x.dtype)
        if ctx.needs_input_grad[1]:
            dWt = torch.matmul(gY, x.to(torch.float32).view(B, G, -1, HW).transpose(2, 3)).sum(0)   # (G, C_out/G * K, C_in/G)
            dw = dWt.view(G, -1, plan.K, C // G).transpose(2, 3).reshape(weight.shape).to(weight.dtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = gy.sum(dim=(0, 2, 3))
        return dx, dw, db, None, None


class _DiscreteContinuousConv(nn.Module):
    """The constructor, attributes, parameters and plan of both DISCO convolutions; `_transpose` selects the geometry of psi_hat."""

    _transpose = False

    def __init__(self, in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type="piecewise linear", basis_norm_mode="mean",
                 groups=1, grid_in="equiangular", grid_out="equiangular", bias=True, theta_cutoff=None):
        super().__init__()
        if theta_cutoff is None:
            name = "DiscreteContinuousConvTransposeS2" if self._transpose else "DiscreteContinuousConvS2"
            raise ValueError(f"{name} needs an explicit theta_cutoff (the default cutoff is not implemented)")
        if theta_cutoff <= 0:
            raise ValueError(f"theta_cutoff must be positive, got {theta_cutoff}")
        basis = get_filter_basis(kernel_shape, basis_type)
        if basis_norm_mode == "nodal":
            raise NotImplementedError("DISCO basis_norm_mode 'nodal' is not implemented")
        if basis_norm_mode not in NORM_MODES:
            raise ValueError(f"unknown basis_norm_mode {basis_norm_mode!r}")
        if in_channels % groups or out_channels % groups:
            raise ValueError(f"in_channels {in_channels} and out_channels {out_channels} must be divisible by groups {groups}")
        self.nlat_in, self.nlon_in = in_shape
        self.nlat_out, self.nlon_out = out_shape
        if self._transpose and self.nlon_out % self.nlon_in:
            raise ValueError(f"nlon_out {self.nlon_out} must be a multiple of nlon_in {self.nlon_in}")
        if not self._transpose and self.nlon_in % self.nlon_out:
            raise ValueError(f"nlon_in {self.nlon_in} must be a multiple of nlon_out {self.nlon_out}")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_shape, self.basis_type, self.basis_norm_mode = basis.kernel_shape, basis_type, basis_norm_mode
        self.grid_in, self.grid_out, self.theta_cutoff = grid_in, grid_out, float(theta_cutoff)
        self.kernel_size = basis.kernel_size
        self.groups = groups
        self.groupsize = in_channels // groups
        if self._transpose:     # psi_T lives on the geometry of the forward convolution from the out grid to the in grid
            self._key = _psi_key(self.kernel_shape, basis_type, basis_norm_mode, out_shape, in_shape, grid_out, grid_in, theta_cutoff, True)
        else:
            self._key = _psi_key(self.kernel_shape, basis_type, basis_norm_mode, in_shape, out_shape, grid_in, grid_out, theta_cutoff)
        psi = get_psi(*self._key)
        # psi_hat (CSR by output latitude) as non-persistent buffers: a state dict holds only weight / bias
        self.register_buffer("psi_row_ptr", torch.from_numpy(psi.row_ptr), persistent=False)
        self.register_buffer("psi_ker", torch.from_numpy(psi.ker), persistent=False)
        self.register_buffer("psi_col", torch.from_numpy(psi.col), persistent=False)
        self.register_buffer("psi_vals", torch.from_numpy(psi.val), persistent=False)
        scale = math.sqrt(1.0 / self.groupsize / self.kernel_size)
        self.weight = nn.Parameter(scale * torch.randn(out_channels, self.groupsize, self.kernel_size))
        self.bias = nn.Parameter(torch.zeros(out_channels)) if bias else None

    def extra_repr(self):
        return (f"in_channels={self.in_channels}, out_channels={self.out_channels}, in_shape={(self.nlat_in, self.nlon_in)}, "
                f"out_shape={(self.nlat_out, self.nlon_out)}, kernel_shape={self.kernel_shape}, basis_type={self.basis_type!r}, "
                f"basis_norm_mode={self.basis_norm_mode!r}, groups={self.groups}, theta_cutoff={self.theta_cutoff}")

    def plan(self, device):
        return get_plan(self._key, device)

    def _check_input(self, x):
        if not x.is_cuda:
            raise B200ShtError(f"{type(self).__name__} runs on CUDA devices only; makani_b200 has no CPU fallback")
        if x.dim() != 4 or x.shape[1] != self.in_channels or tuple(x.shape[2:]) != (self.nlat_in, self.nlon_in):
            raise ValueError(f"expected (B, {self.in_channels}, {self.nlat_in}, {self.nlon_in}), got {tuple(x.shape)}")
        return (x if x.dtype in (torch.float32, torch.bfloat16) else x.to(torch.float32)).contiguous()


class DiscreteContinuousConvS2(_DiscreteContinuousConv):
    """Discrete-continuous convolution on the sphere (drop-in for torch_harmonics.DiscreteContinuousConvS2).

    weight (C_out, C_in / groups, K), initialised sqrt(1 / (C_in / groups) / K) randn; bias (C_out,) zeros.  psi_hat is not part of the state dict."""

    def forward(self, x):
        return _DiscoConv.apply(self._check_input(x), self.weight, self.bias, self.plan(x.device), self.groups)


class DiscreteContinuousConvTransposeS2(_DiscreteContinuousConv):
    """Transposed discrete-continuous convolution on the sphere (drop-in for torch_harmonics.DiscreteContinuousConvTransposeS2), for learnable
    upsampling: x (B, C_in, *in_shape) -> float32 (B, C_out, *out_shape), nlon_out a multiple of nlon_in.

        Y[b, o, k, t, p] = sum_c W[o, c, k] x[b, g(o) C_in / G + c, t, p]              (grouped GEMM on cuBLAS)
        y[b, o, i, j']  = sum_{k, t, p} psi_T[k, t, i, (j' - s p) mod nlon_out] Y[b, o, k, t, p] (+ bias[o]),  s = nlon_out / nlon_in

    psi_T is the filter tensor of the forward convolution from the out grid to the in grid with torch-harmonics' transpose normalisation
    (`precompute_psi(..., transpose=True)`), so the contraction above is the adjoint kernel of that plan and the backward's gY is its forward
    kernel.  Constructor, attributes and parameters as DiscreteContinuousConvS2; weight (C_out, C_in / groups, K)."""

    _transpose = True

    def forward(self, x):
        return _DiscoConvTranspose.apply(self._check_input(x), self.weight, self.bias, self.plan(x.device), self.groups)


def __getattr__(name):
    # the distributed module lives in makani_b200/distributed/disco.py; the reference runners import it from here
    if name in ("DistributedDiscreteContinuousConvS2", "DistributedDiscreteContinuousConvTransposeS2"):
        from .distributed import disco
        return getattr(disco, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")

"""DistributedDiscreteContinuousConvS2 -- `torch_harmonics.distributed.DistributedDiscreteContinuousConvS2` as makani builds it at spatial model
parallelism > 1 (FCN3's encoders, decoders and local processor blocks), on the sm_90a kernels of csrc/disco.cu.

    x local (B, C_in, lat_in_shapes[ih], lon_in_shapes[iw]) -> y local (B, C_out, lat_out_shapes[ih], lon_out_shapes[iw]) float32

    forward : [w-a2a rows of B*C <-> lon] -> [h halo: input rows lo .. hi of this rank's window] -> window contraction
              -> [w-a2a lon <-> rows] -> grouped GEMM (+ bias) on the local pixels
    backward: GEMM^T -> [w-a2a] -> window adjoint -> [h halo adjoint, fixed rank order] -> [w-a2a];  dW, dbias: local partial sums

Every rank derives the windows of all ranks from the same global psi_hat (normalised before slicing), so the halo needs no handshake.  The
window plan holds the global plan's entries of this rank's output rows in the same (i, j) order, with the input rows re-indexed to i - lo:
the forward kernel then sums every element of X over the same points in the same order as on one GPU, and X is bit-identical to the
corresponding slice of the single-GPU X.  As the serial module, the backward recomputes X (kernel + one azimuth all-to-all) rather than
keeping it; only the window of x is saved.  The per-rank stages are replaceable (`set_disco_local_ops`) so the choreography is unit-tested on
CPU with gloo against the serial oracle.

DistributedDiscreteContinuousConvTransposeS2 runs the same stages the other way round on the windows of its psi_T plan, whose output rows
are the module's input latitudes: the backward chain above as its forward, the forward chain as its backward.
"""
import threading
from collections import namedtuple

import numpy as np
import torch

from .._lib import B200ShtError
from ..disco import DiscoPlan, DiscoPsi, DiscreteContinuousConvS2, DiscreteContinuousConvTransposeS2, _grouped, _transposed_mix, get_psi
from .primitives import _all_to_all, _transpose, compute_split_shapes

# output rows [t0, t1) of a rank, its input window [lo, hi) and the entries of those output rows (input rows re-indexed to i - lo)
DiscoWindow = namedtuple("DiscoWindow", "t0 t1 lo hi psi")


def window_psi(psi, t0, t1):
    """the DiscoWindow of output rows [t0, t1) of a global DiscoPsi: [lo, hi) is the minimal range of input rows its entries touch (empty: 0, 0)"""
    a, b = int(psi.row_ptr[t0]), int(psi.row_ptr[t1])
    rows = psi.col[a:b] // psi.nlon_in
    lo, hi = (int(rows.min()), int(rows.max()) + 1) if b > a else (0, 0)
    sub = DiscoPsi(psi.row_ptr[t0 : t1 + 1] - a, psi.ker[a:b], (psi.col[a:b] - lo * psi.nlon_in).astype(np.int32), psi.val[a:b],
                   hi - lo, psi.nlon_in, t1 - t0, psi.nlon_out, psi.kernel_size)
    return DiscoWindow(t0, t1, lo, hi, sub)


def disco_windows(psi, lat_out_shapes):
    """the DiscoWindow of every polar rank"""
    off = np.concatenate([[0], np.cumsum(lat_out_shapes)]).astype(int)
    return [window_psi(psi, int(off[r]), int(off[r + 1])) for r in range(len(lat_out_shapes))]


def halo_plan(windows, lat_in_shapes, rank):
    """(send, recv) of polar rank `rank`: send[p] = local rows [a, b) of this rank that p's window holds, recv[p] = rows of p in this window"""
    off = np.concatenate([[0], np.cumsum(lat_in_shapes)]).astype(int)
    me = windows[rank]
    send, recv = [], []
    for p, wp in enumerate(windows):
        a, b = max(off[rank], wp.lo), min(off[rank + 1], wp.hi)
        send.append((a - off[rank], b - off[rank]) if b > a else (0, 0))
        recv.append(max(0, min(off[p + 1], me.hi) - max(off[p], me.lo)))
    return send, recv


def halo_exchange(x, send, recv, group):
    """x (R, rows of this rank, W) -> (R, hi - lo, W): the rows of this rank's window, gathered from their owners in rank order"""
    sends = [x[:, a:b].contiguous() for a, b in send]
    if len(send) == 1:
        return sends[0]
    recvs = [x.new_empty((x.shape[0], n, x.shape[2])) for n in recv]
    _all_to_all(recvs, sends, group)
    return torch.cat(recvs, dim=1)


def halo_adjoint(g, send, recv, nrows, group):
    """the adjoint of halo_exchange: g (R, hi - lo, W) -> (R, nrows, W), the window rows returned to their owners and added in rank order"""
    chunks = [c.contiguous() for c in torch.split(g, recv, dim=1)]
    if len(send) == 1:
        back = chunks
    else:
        back = [g.new_empty((g.shape[0], b - a, g.shape[2])) for a, b in send]
        _all_to_all(back, chunks, group)
    out = g.new_zeros((g.shape[0], nrows, g.shape[2]))
    for (a, b), c in zip(send, back):
        if b > a:
            out[:, a:b] += c
    return out


def _a2a(x, dim0, dim1, dim1_split_sizes, group):
    """shard dim0, gather dim1 (the forward of _DistributedTranspose, without autograd)"""
    xs, _, _ = _transpose(x.contiguous(), dim0, dim1, dim1_split_sizes, group=group)
    return torch.cat(xs, dim=dim1).contiguous()


# ------------------------------------------------------------------------------------------------------- local stages
_window_plans, _window_lock = {}, threading.Lock()


def window_plan(plan_class, key, window, device, what):
    """plan_class(window.psi, device), cached per plan class, global key, window and device"""
    if device.type != "cuda":
        raise B200ShtError(f"{what} runs on CUDA devices only (got {device}); makani_b200 has no CPU fallback")
    k = (plan_class,) + tuple(key) + (window.t0, window.t1, device.index if device.index is not None else torch.cuda.current_device())
    with _window_lock:
        p = _window_plans.get(k)
    if p is None:
        p = plan_class(window.psi, device)
        with _window_lock:
            p = _window_plans.setdefault(k, p)
    return p


class CudaDiscoLocalOps:
    """The window contraction and its adjoint on the kernels of csrc/disco.cu, on a plan of `layer.window` (cached per key, window, device).
    `layer` has `_key` (the psi_hat key of makani_b200.disco) and `window` (a DiscoWindow)."""

    def __init__(self, layer):
        self.key, self.window = layer._key, layer.window

    def _plan(self, device):
        return window_plan(DiscoPlan, self.key, self.window, device, "the DISCO convolution")

    def contract(self, xwin):
        """xwin (R, hi - lo, nlon_in) fp32 / bf16 -> X (R, K, t1 - t0, nlon_out) fp32"""
        w, R = self.window, xwin.shape[0]
        psi = w.psi
        if w.hi == w.lo:
            return torch.zeros((R, psi.kernel_size, psi.nlat_out, psi.nlon_out), dtype=torch.float32, device=xwin.device)
        X = self._plan(xwin.device).forward(xwin.contiguous().view(R, 1, w.hi - w.lo, psi.nlon_in))
        return X.view(R, psi.kernel_size, psi.nlat_out, psi.nlon_out)

    def adjoint(self, dX):
        """dX (R, K, t1 - t0, nlon_out) fp32 -> dxwin (R, hi - lo, nlon_in) fp32"""
        w, R = self.window, dX.shape[0]
        if w.hi == w.lo:
            return torch.zeros((R, 0, w.psi.nlon_in), dtype=torch.float32, device=dX.device)
        dx = self._plan(dX.device).adjoint(dX.contiguous().view(R, 1, *dX.shape[1:]))
        return dx.view(R, w.hi - w.lo, w.psi.nlon_in)


_OPS_FACTORY = CudaDiscoLocalOps


def set_disco_local_ops(factory):
    """Replace the per-rank stages (tests: a CPU implementation on the oracle).  `factory(layer)` -> object with contract(xwin) and adjoint(dX)
    as CudaDiscoLocalOps; None restores the CUDA stages."""
    global _OPS_FACTORY
    _OPS_FACTORY = factory if factory is not None else CudaDiscoLocalOps


# ------------------------------------------------------------------------------------------------------------ module
class _DistDiscoConv(torch.autograd.Function):
    """y = W_g X_g (+ bias) on the local pixels.  Saves the window of x and W only."""

    @staticmethod
    def forward(ctx, x, weight, bias, m):
        B, C = x.shape[:2]
        xwin = m._window_input(x)
        X = m._pixels(m._ops.contract(xwin), B * C).view(B, m.groups, -1, m.nlat_out_local * m.nlon_out_local)
        y = torch.matmul(_grouped(weight.to(torch.float32), m.groups), X).view(B, weight.shape[0], m.nlat_out_local, m.nlon_out_local)
        if bias is not None:
            y = y + bias.to(torch.float32).view(1, -1, 1, 1)
        ctx.save_for_backward(xwin, weight)
        ctx.m, ctx.B, ctx.x_dtype, ctx.has_bias = m, B, x.dtype, bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        xwin, weight = ctx.saved_tensors
        m, B, G = ctx.m, ctx.B, ctx.m.groups
        C, K, P = m.in_channels, m.kernel_size, m.nlat_out_local * m.nlon_out_local
        gy = gy.to(torch.float32).contiguous()
        gyg = gy.view(B, G, -1, P)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dX = torch.matmul(_grouped(weight.to(torch.float32), G).transpose(1, 2), gyg).view(B * C, K, m.nlat_out_local, m.nlon_out_local)
            dx = m._pixels(m._window_adjoint(dX), B * C).view(B, C, m.nlat_in_local, m.nlon_in_local).to(ctx.x_dtype)
        if ctx.needs_input_grad[1]:
            X = m._pixels(m._ops.contract(xwin), B * C).view(B, G, -1, P)
            dw = torch.matmul(gyg, X.transpose(2, 3)).sum(0).reshape(weight.shape).to(weight.dtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = gy.sum(dim=(0, 2, 3))
        return dx, dw, db, None


class _SpatialGrid:
    """The h x w process grid of the distributed DISCO convolutions and the distributed neighbourhood attention: groups, split shapes, local
    shapes, the windows of a global DiscoPsi's output rows and the halo over its input rows, and the data movements around the per-rank
    stage.  The plan's output rows are the module's output latitudes, and for the transposed convolution (`_transpose`) its input latitudes."""

    def _init_grid(self, psi, ops_factory):
        """psi: the global DiscoPsi whose output rows are windowed; ops_factory(self) -> the per-rank stage (self._ops)"""
        from . import _rank, _size, azimuth_group, polar_group
        self.polar_group, self.azimuth_group = polar_group(), azimuth_group()
        self.comm_size_polar, self.comm_rank_polar = _size(self.polar_group), _rank(self.polar_group)
        self.comm_size_azimuth, self.comm_rank_azimuth = _size(self.azimuth_group), _rank(self.azimuth_group)
        h, w = self.comm_size_polar, self.comm_size_azimuth
        self.lat_in_shapes, self.lon_in_shapes = compute_split_shapes(self.nlat_in, h), compute_split_shapes(self.nlon_in, w)
        self.lat_out_shapes, self.lon_out_shapes = compute_split_shapes(self.nlat_out, h), compute_split_shapes(self.nlon_out, w)
        if min(self.lat_in_shapes + self.lat_out_shapes) < 1 or min(self.lon_in_shapes + self.lon_out_shapes) < 1:
            raise ValueError(f"grids {(self.nlat_in, self.nlon_in)} -> {(self.nlat_out, self.nlon_out)} are too small for {h} x {w} ranks")
        self.nlat_in_local, self.nlon_in_local = self.lat_in_shapes[self.comm_rank_polar], self.lon_in_shapes[self.comm_rank_azimuth]
        self.nlat_out_local, self.nlon_out_local = self.lat_out_shapes[self.comm_rank_polar], self.lon_out_shapes[self.comm_rank_azimuth]
        if self._transpose:
            window_lat, halo_lat, self._window_lon, self._halo_lon = self.lat_in_shapes, self.lat_out_shapes, self.lon_in_shapes, self.lon_out_shapes
        else:
            window_lat, halo_lat, self._window_lon, self._halo_lon = self.lat_out_shapes, self.lat_in_shapes, self.lon_out_shapes, self.lon_in_shapes
        self._halo_rows = halo_lat[self.comm_rank_polar]
        self.windows = disco_windows(psi, window_lat)
        self.window = self.windows[self.comm_rank_polar]
        self._halo_send, self._halo_recv = halo_plan(self.windows, halo_lat, self.comm_rank_polar)
        self._ops = ops_factory(self)

    def extra_repr(self):
        return super().extra_repr() + f", h={self.comm_size_polar}, w={self.comm_size_azimuth}"

    def _window_rows(self, r):
        """r (B*C, local rows, local longitudes, ...) on the plan's input grid -> (rows of B*C on this azimuth rank, hi - lo, all longitudes,
        ...): the rows of this rank's window"""
        if self.comm_size_azimuth > 1:
            r = _a2a(r, 0, 2, self._halo_lon, self.azimuth_group)
        g = halo_exchange(r.reshape(r.shape[0], r.shape[1], -1), self._halo_send, self._halo_recv, self.polar_group)
        return g.view(g.shape[0], g.shape[1], *r.shape[2:])

    def _window_rows_adjoint(self, g, BC):
        """the adjoint of _window_rows: g (rows of B*C on this azimuth rank, hi - lo, all longitudes, ...) -> (B*C, local rows, local
        longitudes, ...), the window rows returned to their owners and added in rank order"""
        d = halo_adjoint(g.reshape(g.shape[0], g.shape[1], -1), self._halo_send, self._halo_recv, self._halo_rows, self.polar_group)
        d = d.view(g.shape[0], self._halo_rows, *g.shape[2:])
        return _a2a(d, 2, 0, compute_split_shapes(BC, self.comm_size_azimuth), self.azimuth_group) if self.comm_size_azimuth > 1 else d

    def _window_adjoint(self, dX):
        """dX (B*C, K, local rows, local longitudes) on the plan's output grid -> (rows of B*C on this azimuth rank, local rows, all
        longitudes) on its input grid: the window adjoint, its rows returned to their owners and added in rank order"""
        if self.comm_size_azimuth > 1:
            dX = _a2a(dX, 0, 3, self._window_lon, self.azimuth_group)
        return halo_adjoint(self._ops.adjoint(dX).to(torch.float32), self._halo_send, self._halo_recv, self._halo_rows, self.polar_group)

    def _pixels(self, X, BC):
        """X (rows of this azimuth rank, ..., all longitudes) -> (B*C, ..., the longitudes of this rank) fp32"""
        X = X.to(torch.float32)
        return _a2a(X, X.dim() - 1, 0, compute_split_shapes(BC, self.comm_size_azimuth), self.azimuth_group) if self.comm_size_azimuth > 1 else X


def _refuse_one_rank(name, serial_name, what="the distributed DISCO convolution"):
    from . import _size, azimuth_group, polar_group
    if _size(polar_group()) * _size(azimuth_group()) == 1:
        raise NotImplementedError(f"{name} needs a process grid of more than one rank ({what} "
                                  "splits latitudes over makani_b200.distributed.polar_group() and longitudes over "
                                  f"azimuth_group()); at spatial model parallelism 1 use {serial_name}")


class DistributedDiscreteContinuousConvS2(_SpatialGrid, DiscreteContinuousConvS2):
    """DISCO convolution under h x w spatial model parallelism: the constructor, attributes, weight (C_out, C_in / groups, K) and bias of
    DiscreteContinuousConvS2, not sharded (makani tags them is_shared_mp = ["spatial"] and all-reduces their gradients).  The groups are
    makani_b200.distributed.polar_group() (latitudes) and azimuth_group() (longitudes), read at construction; a grid of one rank is refused."""

    def __init__(self, in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type="piecewise linear", basis_norm_mode="mean",
                 groups=1, grid_in="equiangular", grid_out="equiangular", bias=True, theta_cutoff=None):
        _refuse_one_rank("DistributedDiscreteContinuousConvS2", "DiscreteContinuousConvS2")
        super().__init__(in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type, basis_norm_mode, groups, grid_in, grid_out,
                         bias, theta_cutoff)
        self._init_grid(get_psi(*self._key), _OPS_FACTORY)

    def _window_input(self, x):
        """x (B, C, nlat_in_local, nlon_in_local) -> (rows of B*C on this azimuth rank, hi - lo, nlon_in)"""
        B, C = x.shape[:2]
        return self._window_rows(x.reshape(B * C, self.nlat_in_local, self.nlon_in_local))

    def forward(self, x):
        want = (self.in_channels, self.nlat_in_local, self.nlon_in_local)
        if x.dim() != 4 or tuple(x.shape[1:]) != want:
            raise ValueError(f"expected the local shard (B, {want[0]}, {want[1]}, {want[2]}), got {tuple(x.shape)}")
        if x.shape[0] * self.in_channels < self.comm_size_azimuth:
            raise ValueError(f"B * C_in = {x.shape[0] * self.in_channels} rows cannot be split over {self.comm_size_azimuth} azimuth ranks")
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.to(torch.float32)
        return _DistDiscoConv.apply(x.contiguous(), self.weight, self.bias, self)


class _DistDiscoConvTranspose(torch.autograd.Function):
    """y = the window adjoint of Y (+ bias), Y = the K-fold channel mix of x on the local pixels.  Saves x and W only."""

    @staticmethod
    def forward(ctx, x, weight, bias, m):
        B, C_out, G = x.shape[0], weight.shape[0], m.groups
        Y = torch.matmul(_transposed_mix(weight.to(torch.float32), G), x.to(torch.float32).view(B, G, -1, m.nlat_in_local * m.nlon_in_local))
        g = m._window_adjoint(Y.view(B * C_out, m.kernel_size, m.nlat_in_local, m.nlon_in_local))
        y = m._pixels(g, B * C_out).view(B, C_out, m.nlat_out_local, m.nlon_out_local)
        if bias is not None:
            y = y + bias.to(torch.float32).view(1, -1, 1, 1)
        ctx.save_for_backward(x, weight)
        ctx.m, ctx.has_bias = m, bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        m, G = ctx.m, ctx.m.groups
        B, C_out, P = x.shape[0], weight.shape[0], m.nlat_in_local * m.nlon_in_local
        gy = gy.to(torch.float32).contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            gwin = m._window_rows(gy.view(B * C_out, m.nlat_out_local, m.nlon_out_local))
            gY = m._pixels(m._ops.contract(gwin), B * C_out).view(B, G, -1, P)                   # (B, G, C_out/G * K, local pixels)
            Wt = _transposed_mix(weight.to(torch.float32), G)
        if ctx.needs_input_grad[0]:
            dx = torch.matmul(Wt.transpose(1, 2), gY).view(x.shape).to(x.dtype)
        if ctx.needs_input_grad[1]:
            dWt = torch.matmul(gY, x.to(torch.float32).view(B, G, -1, P).transpose(2, 3)).sum(0)   # (G, C_out/G * K, C_in/G)
            dw = dWt.view(G, -1, m.kernel_size, m.groupsize).transpose(2, 3).reshape(weight.shape).to(weight.dtype)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = gy.sum(dim=(0, 2, 3))
        return dx, dw, db, None


class DistributedDiscreteContinuousConvTransposeS2(_SpatialGrid, DiscreteContinuousConvTransposeS2):
    """Transposed DISCO convolution under h x w spatial model parallelism: the constructor, attributes, weight and bias of
    DiscreteContinuousConvTransposeS2, not sharded; x local (B, C_in, lat_in_shapes[ih], lon_in_shapes[iw]) -> y local
    (B, C_out, lat_out_shapes[ih], lon_out_shapes[iw]) float32.

        forward : grouped GEMM on the local pixels -> [w-a2a lon <-> rows of B*C_out] -> window adjoint (windows of the in-grid rows)
                  -> [h halo adjoint over the out-grid rows, fixed rank order] -> [w-a2a rows <-> lon] (+ bias)
        backward: [w-a2a] -> [h halo] -> window contraction -> [w-a2a] -> GEMM^T (dx) and local partial sums (dW, dbias)

    the backward chain of DistributedDiscreteContinuousConvS2 run as the forward, and its forward chain as the backward.  A grid of one rank is
    refused."""

    def __init__(self, in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type="piecewise linear", basis_norm_mode="mean",
                 groups=1, grid_in="equiangular", grid_out="equiangular", bias=True, theta_cutoff=None):
        _refuse_one_rank("DistributedDiscreteContinuousConvTransposeS2", "DiscreteContinuousConvTransposeS2")
        super().__init__(in_channels, out_channels, in_shape, out_shape, kernel_shape, basis_type, basis_norm_mode, groups, grid_in, grid_out,
                         bias, theta_cutoff)
        self._init_grid(get_psi(*self._key), _OPS_FACTORY)

    def forward(self, x):
        want = (self.in_channels, self.nlat_in_local, self.nlon_in_local)
        if x.dim() != 4 or tuple(x.shape[1:]) != want:
            raise ValueError(f"expected the local shard (B, {want[0]}, {want[1]}, {want[2]}), got {tuple(x.shape)}")
        if x.shape[0] * self.out_channels < self.comm_size_azimuth:
            raise ValueError(f"B * C_out = {x.shape[0] * self.out_channels} rows cannot be split over {self.comm_size_azimuth} azimuth ranks")
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.to(torch.float32)
        return _DistDiscoConvTranspose.apply(x.contiguous(), self.weight, self.bias, self)

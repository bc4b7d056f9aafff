"""DistributedNeighborhoodAttentionS2 -- NeighborhoodAttentionS2 under h x w spatial model parallelism, on the sm_90a kernels of
csrc/attention.cu run on per-rank window plans of the neighbourhood.

    query local (B, C_in, lat_out_shapes[ih], lon_out_shapes[iw]), key / value local (B, C_in, lat_in_shapes[ih], lon_in_shapes[iw])
    -> out local (B, C_v, lat_out_shapes[ih], lon_out_shapes[iw]) float32

    forward : 1x1 projections on the local pixels -> (B*H, rows, local lon, E) -> [w-a2a (b, h) pairs <-> lon]
              -> [h halo of k and v: input rows lo .. hi of this rank's window] -> attention on the window plan (heads = 1, B = local pairs)
              -> [w-a2a lon <-> pairs] -> output projection on the local pixels
    backward: autograd through the transposes; the query-side and key/value-side kernels on the window plan; the halo's adjoint returns the
              window rows of dk and dv to their owners and adds them in fixed rank order; parameter gradients are local partial sums

The neighbourhood is a K = 1 DiscoPsi, so the windows, the halo plan and the data movements are those of the distributed DISCO convolution
(distributed/disco.py, `_SpatialGrid`).  The window plan holds the global neighbourhood's entries of this rank's output rows in the same (i, j)
order, input rows re-indexed to i - lo, and each (b, h) pair is one CTA's work at any layout: y, lse, D and dq of every rank are bit-identical
to the corresponding slice of the single-GPU kernels' outputs, and so are dk and dv of the input rows that only one rank's output rows reach.
The per-rank stage is replaceable (`set_attention_local_ops`) so the choreography is unit-tested on CPU with gloo against the serial oracle.

DistributedAttentionS2 -- AttentionS2 (global attention) under the same h x w grid, on the kernels of csrc/attention_global.cu: each rank
attends with its own queries to every key, gathered in global order, and its backward runs the query-side and key-side passes of the kernels
on different query and key sets (see the class docstring).  Its per-rank stage is replaceable the same way (`set_global_attention_local_ops`).
"""
import torch
import torch.distributed as dist

from .._lib import B200ShtError
from ..attention import (AttentionPlan, AttentionS2, NeighborhoodAttentionS2, _global_precision, _NeighborhoodAttention, _project_channels,
                         _project_out, _project_points, get_neighbourhood, global_attention_backward_kv, global_attention_backward_q,
                         global_attention_forward, global_attention_rowdot)
from .disco import _refuse_one_rank, _SpatialGrid, window_plan
from .primitives import _DistributedTranspose, compute_split_shapes


class CudaAttentionLocalOps:
    """The window attention on the kernels of csrc/attention.cu, on an AttentionPlan of `layer.window` (cached per neighbourhood key,
    window and device).  `layer` has `_key` (the neighbourhood key of makani_b200.attention) and `window` (a DiscoWindow of the
    neighbourhood).  Has the forward_attention / backward_attention of AttentionPlan, so _NeighborhoodAttention takes it as its plan."""

    def __init__(self, layer):
        self.key, self.window = layer._key, layer.window

    def _plan(self, device):
        return window_plan(AttentionPlan, self.key, self.window, device, "the neighbourhood attention")

    def forward_attention(self, q, k, v, heads, scale):
        """q (R, (t1 - t0) nlon_out, heads E_k), k (R, (hi - lo) nlon_in, heads E_k), v (R, (hi - lo) nlon_in, heads E_v) fp32 contiguous
        -> y (R, (t1 - t0) nlon_out, heads E_v), lse (R, heads, (t1 - t0) nlon_out)"""
        return self._plan(q.device).forward_attention(q, k, v, heads, scale)

    def backward_attention(self, q, k, v, y, lse, dy, heads, scale):
        """-> dq, dk, dv (shapes of q, k, v)"""
        return self._plan(q.device).backward_attention(q, k, v, y, lse, dy, heads, scale)


_OPS_FACTORY = CudaAttentionLocalOps


def set_attention_local_ops(factory):
    """Replace the per-rank stage (tests: a CPU implementation on the oracle).  `factory(layer)` -> object with
    forward_attention(q, k, v, heads, scale) and backward_attention(q, k, v, y, lse, dy, heads, scale) as CudaAttentionLocalOps; None restores
    the CUDA stage."""
    global _OPS_FACTORY
    _OPS_FACTORY = factory if factory is not None else CudaAttentionLocalOps


class _WindowRows(torch.autograd.Function):
    """(B*H, local rows, local longitudes, E) -> (pairs of this azimuth rank, hi - lo, all longitudes, E): the rows of this rank's window.
    backward: the adjoint, window rows returned to their owners and added in rank order, then the inverse all-to-all."""

    @staticmethod
    def forward(ctx, x, m):
        ctx.m, ctx.BH = m, x.shape[0]
        return m._window_rows(x)

    @staticmethod
    def backward(ctx, g):
        return ctx.m._window_rows_adjoint(g.contiguous(), ctx.BH), None


class DistributedNeighborhoodAttentionS2(_SpatialGrid, NeighborhoodAttentionS2):
    """Neighbourhood attention under h x w spatial model parallelism: the constructor, attributes and parameters of NeighborhoodAttentionS2,
    not sharded (tagged is_shared_mp = ["spatial"]: the gradients are local partial sums, all-reduced over the spatial ranks by the caller).
    The groups are makani_b200.distributed.polar_group() (latitudes) and azimuth_group() (longitudes), read at construction; a grid of one
    rank is refused.  The (b, h) pairs are split over the azimuth ranks, so B * num_heads must be at least the azimuth group's size."""

    _transpose = False

    def __init__(self, in_channels, in_shape, out_shape, grid_in="equiangular", grid_out="equiangular", num_heads=1, scale=None, bias=True,
                 theta_cutoff=None, k_channels=None, out_channels=None, optimized_kernel=True):
        _refuse_one_rank("DistributedNeighborhoodAttentionS2", "NeighborhoodAttentionS2", "the distributed neighbourhood attention")
        super().__init__(in_channels, in_shape, out_shape, grid_in, grid_out, num_heads, scale, bias, theta_cutoff, k_channels, out_channels,
                         optimized_kernel)
        for p in self.parameters():
            p.is_shared_mp = ["spatial"]
            p.sharded_dims_mp = [None] * p.dim()
        self._init_grid(get_neighbourhood(*self._key), _OPS_FACTORY)

    def _check_local(self, x, rows, lons, what):
        if x.dim() != 4 or tuple(x.shape[1:]) != (self.in_channels, rows, lons):
            raise ValueError(f"{what}: expected the local shard (B, {self.in_channels}, {rows}, {lons}), got {tuple(x.shape)}")

    def _pairs(self, x, weight, bias, rows, lons):
        """the projection of x (B, C_in, rows, lons) on its pixels -> (B*H, rows, lons, E), each (b, h) pair contiguous"""
        B, H = x.shape[0], self.num_heads
        p = _project_points(x, weight, bias)                                                       # (B, rows lons, H E)
        return p.view(B, rows, lons, H, -1).permute(0, 3, 1, 2, 4).reshape(B * H, rows, lons, -1)

    def forward(self, query, key=None, value=None):
        if (key is None or value is None) and (self.nlat_in, self.nlon_in) != (self.nlat_out, self.nlon_out):
            raise ValueError("key and value default to query, which needs in_shape == out_shape")
        key = query if key is None else key
        value = query if value is None else value
        self._check_local(query, self.nlat_out_local, self.nlon_out_local, "query")
        self._check_local(key, self.nlat_in_local, self.nlon_in_local, "key")
        self._check_local(value, self.nlat_in_local, self.nlon_in_local, "value")
        if key.shape[0] != query.shape[0] or value.shape[0] != query.shape[0]:
            raise ValueError("query, key and value must have the same batch size")
        B, H, w = query.shape[0], self.num_heads, self.comm_size_azimuth
        if B * H < w:
            raise ValueError(f"B * num_heads = {B * H} (b, h) pairs cannot be split over {w} azimuth ranks")
        q = self._pairs(query, self.q_weights, self.q_bias, self.nlat_out_local, self.nlon_out_local)
        k = self._pairs(key, self.k_weights, self.k_bias, self.nlat_in_local, self.nlon_in_local)
        v = self._pairs(value, self.v_weights, self.v_bias, self.nlat_in_local, self.nlon_in_local)
        if w > 1:
            q = _DistributedTranspose.apply(q, (0, 2), self.lon_out_shapes, self.azimuth_group)     # (pairs, local rows, nlon_out, E_k)
        k, v = _WindowRows.apply(k, self), _WindowRows.apply(v, self)                               # (pairs, hi - lo, nlon_in, E)
        R = q.shape[0]
        y = _NeighborhoodAttention.apply(q.reshape(R, -1, q.shape[3]), k.reshape(R, -1, k.shape[3]), v.reshape(R, -1, v.shape[3]), self._ops,
                                         1, self.scale)
        y = y.view(R, self.nlat_out_local, self.nlon_out, -1)
        if w > 1:
            y = _DistributedTranspose.apply(y, (2, 0), compute_split_shapes(B * H, w), self.azimuth_group)   # (B*H, local rows, local lon, E_v)
        P = self.nlat_out_local * self.nlon_out_local
        y = y.view(B, H, P, -1).transpose(1, 2).reshape(B, P, -1)                                  # (B, local pixels, H E_v)
        return _project_out(y, self.proj_weights, self.proj_bias).view(B, self.out_channels, self.nlat_out_local, self.nlon_out_local)


# ------------------------------------------------------------------------------------------------------------------- global attention
class CudaGlobalAttentionLocalOps:
    """The per-rank stage of DistributedAttentionS2 on the kernels of csrc/attention_global.cu: the forward and the three stages of the
    backward (makani_b200.attention.global_attention_*), on fp32 contiguous CUDA tensors."""

    def __init__(self, layer):
        pass

    @staticmethod
    def _cuda(x):
        if not x.is_cuda:
            raise B200ShtError("DistributedAttentionS2 runs on CUDA devices only; makani_b200 has no CPU fallback")

    def forward(self, q, k, v, bias, scale, precision):
        """q (B, H, nq, E_k), k (B, H, nk, E_k), v (B, H, E_v, nk), bias (nk,) -> o (B, H, nq, E_v), lse (B, H, nq)"""
        self._cuda(q)
        return global_attention_forward(q, k, v, bias, scale, precision)

    def rowdot(self, o, do):
        """-> D (B, H, nq) = rowsum(do o)"""
        self._cuda(o)
        return global_attention_rowdot(o, do)

    def backward_q(self, q, k, v, bias, lse, D, do, scale, precision):
        """-> dq of the given queries against the given keys"""
        self._cuda(q)
        return global_attention_backward_q(q, k, v, bias, lse, D, do, scale, precision)

    def backward_kv(self, q, k, v, bias, lse, D, do, scale, precision):
        """-> dk, dv of the given keys against the given queries"""
        self._cuda(q)
        return global_attention_backward_kv(q, k, v, bias, lse, D, do, scale, precision)


_GLOBAL_OPS_FACTORY = CudaGlobalAttentionLocalOps


def set_global_attention_local_ops(factory):
    """Replace the per-rank stage of DistributedAttentionS2 (tests: a CPU implementation on the oracle).  `factory(layer)` -> object with
    forward / rowdot / backward_q / backward_kv as CudaGlobalAttentionLocalOps; None restores the CUDA stage.  Read at construction."""
    global _GLOBAL_OPS_FACTORY
    _GLOBAL_OPS_FACTORY = factory if factory is not None else CudaGlobalAttentionLocalOps


def _gather_dim(x, dim, shapes, group):
    """all_gather of x along `dim` over `group`, shard r of size shapes[r], concatenated in rank order.  Every shard is padded to the largest
    first, so the collective sees equal sizes (gloo's all_gather refuses uneven ones), and narrowed back after it."""
    n = max(shapes)
    if x.shape[dim] != n:
        pad = x.new_zeros(x.shape[:dim] + (n,) + x.shape[dim + 1:])
        pad.narrow(dim, 0, x.shape[dim]).copy_(x)
        x = pad
    x = x.contiguous()
    parts = [torch.empty_like(x) for _ in shapes]
    dist.all_gather(parts, x, group=group)
    return torch.cat([p.narrow(dim, 0, s) for p, s in zip(parts, shapes)], dim=dim)


class _DistGlobalAttention(torch.autograd.Function):
    """o_r = attention of this rank's queries q_r against every key, gathered in global order.  Inputs q_r (B, H, nq_r, E_k), k_r
    (B, H, nk_r, E_k), v_r (B, H, E_v, nk_r): the gathers happen inside, so they need no adjoint.  Saves the local q_r, k_r, v_r, o_r, lse_r.
    backward: dq_r against the re-gathered keys; dk_r, dv_r of this rank's keys against every query (Q, dO, lse, D gathered).  Nothing is
    summed across ranks."""

    @staticmethod
    def forward(ctx, q, k, v, m, bias, bias_local, precision):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        K, V = m._gather_keys(k, v)
        o, lse = m._ops.forward(q, K, V, bias, m.scale, precision)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.m, ctx.bias, ctx.bias_local, ctx.precision = m, bias, bias_local, precision
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        m, prec = ctx.m, ctx.precision
        do = do.to(torch.float32).contiguous()
        D = m._ops.rowdot(o, do)
        K, V = m._gather_keys(k, v)
        dq = m._ops.backward_q(q, K, V, ctx.bias, lse, D, do, m.scale, prec)
        del K, V
        Qg, dOg, lseg, Dg = (m._gather_out(t, 2) for t in (q, do, lse, D))
        dk, dv = m._ops.backward_kv(Qg, k, v, ctx.bias_local, lseg, Dg, dOg, m.scale, prec)
        return dq, dk, dv, None, None, None, None


class DistributedAttentionS2(AttentionS2):
    """Global attention on the sphere under h x w spatial model parallelism: the constructor, attributes, parameters, init and state dict of
    AttentionS2.  The parameters are not sharded (tagged is_shared_mp = ["spatial"]: their gradients are local partial sums, all-reduced
    over the spatial ranks by the caller).  The groups are makani_b200.distributed.polar_group() (latitudes) and azimuth_group() (longitudes),
    read at construction; a grid of one rank is refused.

        query local (B, C_in, lat_out_shapes[ih], lon_out_shapes[iw]), key / value local (B, C_in, lat_in_shapes[ih], lon_in_shapes[iw])
        -> out local (B, C_v, lat_out_shapes[ih], lon_out_shapes[iw]) float32

        forward : 1x1 projections on the local pixels -> all-gather of k and v in global (lat, lon) order (azimuth group along longitude,
                  then polar group along latitude) -> the attention of the local queries against every key -> output projection
        backward: D_r = rowsum(dO_r o_r) -> re-gather k, v -> dq_r (q pass) -> gather q, dO, lse, D over the output grid
                  -> dk_r, dv_r of the local keys against every query (kv pass)

    Each row of o, lse and dq depends only on its query and on all keys, each row of dk and dv only on its key and on all queries, visited in
    the same block order as on one GPU: every rank's outputs equal the matching slices of the single-GPU kernels' outputs bit for bit, with
    no reduction across ranks.  Only local tensors are saved for the backward."""

    def __init__(self, in_channels, num_heads, in_shape, out_shape, grid_in="equiangular", grid_out="equiangular", scale=None, bias=True,
                 k_channels=None, out_channels=None, drop_rate=0.0):
        from . import _rank, _size, azimuth_group, polar_group
        _refuse_one_rank("DistributedAttentionS2", "AttentionS2", "the distributed global attention")
        super().__init__(in_channels, num_heads, in_shape, out_shape, grid_in, grid_out, scale, bias, k_channels, out_channels, drop_rate)
        for p in self.parameters():
            p.is_shared_mp = ["spatial"]
            p.sharded_dims_mp = [None] * p.dim()
        self.polar_group, self.azimuth_group = polar_group(), azimuth_group()
        self.comm_size_polar, self.comm_rank_polar = _size(self.polar_group), _rank(self.polar_group)
        self.comm_size_azimuth, self.comm_rank_azimuth = _size(self.azimuth_group), _rank(self.azimuth_group)
        h, w = self.comm_size_polar, self.comm_size_azimuth
        self.lat_in_shapes, self.lon_in_shapes = compute_split_shapes(self.nlat_in, h), compute_split_shapes(self.nlon_in, w)
        self.lat_out_shapes, self.lon_out_shapes = compute_split_shapes(self.nlat_out, h), compute_split_shapes(self.nlon_out, w)
        if min(self.lat_in_shapes + self.lat_out_shapes) < 1 or min(self.lon_in_shapes + self.lon_out_shapes) < 1:
            raise ValueError(f"grids {(self.nlat_in, self.nlon_in)} -> {(self.nlat_out, self.nlon_out)} are too small for {h} x {w} ranks")
        ih, iw = self.comm_rank_polar, self.comm_rank_azimuth
        self.nlat_in_local, self.nlon_in_local = self.lat_in_shapes[ih], self.lon_in_shapes[iw]
        self.nlat_out_local, self.nlon_out_local = self.lat_out_shapes[ih], self.lon_out_shapes[iw]
        lat0, lon0 = sum(self.lat_in_shapes[:ih]), sum(self.lon_in_shapes[:iw])
        local = self.key_bias.view(self.nlat_in, self.nlon_in)[lat0:lat0 + self.nlat_in_local, lon0:lon0 + self.nlon_in_local]
        self.register_buffer("key_bias_local", local.reshape(-1).contiguous(), persistent=False)
        self._ops = _GLOBAL_OPS_FACTORY(self)

    def extra_repr(self):
        return super().extra_repr() + f", h={self.comm_size_polar}, w={self.comm_size_azimuth}"

    def _gather_grid(self, x, lat_dim, lat_shapes, lon_shapes):
        """x with this rank's (latitude, longitude) block at dims lat_dim, lat_dim + 1 -> the whole grid there, in global order: the azimuth
        gather along longitude, then the polar gather along latitude"""
        if self.comm_size_azimuth > 1:
            x = _gather_dim(x, lat_dim + 1, lon_shapes, self.azimuth_group)
        if self.comm_size_polar > 1:
            x = _gather_dim(x, lat_dim, lat_shapes, self.polar_group)
        return x

    def _gather_keys(self, k, v):
        """k_r (B, H, nk_r, E_k), v_r (B, H, E_v, nk_r) -> K (B, H, N_k, E_k), V (B, H, E_v, N_k), fp32 contiguous"""
        B, H, rows, lons = k.shape[0], k.shape[1], self.nlat_in_local, self.nlon_in_local
        K = self._gather_grid(k.view(B, H, rows, lons, -1), 2, self.lat_in_shapes, self.lon_in_shapes)
        V = self._gather_grid(v.view(B, H, -1, rows, lons), 3, self.lat_in_shapes, self.lon_in_shapes)
        return K.reshape(B, H, -1, K.shape[-1]).contiguous(), V.reshape(B, H, V.shape[2], -1).contiguous()

    def _gather_out(self, t, point_dim):
        """t with this rank's output points (row-major over its block) at dim point_dim -> every output point in global order"""
        shape = t.shape[:point_dim] + (self.nlat_out_local, self.nlon_out_local) + t.shape[point_dim + 1:]
        g = self._gather_grid(t.reshape(shape), point_dim, self.lat_out_shapes, self.lon_out_shapes)
        return g.reshape(t.shape[:point_dim] + (-1,) + t.shape[point_dim + 1:]).contiguous()

    def _check_local(self, x, rows, lons, what):
        if x.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"{what}: float32 or bfloat16 inputs are served, got {x.dtype}")
        if x.dim() != 4 or tuple(x.shape[1:]) != (self.in_channels, rows, lons):
            raise ValueError(f"{what}: expected the local shard (B, {self.in_channels}, {rows}, {lons}), got {tuple(x.shape)}")

    def forward(self, query, key=None, value=None):
        if (key is None or value is None) and (self.nlat_in, self.nlon_in) != (self.nlat_out, self.nlon_out):
            raise ValueError("key and value default to query, which needs in_shape == out_shape")
        if self.training and self.drop_rate > 0.0:
            raise NotImplementedError("DistributedAttentionS2: attention dropout (drop_rate > 0 in training) is not implemented")
        key = query if key is None else key
        value = query if value is None else value
        self._check_local(query, self.nlat_out_local, self.nlon_out_local, "query")
        self._check_local(key, self.nlat_in_local, self.nlon_in_local, "key")
        self._check_local(value, self.nlat_in_local, self.nlon_in_local, "value")
        if key.shape[0] != query.shape[0] or value.shape[0] != query.shape[0]:
            raise ValueError("query, key and value must have the same batch size")
        B, H = query.shape[0], self.num_heads
        ek, ev = self.k_channels // H, self.out_channels // H
        nq, nk = self.nlat_out_local * self.nlon_out_local, self.nlat_in_local * self.nlon_in_local
        q = _project_channels(query, self.q_weights, self.q_bias).view(B, H, ek, nq).transpose(2, 3)   # (B, H, nq_r, ek)
        k = _project_channels(key, self.k_weights, self.k_bias).view(B, H, ek, nk).transpose(2, 3)
        v = _project_channels(value, self.v_weights, self.v_bias).view(B, H, ev, nk)
        o = _DistGlobalAttention.apply(q, k, v, self, self.key_bias.to(query.device), self.key_bias_local.to(query.device),
                                       _global_precision())                                                # (B, H, nq_r, ev)
        y = o.transpose(2, 3).reshape(B, self.out_channels, nq)
        wp = self.proj_weights.to(torch.float32).reshape(self.out_channels, self.out_channels).expand(B, -1, -1)
        out = torch.bmm(wp, y) if self.proj_bias is None else torch.baddbmm(self.proj_bias.to(torch.float32).view(1, -1, 1).expand(B, -1, nq), wp, y)
        return out.view(B, self.out_channels, self.nlat_out_local, self.nlon_out_local)

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
"""
import torch

from ..attention import AttentionPlan, NeighborhoodAttentionS2, _NeighborhoodAttention, _project_out, _project_points, get_neighbourhood
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

"""DistributedGeometricInstanceNormS2 -- makani's quadrature-weighted instance norm under h x w spatial model parallelism
(makani/mpu/layer_norm.py:173-253), on the kernels of csrc/norm.cu.

    x local (B, C, crop_h_shapes[ih], crop_w_shapes[iw]) -> y local, same shape and dtype

    forward : this shard's fp64 (sum q, mean, M2) per (b, c) -> all-gather over the azimuth group, then the polar group: every rank holds the same
              [h][w] array -> Chan / Welford combine in that fixed order (`finalize`), so the statistics are bit-identical on every rank -> apply
    backward: this shard's fp64 (S1, S2) -> the same gather -> dx;  dgamma / dbeta are this rank's partial sums (`is_shared_mp = ["spatial"]`,
              as makani: its gradient hooks add them up over the spatial group)

Each rank's weights are its `compute_split_shapes` slice of the global crop; the normaliser D is the total weight of the global crop, so the
statistics are those of the whole crop (makani's Welford form).  A 1 x 1 grid runs the same stages with nothing to gather.  The per-rank stage is
replaceable (`set_norm_local_ops`) so the choreography is unit-tested on CPU with gloo against the serial oracle.

DistributedInstanceNorm2d (makani/mpu/layer_norm.py:108-170, SFNO's default `instance_norm` under h x w) is the same formula with every latitude
weight q = 1 and D = the point count of the global field, so it runs the same stages and the same gather.  makani's layer knows no image shape:
D is the sum of every rank's H_loc * W_loc, exchanged once per distinct local shape and cached, so later calls copy nothing to the host.
"""
import torch
import torch.distributed as dist
import torch.nn as nn

from ..norm import _CUDA_STAGES, _TORCH_STAGES, GeometricInstanceNormS2, _GeometricNormFn, _usable
from .primitives import compute_split_shapes

_OPS_FACTORY = None


def set_norm_local_ops(factory):
    """Replace the per-rank stage (tests: a CPU implementation on the oracle).  `factory(layer)` -> object with partials / finalize / apply /
    backward_sums / backward_apply / param_grads as makani_b200.norm.CudaGeometricNormStages; None restores the default (the kernels for the inputs they take,
    torch operators otherwise)."""
    global _OPS_FACTORY
    _OPS_FACTORY = factory


def _all_gather_stack(t, group):
    from . import _size
    if _size(group) == 1:
        return t.unsqueeze(0)
    parts = [torch.empty_like(t) for _ in range(_size(group))]
    dist.all_gather(parts, t.contiguous(), group=group)
    return torch.stack(parts, dim=0)


def _gather_grid(t):
    """this rank's per-row tensor -> every rank's, [h * w][...] in (polar rank, azimuth rank) order on every rank"""
    from . import azimuth_group, polar_group
    tw = _all_gather_stack(t, azimuth_group())               # [w][...]
    th = _all_gather_stack(tw, polar_group())                # [h][w][...]
    return th.reshape(-1, *t.shape)


class DistributedGeometricInstanceNormS2(GeometricInstanceNormS2):
    """Same constructor, parameters and state dict as GeometricInstanceNormS2 (and makani's class); the input is this rank's shard of the crop."""

    def __init__(self, img_shape, crop_shape, crop_offset, grid_type, num_features, eps=1e-05, affine=False):
        from . import azimuth_group_rank, azimuth_group_size, polar_group_rank, polar_group_size

        super().__init__(img_shape, crop_shape, crop_offset, grid_type, num_features, eps=eps, affine=affine)
        if self.affine:
            self.weight.is_shared_mp = ["spatial"]
            self.bias.is_shared_mp = ["spatial"]
        h_shapes = compute_split_shapes(self.crop_shape[0], polar_group_size())
        w_shapes = compute_split_shapes(self.crop_shape[1], azimuth_group_size())
        self.comm_size_polar, self.comm_size_azimuth = polar_group_size(), azimuth_group_size()
        self._init_quadrature(h_shapes, polar_group_rank(), w_shapes[azimuth_group_rank()])
        # D: the weight of the whole global crop, from the float32 weights the kernels read, summed in fp64 the same way on every rank
        from ..quadrature import crop_quadrature_np
        q_crop = crop_quadrature_np(self.grid_type, self.img_shape, self.crop_shape, self.crop_offset).astype("float32").astype("float64")
        self._D = float(q_crop.sum() * self.crop_shape[1])
        self._ops = _OPS_FACTORY(self) if _OPS_FACTORY is not None else None

    def _normaliser(self):
        return self._D

    def _gather(self):
        return _gather_grid

    def _stages(self, x):
        if self._ops is not None:
            return self._ops
        return super()._stages(x)

    def extra_repr(self):
        return f"crop={self.crop_shape}, local={self.local_shape}, grid={self.grid_type}, h={self.comm_size_polar}, w={self.comm_size_azimuth}"


class DistributedInstanceNorm2d(nn.Module):
    """makani's DistributedInstanceNorm2d (same constructor, parameters `weight` / `bias` tagged `is_shared_mp = ["spatial"]`, state dict): instance
    norm of this rank's shard (B, C, H_loc, W_loc) with the statistics of the global field, computed in fp32 with autocast off and returned in the
    dtype of the input.  CUDA float32 / bfloat16 inputs run on the kernels of csrc/norm.cu, other inputs on the same stages in torch operators."""

    def __init__(self, num_features, eps=1e-05, affine=False):
        from . import azimuth_group_size, polar_group_size

        super().__init__()
        self.num_features, self.eps, self.affine = num_features, eps, affine
        if self.affine:
            self.weight = nn.Parameter(torch.ones(num_features))
            self.bias = nn.Parameter(torch.zeros(num_features))
            self.weight.is_shared_mp = ["spatial"]
            self.bias.is_shared_mp = ["spatial"]
        self.comm_size_polar, self.comm_size_azimuth = polar_group_size(), azimuth_group_size()
        self._points = {}       # (H_loc, W_loc) -> D, the point count of the global field
        self._ones = {}         # (H_loc, device) -> fp32 ones, the latitude weights
        self._ops = _OPS_FACTORY(self) if _OPS_FACTORY is not None else None

    def _normaliser(self, x):
        """D = sum over every rank of H_loc * W_loc: one exchange per distinct local shape (every rank meets a new shape in the same call)"""
        key = tuple(x.shape[-2:])
        D = self._points.get(key)
        if D is None:
            n = torch.tensor([float(key[0] * key[1])], dtype=torch.float64, device=x.device)
            D = self._points[key] = float(_gather_grid(n).sum())
        return D

    def _q(self, x):
        key = (x.shape[-2], x.device)
        q = self._ones.get(key)
        if q is None:
            q = self._ones[key] = torch.ones(x.shape[-2], dtype=torch.float32, device=x.device)
        return q

    def _stages(self, x):
        if self._ops is not None:
            return self._ops
        return _CUDA_STAGES if _usable(x) and (self.weight.is_cuda if self.affine else True) else _TORCH_STAGES

    def forward(self, x):
        if x.dim() != 4 or (self.affine and x.shape[1] != self.num_features):
            raise ValueError(f"expected input of shape (B, {self.num_features}, H_local, W_local), got {tuple(x.shape)}")
        w, b = (self.weight, self.bias) if self.affine else (None, None)
        with torch.autocast(device_type=x.device.type, enabled=False):
            return _GeometricNormFn.apply(x, w, b, self._q(x), self._normaliser(x), self.eps, False, self._stages(x), _gather_grid)

    def extra_repr(self):
        return f"{self.num_features}, eps={self.eps}, affine={self.affine}, h={self.comm_size_polar}, w={self.comm_size_azimuth}"


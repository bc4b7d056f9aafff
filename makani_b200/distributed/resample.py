"""DistributedResampleS2 -- `torch_harmonics.distributed.DistributedResampleS2` as makani builds it at spatial model parallelism > 1 (FCN3's and
SNO's `DiscreteContinuousDecoder` with upsample_sht=False), on the sm_90a kernels of csrc/resample.cu.

    x local (..., lat_in_shapes[ih], lon_in_shapes[iw]) float32 -> y local (..., lat_out_shapes[ih], lon_out_shapes[iw]) float32

    planes -> [h-a2a planes <-> lat] -> [w-a2a planes <-> lon] -> forward kernel on whole spheres (the serial plan) -> [w-a2a] -> [h-a2a]

Every plane is resampled on its own, so the forward and the input gradient (autograd through the transposes and the adjoint kernel) are
bit-identical to the single-GPU module.  The resampling is about 1 % of the decoder step (DESIGN.md section 9): a latitude halo, as in the
distributed DISCO convolution, would not repay its code.  The per-rank stages are replaceable (`set_resample_local_ops`).
"""
import math

import torch

from .._lib import B200ShtError
from ..resample import ResampleS2, _Resample, get_plan
from .primitives import _DistributedTranspose, compute_split_shapes


class CudaResampleLocalOps:
    """The forward and adjoint kernels on the serial plan of `layer._key` (the `plan` interface that `_Resample` drives)."""

    def __init__(self, layer):
        self.key = layer._key

    def forward(self, x):
        """x (planes, nlat_in, nlon_in) fp32 -> (planes, nlat_out, nlon_out)"""
        return get_plan(self.key, x.device).forward(x)

    def adjoint(self, dy):
        """dy (planes, nlat_out, nlon_out) fp32 -> (planes, nlat_in, nlon_in)"""
        return get_plan(self.key, dy.device).adjoint(dy)


_OPS_FACTORY = CudaResampleLocalOps


def set_resample_local_ops(factory):
    """Replace the per-rank stages (tests: a CPU implementation on the oracle).  `factory(layer)` -> object with forward(x) and adjoint(dy) as
    CudaResampleLocalOps; None restores the CUDA stages."""
    global _OPS_FACTORY
    _OPS_FACTORY = factory if factory is not None else CudaResampleLocalOps


class DistributedResampleS2(ResampleS2):
    """Bilinear resampling under h x w spatial model parallelism: the constructor and attributes of ResampleS2 (fp32 only).  The groups are
    makani_b200.distributed.polar_group() and azimuth_group(), read at construction; a grid of one rank is refused."""

    def __init__(self, nlat_in, nlon_in, nlat_out, nlon_out, grid_in="equiangular", grid_out="equiangular", mode="bilinear"):
        from . import _rank, _size, azimuth_group, polar_group
        if _size(polar_group()) * _size(azimuth_group()) == 1:
            raise NotImplementedError("DistributedResampleS2 needs a process grid of more than one rank (the distributed resampling splits "
                                      "latitudes over makani_b200.distributed.polar_group() and longitudes over azimuth_group()); at spatial "
                                      "model parallelism 1 use ResampleS2")
        super().__init__(nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out, mode)
        self.polar_group, self.azimuth_group = polar_group(), azimuth_group()
        self.comm_size_polar, self.comm_rank_polar = _size(self.polar_group), _rank(self.polar_group)
        self.comm_size_azimuth, self.comm_rank_azimuth = _size(self.azimuth_group), _rank(self.azimuth_group)
        h, w = self.comm_size_polar, self.comm_size_azimuth
        self.lat_in_shapes, self.lon_in_shapes = compute_split_shapes(nlat_in, h), compute_split_shapes(nlon_in, w)
        self.lat_out_shapes, self.lon_out_shapes = compute_split_shapes(nlat_out, h), compute_split_shapes(nlon_out, w)
        if min(self.lat_in_shapes + self.lat_out_shapes) < 1 or min(self.lon_in_shapes + self.lon_out_shapes) < 1:
            raise ValueError(f"grids ({nlat_in}, {nlon_in}) -> ({nlat_out}, {nlon_out}) are too small for {h} x {w} ranks")
        self.nlat_in_local, self.nlon_in_local = self.lat_in_shapes[self.comm_rank_polar], self.lon_in_shapes[self.comm_rank_azimuth]
        self.nlat_out_local, self.nlon_out_local = self.lat_out_shapes[self.comm_rank_polar], self.lon_out_shapes[self.comm_rank_azimuth]
        self._ops = _OPS_FACTORY(self)

    def extra_repr(self):
        return super().extra_repr() + f", h={self.comm_size_polar}, w={self.comm_size_azimuth}"

    def forward(self, x):
        if self.skip_resampling:
            return x
        if x.dim() < 2 or tuple(x.shape[-2:]) != (self.nlat_in_local, self.nlon_in_local):
            raise ValueError(f"expected the local shard (..., {self.nlat_in_local}, {self.nlon_in_local}), got {tuple(x.shape)}")
        if x.dtype != torch.float32:
            raise B200ShtError(f"DistributedResampleS2 takes float32 input (got {x.dtype})")
        h, w = self.comm_size_polar, self.comm_size_azimuth
        lead = tuple(x.shape[:-2])
        planes = math.prod(lead)
        plane_shapes = compute_split_shapes(planes, h)
        if planes < h or min(plane_shapes) < w:
            raise ValueError(f"{planes} planes cannot be split over {h} x {w} ranks")
        y = x.contiguous().view(planes, self.nlat_in_local, self.nlon_in_local)
        if h > 1:
            y = _DistributedTranspose.apply(y, (0, 1), self.lat_in_shapes, self.polar_group)
        if w > 1:
            y = _DistributedTranspose.apply(y, (0, 2), self.lon_in_shapes, self.azimuth_group)
        y = _Resample.apply(y.contiguous(), self._ops)
        if w > 1:
            y = _DistributedTranspose.apply(y, (2, 0), compute_split_shapes(plane_shapes[self.comm_rank_polar], w), self.azimuth_group)
        if h > 1:
            y = _DistributedTranspose.apply(y, (1, 0), plane_shapes, self.polar_group)
        return y.reshape(lead + (self.nlat_out_local, self.nlon_out_local))

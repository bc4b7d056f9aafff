"""ResampleS2 -- drop-in for `torch_harmonics.ResampleS2(mode="bilinear")` as FCN3's and SNO's `DiscreteContinuousDecoder` build it with
upsample_sht=False (makani/models/networks/fourcastnet3.py:356-358, snonet.py), on the sm_90a kernels of csrc/resample.cu.

    ResampleS2(nlat_in, nlon_in, nlat_out, nlon_out, grid_in="equiangular", grid_out="equiangular", mode="bilinear")
    forward: x (..., nlat_in, nlon_in) float32 on a CUDA device -> (..., nlat_out, nlon_out) float32

The interpolation tables are built here on the host in fp64 from the colatitudes and longitudes of `makani_b200.quadrature` (`precompute_tables`,
the contract restated in include/b200sht.h and DESIGN.md section 4.8) and rounded to fp32 once.  Leading dimensions are flattened into planes;
the backward is the library's adjoint kernel.  Only mode "bilinear" is implemented; any other mode ("bilinear-spherical" included) raises
NotImplementedError.  Inputs that are not fp32 raise B200ShtError: makani's decoder calls the layer in fp32 with autocast off.
"""
import math
import threading
from collections import namedtuple

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import B200ShtError, launch_stream as _stream, ptr as _ptr
from .quadrature import precompute_latitudes, precompute_longitudes

# lat_idx / lat_w (nlat_out): expanded input rows a, a + 1 and weight of output row t; lon_left / lon_right / lon_w (nlon_out)
ResampleTables = namedtuple("ResampleTables", "lat_idx lat_w lon_left lon_right lon_w expand_poles")


def precompute_tables(nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out):
    """the bilinear tables in fp64, weights rounded to fp32, as ResampleTables (indices int64)"""
    lats_in = precompute_latitudes(nlat_in, grid_in)[0].numpy()
    lats_out = precompute_latitudes(nlat_out, grid_out)[0].numpy()
    expand = bool(np.any(lats_out < lats_in[0]) or np.any(lats_out > lats_in[-1]))
    if expand:
        lats_in = np.concatenate([[0.0], lats_in, [math.pi]])
    lat_idx = np.searchsorted(lats_in, lats_out, side="right") - 1
    lat_idx = np.where(lats_out == lats_in[-1], lat_idx - 1, lat_idx)
    lat_w = ((lats_out - lats_in[lat_idx]) / (lats_in[lat_idx + 1] - lats_in[lat_idx])).astype(np.float32)
    lons_in, lons_out = precompute_longitudes(nlon_in).numpy(), precompute_longitudes(nlon_out).numpy()
    left = np.searchsorted(lons_in, lons_out, side="right") - 1
    right = np.where(lons_out >= lons_in[-1], 0, left + 1)
    diff = lons_in[right] - lons_in[left]
    diff = np.where(diff < 0.0, diff + 2.0 * math.pi, diff)
    lon_w = ((lons_out - lons_in[left]) / diff).astype(np.float32)
    return ResampleTables(lat_idx.astype(np.int64), lat_w, left.astype(np.int64), right.astype(np.int64), lon_w, expand)


class ResamplePlan:
    """Owner of a b200sht_resample_plan (the tables and the adjoint's two CSR lists on the device)."""

    def __init__(self, nlat_in, nlon_in, nlat_out, nlon_out, tables, device):
        lib = _lib.load()
        self.device = torch.device(device)
        self.nlat_in, self.nlon_in, self.nlat_out, self.nlon_out = nlat_in, nlon_in, nlat_out, nlon_out
        i32 = lambda a: np.ascontiguousarray(a, dtype=np.int32)     # noqa: E731
        f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)   # noqa: E731
        lat_idx, lat_w, left, right, lon_w = i32(tables.lat_idx), f32(tables.lat_w), i32(tables.lon_left), i32(tables.lon_right), f32(tables.lon_w)
        h = _lib.c_void_p()
        _lib.call("b200sht_resample_plan_create", _lib.ctypes.byref(h), nlat_in, nlon_in, nlat_out, nlon_out, int(tables.expand_poles),
                  lat_idx.ctypes.data, lat_w.ctypes.data, left.ctypes.data, right.ctypes.data, lon_w.ctypes.data, _stream(self.device))
        self.handle, self._lib = h, lib

    def query(self, what):
        return int(self._lib.b200sht_resample_plan_query(self.handle, what))

    def __del__(self):
        h = getattr(self, "handle", None)
        if h is not None and h.value and getattr(self, "_lib", None) is not None:
            self._lib.b200sht_resample_plan_destroy(h)
            self.handle = None

    def forward(self, x):
        """x (planes, nlat_in, nlon_in) fp32 contiguous -> y (planes, nlat_out, nlon_out) fp32"""
        y = torch.empty((x.shape[0], self.nlat_out, self.nlon_out), dtype=torch.float32, device=x.device)
        _lib.call("b200sht_resample_forward", self.handle, _ptr(x), _ptr(y), x.shape[0], _stream(x.device))
        return y

    def adjoint(self, dy):
        """dy (planes, nlat_out, nlon_out) fp32 contiguous -> dx (planes, nlat_in, nlon_in) fp32"""
        dx = torch.empty((dy.shape[0], self.nlat_in, self.nlon_in), dtype=torch.float32, device=dy.device)
        _lib.call("b200sht_resample_adjoint", self.handle, _ptr(dy), _ptr(dx), dy.shape[0], _stream(dy.device))
        return dx


_tables_cache, _plan_cache, _cache_lock = {}, {}, threading.Lock()


def get_tables(*key):
    """precompute_tables, cached per (nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out)"""
    with _cache_lock:
        if key not in _tables_cache:
            _tables_cache[key] = precompute_tables(*key)
        return _tables_cache[key]


def get_plan(key, device):
    """the device plan of get_tables(*key), cached per key and device"""
    device = torch.device(device)
    if device.type != "cuda":
        raise B200ShtError(f"ResampleS2 runs on CUDA devices only (got {device}); makani_b200 has no CPU fallback")
    dkey = key + (device.index if device.index is not None else torch.cuda.current_device(),)
    with _cache_lock:
        plan = _plan_cache.get(dkey)
    if plan is None:
        plan = ResamplePlan(*key[:4], get_tables(*key), device)
        with _cache_lock:
            plan = _plan_cache.setdefault(dkey, plan)
    return plan


class _Resample(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan):
        ctx.plan = plan
        return plan.forward(x)

    @staticmethod
    def backward(ctx, gy):
        return ctx.plan.adjoint(gy.to(torch.float32).contiguous()), None


class ResampleS2(nn.Module):
    """Bilinear resampling between two grids on the sphere (drop-in for torch_harmonics.ResampleS2 with mode="bilinear").

    The tables live in non-persistent buffers: the state dict is empty."""

    def __init__(self, nlat_in, nlon_in, nlat_out, nlon_out, grid_in="equiangular", grid_out="equiangular", mode="bilinear"):
        super().__init__()
        if mode != "bilinear":
            raise NotImplementedError(f"ResampleS2 mode {mode!r} is not implemented (only 'bilinear' is)")
        self.nlat_in, self.nlon_in, self.nlat_out, self.nlon_out = nlat_in, nlon_in, nlat_out, nlon_out
        self.grid_in, self.grid_out, self.mode = grid_in, grid_out, mode
        self._key = (nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out)
        tab = get_tables(*self._key)
        self.expand_poles = tab.expand_poles
        self.skip_resampling = (nlat_in, nlon_in, grid_in) == (nlat_out, nlon_out, grid_out)
        self.register_buffer("lat_idx", torch.from_numpy(tab.lat_idx), persistent=False)
        self.register_buffer("lat_weights", torch.from_numpy(tab.lat_w), persistent=False)
        self.register_buffer("lon_idx_left", torch.from_numpy(tab.lon_left), persistent=False)
        self.register_buffer("lon_idx_right", torch.from_numpy(tab.lon_right), persistent=False)
        self.register_buffer("lon_weights", torch.from_numpy(tab.lon_w), persistent=False)

    def extra_repr(self):
        return (f"in_shape={(self.nlat_in, self.nlon_in)}, out_shape={(self.nlat_out, self.nlon_out)}, grid_in={self.grid_in!r}, "
                f"grid_out={self.grid_out!r}, mode={self.mode!r}")

    def plan(self, device):
        return get_plan(self._key, device)

    def forward(self, x):
        if self.skip_resampling:
            return x
        if x.dim() < 2 or tuple(x.shape[-2:]) != (self.nlat_in, self.nlon_in):
            raise ValueError(f"expected (..., {self.nlat_in}, {self.nlon_in}), got {tuple(x.shape)}")
        if x.dtype != torch.float32:
            raise B200ShtError(f"ResampleS2 takes float32 input (got {x.dtype})")
        if not x.is_cuda:
            raise B200ShtError("ResampleS2 runs on CUDA devices only; makani_b200 has no CPU fallback")
        lead = tuple(x.shape[:-2])
        planes = math.prod(lead)
        if planes == 0:
            return x.new_empty(lead + (self.nlat_out, self.nlon_out))
        y = _Resample.apply(x.contiguous().view(planes, self.nlat_in, self.nlon_in), self.plan(x.device))
        return y.view(lead + (self.nlat_out, self.nlon_out))


def __getattr__(name):
    # the distributed module lives in makani_b200/distributed/resample.py; the reference runners import it from here
    if name == "DistributedResampleS2":
        from .distributed.resample import DistributedResampleS2
        return DistributedResampleS2
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")

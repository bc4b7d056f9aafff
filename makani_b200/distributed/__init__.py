"""h x w spatial model parallelism of the SHT -- mirror of `torch_harmonics.distributed` as makani uses it
(/root/reference/makani/models/networks/sfnonet.py:786-799, makani/models/common/spectral_convolution.py:169-173,
makani/mpu/fft.py:148-249 for the choreography; SURVEY.md section 3.3 and Appendix A).

    forward : [w-a2a chan<->lon] -> longitude FFT -> [w-a2a m<->chan] -> [h-a2a chan<->lat] -> Legendre -> [h-a2a l<->chan]
    inverse : the mirror image

The local stages run on the CUDA kernels of this package: an FFT-only plan for this rank's latitude rows and a Legendre plan for
this rank's orders (`b200sht_plan_create_ex`); the exchanged tensors use the plain complex layout, converted by
`b200sht_latspec_(un)pack` / `b200sht_spec_(un)pack_ex`.  The local-stage backend is replaceable (`set_local_ops`) so that the
choreography is unit-tested on CPU with gloo against the serial oracle.

DistributedRealVectorSHT / DistributedInverseRealVectorSHT (torch_harmonics' distributed vector transforms, built by makani's VortDivCRPSLoss
and GradientCRPSLoss with spatial_distributed=True) run the same choreography on (B, C, 2, ., .) fields: the transposes split the vector
channels, the longitude stages see the 2C component rows and the Legendre stage runs on a vector plan of this rank's orders
(B200SHT_PLAN_VECTOR with an order offset, `b200sht_vector_*`).

DistributedDiscreteContinuousConvS2 (distributed/disco.py: a latitude halo and window plans of psi_hat) and DistributedResampleS2
(distributed/resample.py: whole spheres of a subset of planes) are FCN3's local operators under the same h x w grid;
DistributedDiscreteContinuousConvTransposeS2 runs the DISCO stages the other way round, and DistributedNeighborhoodAttentionS2
(distributed/attention.py) runs the attention kernels on window plans of the neighbourhood, over the same halo.  DistributedAttentionS2
(distributed/attention.py) is the global attention on the same grid: each rank attends with its own queries to every key, gathered in
global (lat, lon) order, and its backward splits the kernels' query-side and key-side passes over the ranks' own queries and keys.
DistributedGeometricInstanceNormS2 and DistributedInstanceNorm2d (distributed/norm.py) gather per-rank statistics between the staged norm kernels.
"""
import ctypes

import torch
import torch.distributed as dist
import torch.nn as nn

from . import primitives
from .primitives import compute_split_shapes, split_tensor_along_dim, _transpose, _gather, _split, _reduce, _DistributedTranspose  # noqa: F401

_POLAR_GROUP = None
_AZIMUTH_GROUP = None
_IS_INITIALIZED = False


def init(polar_process_group, azimuth_process_group):
    """polar = latitude / degree (`h`) group, azimuth = longitude / order (`w`) group; either may be None (size 1)."""
    global _POLAR_GROUP, _AZIMUTH_GROUP, _IS_INITIALIZED
    _POLAR_GROUP, _AZIMUTH_GROUP, _IS_INITIALIZED = polar_process_group, azimuth_process_group, True


def finalize():
    global _POLAR_GROUP, _AZIMUTH_GROUP, _IS_INITIALIZED
    _POLAR_GROUP, _AZIMUTH_GROUP, _IS_INITIALIZED = None, None, False


def is_initialized():
    return _IS_INITIALIZED


def polar_group():
    return _POLAR_GROUP


def azimuth_group():
    return _AZIMUTH_GROUP


def _size(g):
    return dist.get_world_size(group=g) if (g is not None and dist.is_initialized()) else 1


def _rank(g):
    return dist.get_rank(group=g) if (g is not None and dist.is_initialized()) else 0


def polar_group_size():
    return _size(_POLAR_GROUP)


def azimuth_group_size():
    return _size(_AZIMUTH_GROUP)


def polar_group_rank():
    return _rank(_POLAR_GROUP)


def azimuth_group_rank():
    return _rank(_AZIMUTH_GROUP)


def distributed_transpose_azimuth(x, dims, dim1_split_sizes):
    return _DistributedTranspose.apply(x, dims, dim1_split_sizes, _AZIMUTH_GROUP)


def distributed_transpose_polar(x, dims, dim1_split_sizes):
    return _DistributedTranspose.apply(x, dims, dim1_split_sizes, _POLAR_GROUP)


# ------------------------------------------------------------------------------------------------------- local stages
class CudaLocalOps:
    """The four local stages on the CUDA kernels (fp32 or tf32 per `precision`)."""

    def __init__(self, t):
        self.t = t

    # -- plans ---------------------------------------------------------------------------------------------------
    def _fft_plan(self, device):
        from ..sht import Plan, _plan_cache, _plan_lock
        from ..quadrature import _grid_np
        t = self.t
        key = ("dist-fft", t.nlat, t.nlon, t.mmax, t.grid, t.lat_offset, t.nlat_local, device.index)
        with _plan_lock:
            p = _plan_cache.get(key)
            if p is None:
                cost, w = _grid_np(t.nlat, t.grid)
                sl = slice(t.lat_offset, t.lat_offset + t.nlat_local)
                p = Plan.create_ex(t.nlat_local, t.nlon, 1, t.mmax, 0, 1, cost[sl], w[sl], t.csphase, device)
                _plan_cache[key] = p
            return p

    def _leg_plan(self, device):
        from ..sht import Plan, _plan_cache, _plan_lock
        from ..quadrature import _grid_np
        t = self.t
        key = ("dist-leg", t.nlat, t.nlon, t.lmax, t.mmax, t.grid, t.m_offset, t.mmax_local, bool(t.csphase), device.index)
        with _plan_lock:
            p = _plan_cache.get(key)
            if p is None:
                cost, w = _grid_np(t.nlat, t.grid)
                p = Plan.create_ex(t.nlat, t.nlon, t.lmax, t.mmax_local, t.m_offset, 0, cost, w, t.csphase, device)
                _plan_cache[key] = p
            return p

    def _vleg_plan(self, device):
        """vector plan (tables D and Q) of this rank's orders m_offset .. m_offset + mmax_local - 1 over all latitudes"""
        from .. import _lib as L
        from ..sht import Plan, _plan_cache, _plan_lock
        from ..quadrature import _grid_np
        t = self.t
        key = ("dist-vleg", t.nlat, t.nlon, t.lmax, t.mmax, t.grid, t.m_offset, t.mmax_local, bool(t.csphase), device.index)
        with _plan_lock:
            p = _plan_cache.get(key)
            if p is None:
                cost, w = _grid_np(t.nlat, t.grid)
                p = Plan.create_ex(t.nlat, t.nlon, t.lmax, t.mmax_local, t.m_offset, L.PLAN_VECTOR, cost, w, t.csphase, device)
                _plan_cache[key] = p
            return p

    def _prec(self):
        from ..sht import resolve_precision
        return resolve_precision(self.t.precision)

    def _vprec(self):
        from ..vector_sht import _vector_precision
        return _vector_precision(self.t.precision)

    # -- stages --------------------------------------------------------------------------------------------------
    def fft(self, x):
        """real (B, C, nlat_loc, nlon) -> complex (B, C, nlat_loc, mmax), quadrature weights and 2 pi / nlon applied"""
        return _LocalFFT.apply(x.contiguous(), self._fft_plan(x.device), self._prec())

    def ifft(self, xc, dtype):
        return _LocalIFFT.apply(xc.to(torch.complex64).contiguous(), self._fft_plan(xc.device), self._prec(), dtype)

    def legendre(self, xc):
        """complex (B, C, nlat, m_loc) -> complex (B, C, lmax, m_loc)"""
        return _LocalLegendre.apply(xc.to(torch.complex64).contiguous(), self._leg_plan(xc.device), self._prec())

    def ilegendre(self, xc):
        return _LocalILegendre.apply(xc.to(torch.complex64).contiguous(), self._leg_plan(xc.device), self._prec())

    def vlegendre(self, xc):
        """complex (B, C, 2, nlat, m_loc) -> complex (B, C, 2, lmax, m_loc): (theta, phi) components -> (S, T) coefficients"""
        return _LocalVLegendre.apply(xc.to(torch.complex64).contiguous(), self._vleg_plan(xc.device), self._vprec())

    def ivlegendre(self, xc):
        """complex (B, C, 2, lmax, m_loc) -> complex (B, C, 2, nlat, m_loc)"""
        return _LocalIVLegendre.apply(xc.to(torch.complex64).contiguous(), self._vleg_plan(xc.device), self._vprec())


def _lib():
    from .. import _lib as L
    return L


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _st(dev):
    return _lib().launch_stream(dev)


def _dt(dtype):
    from ..sht import _dtype_code
    return _dtype_code(dtype)


class _LocalFFT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, plan, prec):
        L = _lib()
        B, C = x.shape[:2]
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=x.device)
        out = torch.empty(B, C, plan.nlat, plan.mmax, dtype=torch.complex64, device=x.device)
        L.call("b200sht_fft_analysis", plan.handle, _p(x), _dt(x.dtype), B, C, _p(lat), 0 | (2 if prec == L.PREC_TF32 else 0), _st(x.device))
        L.call("b200sht_latspec_unpack", plan.handle, _p(lat), _p(out), B, C, _st(x.device))
        ctx.plan, ctx.shape, ctx.dtype, ctx.prec = plan, tuple(x.shape), x.dtype, prec
        return out

    @staticmethod
    def backward(ctx, g):
        L = _lib()
        plan = ctx.plan
        B, C = ctx.shape[:2]
        g = g.contiguous()
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=g.device)
        gx = torch.empty(ctx.shape, dtype=ctx.dtype, device=g.device)
        L.call("b200sht_latspec_pack", plan.handle, _p(g), _p(lat), B, C, _st(g.device))
        L.call("b200sht_fft_synthesis", plan.handle, _p(lat), _p(gx), _dt(ctx.dtype), B, C, ctypes.c_void_p(0), 1, _st(g.device))   # standard latspec layout (from the transposes): CUDA-core FFT
        return gx, None, None


class _LocalIFFT(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xc, plan, prec, dtype):
        L = _lib()
        B, C = xc.shape[:2]
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=xc.device)
        y = torch.empty(B, C, plan.nlat, plan.nlon, dtype=dtype, device=xc.device)
        L.call("b200sht_latspec_pack", plan.handle, _p(xc), _p(lat), B, C, _st(xc.device))
        L.call("b200sht_fft_synthesis", plan.handle, _p(lat), _p(y), _dt(dtype), B, C, ctypes.c_void_p(0), 0, _st(xc.device))
        ctx.plan, ctx.prec = plan, prec
        return y

    @staticmethod
    def backward(ctx, gy):
        L = _lib()
        plan = ctx.plan
        gy = gy.contiguous()
        B, C = gy.shape[:2]
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=gy.device)
        g = torch.empty(B, C, plan.nlat, plan.mmax, dtype=torch.complex64, device=gy.device)
        L.call("b200sht_fft_analysis", plan.handle, _p(gy), _dt(gy.dtype), B, C, _p(lat), 1 | (2 if ctx.prec == L.PREC_TF32 else 0), _st(gy.device))
        L.call("b200sht_latspec_unpack", plan.handle, _p(lat), _p(g), B, C, _st(gy.device))
        return g, None, None, None


def _legendre_call(plan, prec, xc, direction):
    """direction 0: (B,C,nlat,m) -> (B,C,L,m); 1: (B,C,L,m) -> (B,C,nlat,m)"""
    L = _lib()
    B, C = xc.shape[:2]
    dev = xc.device
    lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=dev)
    spec = torch.empty(plan.spec_elems(B, C), dtype=torch.float32, device=dev)
    if direction == 0:
        out = torch.empty(B, C, plan.lmax, plan.mmax, dtype=torch.complex64, device=dev)
        L.call("b200sht_latspec_pack", plan.handle, _p(xc), _p(lat), B, C, _st(dev))
        L.call("b200sht_legendre_analysis", plan.handle, _p(lat), _p(spec), B, C, prec, _st(dev))
        L.call("b200sht_spec_unpack_ex", plan.lmax, plan.mmax, plan.m_offset, 0, _p(spec), _p(out), B, C, _st(dev))
    else:
        out = torch.empty(B, C, plan.nlat, plan.mmax, dtype=torch.complex64, device=dev)
        L.call("b200sht_spec_pack_ex", plan.lmax, plan.mmax, plan.m_offset, 0, _p(xc), _p(spec), B, C, _st(dev))
        L.call("b200sht_legendre_synthesis", plan.handle, _p(spec), _p(lat), B, C, prec, _st(dev))
        L.call("b200sht_latspec_unpack", plan.handle, _p(lat), _p(out), B, C, _st(dev))
    return out


class _LocalLegendre(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xc, plan, prec):
        ctx.plan, ctx.prec = plan, prec
        return _legendre_call(plan, prec, xc, 0)

    @staticmethod
    def backward(ctx, g):
        return _legendre_call(ctx.plan, ctx.prec, g.contiguous(), 1), None, None


class _LocalILegendre(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xc, plan, prec):
        ctx.plan, ctx.prec = plan, prec
        return _legendre_call(plan, prec, xc, 1)

    @staticmethod
    def backward(ctx, g):
        return _legendre_call(ctx.plan, ctx.prec, g.contiguous(), 0), None, None


def _vlegendre_call(plan, prec, xc, direction, scaled):
    """vector plan of an order shard.  direction 0: (B,C,2,nlat,m) -> (B,C,2,L,m), latspec pack -> analysis -> vector_spec_unpack(scaled);
    1: (B,C,2,L,m) -> (B,C,2,nlat,m), vector_spec_pack(scaled) -> synthesis -> latspec unpack.  The C vector fields are 2C component rows."""
    L = _lib()
    B, C = xc.shape[:2]
    dev = xc.device
    lat = torch.empty(plan.latspec_elems(B, 2 * C), dtype=torch.float32, device=dev)
    spec = torch.empty(plan.spec_elems(B, 2 * C), dtype=torch.float32, device=dev)
    if direction == 0:
        out = torch.empty(B, C, 2, plan.lmax, plan.mmax, dtype=torch.complex64, device=dev)
        L.call("b200sht_latspec_pack", plan.handle, _p(xc), _p(lat), B, 2 * C, _st(dev))
        L.call("b200sht_vector_legendre_analysis", plan.handle, _p(lat), _p(spec), B, C, prec, _st(dev))
        L.call("b200sht_vector_spec_unpack", plan.handle, _p(spec), _p(out), B, C, scaled, _st(dev))
    else:
        out = torch.empty(B, C, 2, plan.nlat, plan.mmax, dtype=torch.complex64, device=dev)
        L.call("b200sht_vector_spec_pack", plan.handle, _p(xc), _p(spec), B, C, scaled, _st(dev))
        L.call("b200sht_vector_legendre_synthesis", plan.handle, _p(spec), _p(lat), B, C, prec, _st(dev))
        L.call("b200sht_latspec_unpack", plan.handle, _p(lat), _p(out), B, 2 * C, _st(dev))
    return out


class _LocalVLegendre(torch.autograd.Function):
    """analysis with the 1 / (l (l + 1)) scaling; backward: its adjoint, vector_spec_pack(scaled=1) -> synthesis"""

    @staticmethod
    def forward(ctx, xc, plan, prec):
        ctx.plan, ctx.prec = plan, prec
        return _vlegendre_call(plan, prec, xc, 0, 1)

    @staticmethod
    def backward(ctx, g):
        return _vlegendre_call(ctx.plan, ctx.prec, g.to(torch.complex64).contiguous(), 1, 1), None, None


class _LocalIVLegendre(torch.autograd.Function):
    """synthesis without scaling; backward: its adjoint, analysis -> vector_spec_unpack(scaled=0)"""

    @staticmethod
    def forward(ctx, xc, plan, prec):
        ctx.plan, ctx.prec = plan, prec
        return _vlegendre_call(plan, prec, xc, 1, 0)

    @staticmethod
    def backward(ctx, g):
        return _vlegendre_call(ctx.plan, ctx.prec, g.to(torch.complex64).contiguous(), 0, 0), None, None


_LOCAL_OPS_FACTORY = CudaLocalOps


def set_local_ops(factory):
    """Replace the local-stage backend (tests: a CPU implementation built on the oracle).  `factory(transform)` -> object with
    fft / ifft / legendre / ilegendre, and for DistributedRealVectorSHT / DistributedInverseRealVectorSHT also
    vlegendre(xc): complex (B, C, 2, nlat, m_loc) -> (B, C, 2, lmax, m_loc), the Legendre stage of the forward vector transform on this rank's
    orders (theta / phi components in, spheroidal / toroidal coefficients out, 1 / (l (l + 1)) applied), and ivlegendre, its inverse-transform
    counterpart (B, C, 2, lmax, m_loc) -> (B, C, 2, nlat, m_loc)."""
    global _LOCAL_OPS_FACTORY
    _LOCAL_OPS_FACTORY = factory if factory is not None else CudaLocalOps


# ------------------------------------------------------------------------------------------------------------ modules
class _DistributedBase(nn.Module):
    packed_dense = True  # SpectralConv: the l/m-sharded packed spectra store every entry (no block triangle)

    def __init__(self, nlat, nlon, lmax=None, mmax=None, grid="equiangular", norm="ortho", csphase=True, precision="auto"):
        super().__init__()
        if norm != "ortho":
            raise NotImplementedError("makani_b200 implements norm='ortho'")
        if grid not in ("equiangular", "legendre-gauss"):
            raise ValueError(f"Unknown quadrature mode {grid}")
        self.nlat, self.nlon, self.grid, self.norm, self.csphase, self.precision = int(nlat), int(nlon), grid, norm, csphase, precision
        self.lmax = int(lmax or self.nlat)
        self.mmax = int(mmax or self.nlon // 2 + 1)
        self.comm_size_polar, self.comm_rank_polar = polar_group_size(), polar_group_rank()
        self.comm_size_azimuth, self.comm_rank_azimuth = azimuth_group_size(), azimuth_group_rank()
        self.lat_shapes = compute_split_shapes(self.nlat, self.comm_size_polar)
        self.lon_shapes = compute_split_shapes(self.nlon, self.comm_size_azimuth)
        self.l_shapes = compute_split_shapes(self.lmax, self.comm_size_polar)
        self.m_shapes = compute_split_shapes(self.mmax, self.comm_size_azimuth)
        self.nlat_local = self.lat_shapes[self.comm_rank_polar]
        self.nlon_local = self.lon_shapes[self.comm_rank_azimuth]
        self.lmax_local = self.l_shapes[self.comm_rank_polar]
        self.mmax_local = self.m_shapes[self.comm_rank_azimuth]
        self.lat_offset = sum(self.lat_shapes[: self.comm_rank_polar])
        self.m_offset = sum(self.m_shapes[: self.comm_rank_azimuth])
        self.l_offset = sum(self.l_shapes[: self.comm_rank_polar])
        self._ops = _LOCAL_OPS_FACTORY(self)

    def extra_repr(self):
        return (f"nlat={self.nlat}, nlon={self.nlon}, lmax={self.lmax}, mmax={self.mmax}, grid={self.grid}, "
                f"h={self.comm_size_polar}, w={self.comm_size_azimuth}")


class DistributedRealSHT(_DistributedBase):
    """x local (B, C, nlat_loc, nlon_loc) -> coefficients local (B, C, l_loc, m_loc)."""

    def forward(self, x):
        if x.dim() < 3:
            raise ValueError(f"Expected tensor with at least 3 dimensions but got {x.dim()} instead")
        lead = x.shape[:-2]
        x4 = x if x.dim() == 4 else x.reshape(1, -1, *x.shape[-2:])
        if x4.shape[-2] != self.nlat_local or x4.shape[-1] != self.nlon_local:
            raise ValueError(f"DistributedRealSHT: expected local grid ({self.nlat_local}, {self.nlon_local}), got {tuple(x4.shape[-2:])}")
        num_chans = x4.shape[1]
        if self.comm_size_azimuth > 1:
            x4 = distributed_transpose_azimuth(x4, (1, -1), self.lon_shapes)
        xc = self._ops.fft(x4)
        if self.comm_size_azimuth > 1:
            xc = distributed_transpose_azimuth(xc, (-1, 1), compute_split_shapes(num_chans, self.comm_size_azimuth))
        if self.comm_size_polar > 1:
            xc = distributed_transpose_polar(xc, (1, -2), self.lat_shapes)
        xc = self._ops.legendre(xc)
        if self.comm_size_polar > 1:
            xc = distributed_transpose_polar(xc, (-2, 1), compute_split_shapes(num_chans, self.comm_size_polar))
        return xc if x.dim() == 4 else xc.reshape(*lead, self.lmax_local, self.mmax_local)

    def forward_packed(self, x):
        from ..sht import _SpecPackEx
        return _SpecPackEx.apply(self.forward(x), 0, 1)


class DistributedInverseRealSHT(_DistributedBase):
    """coefficients local (B, C, l_loc, m_loc) -> x local (B, C, nlat_loc, nlon_loc)."""

    def forward(self, x, dtype=torch.float32):
        if x.dim() < 3:
            raise ValueError(f"Expected tensor with at least 3 dimensions but got {x.dim()} instead")
        lead = x.shape[:-2]
        x4 = x if x.dim() == 4 else x.reshape(1, -1, *x.shape[-2:])
        if x4.shape[-2] != self.lmax_local or x4.shape[-1] != self.mmax_local:
            raise ValueError(f"DistributedInverseRealSHT: expected local modes ({self.lmax_local}, {self.mmax_local}), got {tuple(x4.shape[-2:])}")
        num_chans = x4.shape[1]
        if self.comm_size_polar > 1:
            x4 = distributed_transpose_polar(x4, (1, -2), self.l_shapes)
        xc = self._ops.ilegendre(x4)
        if self.comm_size_polar > 1:
            xc = distributed_transpose_polar(xc, (-2, 1), compute_split_shapes(num_chans, self.comm_size_polar))
        if self.comm_size_azimuth > 1:
            xc = distributed_transpose_azimuth(xc, (1, -1), self.m_shapes)
        y = self._ops.ifft(xc, dtype)
        if self.comm_size_azimuth > 1:
            y = distributed_transpose_azimuth(y, (-1, 1), compute_split_shapes(num_chans, self.comm_size_azimuth))
        return y if x.dim() == 4 else y.reshape(*lead, self.nlat_local, self.nlon_local)

    def forward_packed(self, spec, B, C, dtype=torch.float32, bias=None):
        from ..sht import _SpecUnpackEx
        xc = _SpecUnpackEx.apply(spec, self.lmax_local, self.mmax_local, B, C, 0, 1)
        y = self.forward(xc, dtype)
        if bias is not None:
            y = y + bias.to(y.dtype)
        return y


# ----------------------------------------------------------------------------------------------------- vector modules
def _as_vector_fields(x, tail, who):
    """(..., 2, a, b) -> (B, C, 2, a, b) (leading dimensions flattened into vector channels unless x is 5-D) plus the leading shape"""
    if x.dim() < 3 or tuple(x.shape[-3:]) != tail:
        raise ValueError(f"{who}: expected local shape (..., {tail[0]}, {tail[1]}, {tail[2]}), got {tuple(x.shape)}")
    return (x if x.dim() == 5 else x.reshape(1, -1, *tail)), x.shape[:-3]


class DistributedRealVectorSHT(_DistributedBase):
    """x local (..., 2, nlat_loc, nlon_loc) float32 / bf16 -> coefficients local complex (..., 2, l_loc, m_loc) (component 0 theta, 1 phi in;
    spheroidal S, toroidal T out).  The transposes of DistributedRealSHT on the 5-D (B, C, 2, ., .) tensor: they split the vector channels
    (dim 1), so both components of a field stay on one rank; the longitude stages see its 2C component rows."""

    def forward(self, x):
        from ..vector_sht import _vector_precision
        _vector_precision(self.precision)
        x5, lead = _as_vector_fields(x, (2, self.nlat_local, self.nlon_local), "DistributedRealVectorSHT")
        num_chans = x5.shape[1]
        if self.comm_size_azimuth > 1:
            x5 = distributed_transpose_azimuth(x5, (1, -1), self.lon_shapes)
        B, C = x5.shape[:2]
        xc = self._ops.fft(x5.reshape(B, 2 * C, self.nlat_local, self.nlon)).reshape(B, C, 2, self.nlat_local, self.mmax)
        if self.comm_size_azimuth > 1:
            xc = distributed_transpose_azimuth(xc, (-1, 1), compute_split_shapes(num_chans, self.comm_size_azimuth))
        if self.comm_size_polar > 1:
            xc = distributed_transpose_polar(xc, (1, -2), self.lat_shapes)
        xc = self._ops.vlegendre(xc)
        if self.comm_size_polar > 1:
            xc = distributed_transpose_polar(xc, (-2, 1), compute_split_shapes(num_chans, self.comm_size_polar))
        return xc if x.dim() == 5 else xc.reshape(*lead, 2, self.lmax_local, self.mmax_local)


class DistributedInverseRealVectorSHT(_DistributedBase):
    """coefficients local complex (..., 2, l_loc, m_loc) -> x local (..., 2, nlat_loc, nlon_loc) (float32 unless `dtype` says otherwise);
    the transposes of DistributedInverseRealSHT on the vector channels, as in DistributedRealVectorSHT."""

    def forward(self, x, dtype=torch.float32):
        from ..vector_sht import _vector_precision
        _vector_precision(self.precision)
        x5, lead = _as_vector_fields(x, (2, self.lmax_local, self.mmax_local), "DistributedInverseRealVectorSHT")
        num_chans = x5.shape[1]
        if self.comm_size_polar > 1:
            x5 = distributed_transpose_polar(x5, (1, -2), self.l_shapes)
        xc = self._ops.ivlegendre(x5)
        if self.comm_size_polar > 1:
            xc = distributed_transpose_polar(xc, (-2, 1), compute_split_shapes(num_chans, self.comm_size_polar))
        if self.comm_size_azimuth > 1:
            xc = distributed_transpose_azimuth(xc, (1, -1), self.m_shapes)
        B, C = xc.shape[:2]
        y = self._ops.ifft(xc.reshape(B, 2 * C, self.nlat_local, self.mmax), dtype).reshape(B, C, 2, self.nlat_local, self.nlon)
        if self.comm_size_azimuth > 1:
            y = distributed_transpose_azimuth(y, (-1, 1), compute_split_shapes(num_chans, self.comm_size_azimuth))
        return y if x.dim() == 5 else y.reshape(*lead, 2, self.nlat_local, self.nlon_local)


from .disco import DistributedDiscreteContinuousConvS2, DistributedDiscreteContinuousConvTransposeS2, set_disco_local_ops  # noqa: E402,F401
from .resample import DistributedResampleS2, set_resample_local_ops  # noqa: E402,F401
from .attention import DistributedAttentionS2, DistributedNeighborhoodAttentionS2, set_attention_local_ops, set_global_attention_local_ops  # noqa: E402,F401,E501
from .norm import DistributedGeometricInstanceNormS2, DistributedInstanceNorm2d, set_norm_local_ops  # noqa: E402,F401

"""RealSHT / InverseRealSHT -- drop-in for `torch_harmonics.RealSHT` / `InverseRealSHT` as makani uses them
(/root/reference/makani/models/networks/sfnonet.py:792-805, /root/reference/makani/models/common/spectral_convolution.py:239-253),
computed by the hand-written sm_90a kernels in `csrc/` through the C ABI in include/b200sht.h.

Same constructor signature, attributes (.nlat .nlon .lmax .mmax .grid .norm .csphase) and call convention:
    RealSHT(nlat, nlon, lmax=None, mmax=None, grid="equiangular", norm="ortho", csphase=True)(x: (..., nlat, nlon)) -> complex (..., lmax, mmax)
The Legendre tables live inside a device-side plan (no state-dict entries, like the reference's non-persistent buffers).

Inside SpectralConv the transforms exchange *packed* spectral tensors (float32 [L][M][2][B][cp], see DESIGN.md) so that
no layout conversion kernel runs between the Legendre stage and the channel mix.
"""
import ctypes
import threading

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import B200ShtError, c_void_p as _VP, dtype_code as _dtype_code, launch_stream as _stream, ptr as _ptr  # scripts import these from here
from .quadrature import _grid_np


def resolve_precision(precision="auto"):
    """'fp32' -> CUDA-core fp32 FMA; 'tf32' -> tensor-core TF32; 'fp32x3' -> fp32 operands with the Legendre stages as 3 x TF32 on the
    tensor cores (rtol 1e-5 element bound, ~1.7 x faster than 'fp32'; see B200SHT_PREC_FP32X3 in include/b200sht.h); 'auto' follows
    torch.backends.cuda.matmul.allow_tf32, which is how the reference picks its arithmetic (train.py:87 sets allow_tf32=True,
    tests/testutils.py:55-66 disable it)."""
    if precision == "auto":
        precision = "tf32" if torch.backends.cuda.matmul.allow_tf32 else "fp32"
    if precision == "fp32":
        return _lib.PREC_FP32
    if precision == "tf32":
        return _lib.PREC_TF32
    if precision == "fp32x3":
        return _lib.PREC_FP32X3
    raise ValueError(f"unknown precision {precision!r}")


class Plan:
    """Owns one `b200sht_plan` (Legendre table, FFT twiddles, TMA descriptors) on one CUDA device."""

    def __init__(self, nlat, nlon, lmax, mmax, grid, csphase, device, vector=False):
        """vector=True: a vector-SHT plan (tables D and Q instead of P) for RealVectorSHT / InverseRealVectorSHT."""
        cost, w = _grid_np(nlat, grid)
        self._create(nlat, nlon, lmax, mmax, 0, _lib.PLAN_VECTOR if vector else 0, cost, w, csphase, device)

    @classmethod
    def create_ex(cls, nlat, nlon, lmax, mmax, m_offset, flags, cost, quad_w, csphase, device):
        """Sub-plans of the distributed SHT (b200sht_plan_create_ex): order offset and/or FFT-only (flags & 1)."""
        self = cls.__new__(cls)
        self._create(nlat, nlon, lmax, mmax, m_offset, flags, cost, quad_w, csphase, device)
        return self

    def _create(self, nlat, nlon, lmax, mmax, m_offset, flags, cost, quad_w, csphase, device):
        if device.type != "cuda":
            raise B200ShtError("makani_b200 transforms run on CUDA devices only (no CPU fallback)")
        cost = np.ascontiguousarray(cost, dtype=np.float64)
        quad_w = np.ascontiguousarray(quad_w, dtype=np.float64)
        handle = _VP()
        _lib.call("b200sht_plan_create_ex", ctypes.byref(handle), nlat, nlon, lmax, mmax, m_offset, flags, cost.ctypes.data_as(_VP),
                  quad_w.ctypes.data_as(_VP), 1 if csphase else 0, _stream(device))
        lib = _lib.load()
        self.handle = handle
        self.device = device
        self.nlat, self.nlon, self.lmax, self.mmax, self.m_offset = nlat, nlon, lmax, mmax, m_offset
        self.kp = int(lib.b200sht_plan_query(handle, 4))
        self.umma_ok = bool(lib.b200sht_plan_query(handle, 6))
        self.dft_ok = bool(lib.b200sht_plan_query(handle, 8))
        self.vector = bool(lib.b200sht_plan_query(handle, 9))

    def query(self, what):
        """b200sht_plan_query: 0 nlat, 1 nlon, 2 lmax, 3 mmax, 4 kp, 5 table bytes, 6 tensor-core path available, 7 m_offset, 8 tensor-core DFT available,
        9 vector plan."""
        return int(_lib.load().b200sht_plan_query(self.handle, what))

    def latspec_elems(self, B, C):
        return int(_lib.load().b200sht_latspec_elems(self.handle, B, C))

    def spec_elems(self, B, C):
        return int(_lib.load().b200sht_spec_elems(self.handle, B, C))

    def table(self):
        """Device copy of the fp32 Legendre table [mmax][lmax][kp]; of a vector plan the tables D and Q as [2][mmax][lmax][kp] (testing / inspection)."""
        nt = 2 if self.vector else 1
        out = torch.empty(nt * self.mmax * self.lmax * self.kp, dtype=torch.float32, device=self.device)
        _lib.call("b200sht_plan_copy_table", self.handle, _ptr(out), _stream(self.device))
        return out.view(nt, self.mmax, self.lmax, self.kp) if self.vector else out.view(self.mmax, self.lmax, self.kp)

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                _lib.load().b200sht_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


_plan_cache = {}
_plan_lock = threading.Lock()


def get_plan(nlat, nlon, lmax, mmax, grid, csphase, device, vector=False):
    """Plans are shared between modules with the same geometry on the same device (SFNO builds 4 transforms, FCN3 2).  vector=True: the
    vector-SHT plan of that geometry (shared by RealVectorSHT and InverseRealVectorSHT), cached under its own key."""
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    key = (nlat, nlon, lmax, mmax, grid, bool(csphase), device.index)
    if vector:
        key = key + ("vector",)
    with _plan_lock:
        p = _plan_cache.get(key)
        if p is None:
            p = Plan(nlat, nlon, lmax, mmax, grid, csphase, device, vector=vector)
            _plan_cache[key] = p
        return p


def _synthesis_pair(plan, spec, lat, y, dtype, B, C, bias32, mode, precision, st):
    """Legendre synthesis + longitude synthesis.  TF32 on a grid the tensor-core DFT covers: tiled latspec layout + dft.cu kernels."""
    if precision == _lib.PREC_TF32 and plan.dft_ok:
        _lib.call("b200sht_legendre_synthesis_tiled", plan.handle, _ptr(spec), _ptr(lat), B, C, st)
        _lib.call("b200sht_fft_synthesis", plan.handle, _ptr(lat), _ptr(y), _dtype_code(dtype), B, C, _ptr(bias32), mode | 2, st)
    else:
        _lib.call("b200sht_legendre_synthesis", plan.handle, _ptr(spec), _ptr(lat), B, C, precision, st)
        _lib.call("b200sht_fft_synthesis", plan.handle, _ptr(lat), _ptr(y), _dtype_code(dtype), B, C, _ptr(bias32), mode, st)


# ----------------------------------------------------------------------------------------------------------------
# autograd functions on packed tensors
# ----------------------------------------------------------------------------------------------------------------
class _AnalysisPacked(torch.autograd.Function):
    """x (B, C, nlat, nlon) -> packed spec.  Backward = Legendre synthesis + longitude synthesis with adjoint scaling."""

    @staticmethod
    def forward(ctx, x, plan, precision):
        B, C = x.shape[0], x.shape[1]
        dev = x.device
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=dev)
        spec = torch.empty(plan.spec_elems(B, C), dtype=torch.float32, device=dev)
        st = _stream(dev)
        _lib.call("b200sht_fft_analysis", plan.handle, _ptr(x), _dtype_code(x.dtype), B, C, _ptr(lat), 0 | (2 if precision == _lib.PREC_TF32 else 0), st)
        _lib.call("b200sht_legendre_analysis", plan.handle, _ptr(lat), _ptr(spec), B, C, precision, st)
        ctx.plan, ctx.precision, ctx.shape, ctx.dtype = plan, precision, tuple(x.shape), x.dtype
        return spec

    @staticmethod
    def backward(ctx, gspec):
        plan, (B, C, H, W) = ctx.plan, ctx.shape
        gspec = gspec.contiguous()
        dev = gspec.device
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=dev)
        gx = torch.empty(ctx.shape, dtype=ctx.dtype, device=dev)
        st = _stream(dev)
        _synthesis_pair(plan, gspec, lat, gx, ctx.dtype, B, C, None, 1, ctx.precision, st)
        return gx, None, None


class _SynthesisPacked(torch.autograd.Function):
    """packed spec -> y (B, C, nlat, nlon) (+ per-channel bias).  Backward = longitude analysis (adjoint scaling) + Legendre analysis."""

    @staticmethod
    def forward(ctx, spec, bias, plan, precision, B, C, dtype):
        dev = spec.device
        spec = spec.contiguous()
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=dev)
        y = torch.empty((B, C, plan.nlat, plan.nlon), dtype=dtype, device=dev)
        st = _stream(dev)
        b32 = None
        if bias is not None:
            b32 = bias.detach().reshape(-1).to(torch.float32).contiguous()
        _synthesis_pair(plan, spec, lat, y, dtype, B, C, b32, 0, precision, st)
        ctx.plan, ctx.precision, ctx.B, ctx.C = plan, precision, B, C
        ctx.has_bias = bias is not None
        ctx.bias_shape = tuple(bias.shape) if bias is not None else None
        ctx.bias_dtype = bias.dtype if bias is not None else None
        return y

    @staticmethod
    def backward(ctx, gy):
        plan, B, C = ctx.plan, ctx.B, ctx.C
        gy = gy.contiguous()
        dev = gy.device
        lat = torch.empty(plan.latspec_elems(B, C), dtype=torch.float32, device=dev)
        st = _stream(dev)
        _lib.call("b200sht_fft_analysis", plan.handle, _ptr(gy), _dtype_code(gy.dtype), B, C, _ptr(lat), 1 | (2 if ctx.precision == _lib.PREC_TF32 else 0), st)
        gbias = None
        if ctx.has_bias and ctx.needs_input_grad[1]:
            gb = torch.empty(C, dtype=torch.float32, device=dev)
            _lib.call("b200sht_bias_grad", plan.handle, _ptr(lat), _ptr(gb), B, C, st)
            gbias = gb.reshape(ctx.bias_shape).to(ctx.bias_dtype)
        gspec = None
        if ctx.needs_input_grad[0]:
            gspec = torch.empty(plan.spec_elems(B, C), dtype=torch.float32, device=dev)
            _lib.call("b200sht_legendre_analysis", plan.handle, _ptr(lat), _ptr(gspec), B, C, ctx.precision, st)
        return gspec, gbias, None, None, None, None, None


class _SpecUnpack(torch.autograd.Function):
    """packed spec -> complex64 (B, C, L, M) (exact zeros for l < m)."""

    @staticmethod
    def forward(ctx, spec, L, M, B, C):
        out = torch.empty((B, C, L, M), dtype=torch.complex64, device=spec.device)
        _lib.call("b200sht_spec_unpack", L, M, _ptr(spec.contiguous()), _ptr(out), B, C, _stream(spec.device))
        ctx.dims = (L, M, B, C)
        return out

    @staticmethod
    def backward(ctx, g):
        L, M, B, C = ctx.dims
        g = g.contiguous()
        spec = torch.empty(int(_lib.load().b200sht_spec_elems_lm(L, M, B, C)), dtype=torch.float32, device=g.device)
        _lib.call("b200sht_spec_pack", L, M, _ptr(g), _ptr(spec), B, C, _stream(g.device))
        return spec, None, None, None, None


class _SpecPack(torch.autograd.Function):
    """complex64 (B, C, L, M) -> packed spec."""

    @staticmethod
    def forward(ctx, coeffs):
        B, C, L, M = coeffs.shape
        coeffs = coeffs.contiguous()
        spec = torch.empty(int(_lib.load().b200sht_spec_elems_lm(L, M, B, C)), dtype=torch.float32, device=coeffs.device)
        _lib.call("b200sht_spec_pack", L, M, _ptr(coeffs), _ptr(spec), B, C, _stream(coeffs.device))
        ctx.dims = (L, M, B, C)
        return spec

    @staticmethod
    def backward(ctx, gspec):
        L, M, B, C = ctx.dims
        out = torch.empty((B, C, L, M), dtype=torch.complex64, device=gspec.device)
        _lib.call("b200sht_spec_unpack", L, M, _ptr(gspec.contiguous()), _ptr(out), B, C, _stream(gspec.device))
        return out


class _SpecUnpackEx(torch.autograd.Function):
    """packed spec -> complex64 (B, C, L, M) with an order offset and/or dense storage (distributed path)."""

    @staticmethod
    def forward(ctx, spec, L, M, B, C, m_offset, dense):
        out = torch.empty((B, C, L, M), dtype=torch.complex64, device=spec.device)
        _lib.call("b200sht_spec_unpack_ex", L, M, m_offset, dense, _ptr(spec.contiguous()), _ptr(out), B, C, _stream(spec.device))
        ctx.dims = (L, M, B, C, m_offset, dense)
        return out

    @staticmethod
    def backward(ctx, g):
        L, M, B, C, m_offset, dense = ctx.dims
        g = g.contiguous()
        spec = torch.empty(int(_lib.load().b200sht_spec_elems_lm(L, M, B, C)), dtype=torch.float32, device=g.device)
        _lib.call("b200sht_spec_pack_ex", L, M, m_offset, dense, _ptr(g), _ptr(spec), B, C, _stream(g.device))
        return spec, None, None, None, None, None, None


class _SpecPackEx(torch.autograd.Function):
    """complex64 (B, C, L, M) -> packed spec with an order offset and/or dense storage."""

    @staticmethod
    def forward(ctx, coeffs, m_offset, dense):
        B, C, L, M = coeffs.shape
        coeffs = coeffs.contiguous()
        spec = torch.empty(int(_lib.load().b200sht_spec_elems_lm(L, M, B, C)), dtype=torch.float32, device=coeffs.device)
        _lib.call("b200sht_spec_pack_ex", L, M, m_offset, dense, _ptr(coeffs), _ptr(spec), B, C, _stream(coeffs.device))
        ctx.dims = (L, M, B, C, m_offset, dense)
        return spec

    @staticmethod
    def backward(ctx, gspec):
        L, M, B, C, m_offset, dense = ctx.dims
        out = torch.empty((B, C, L, M), dtype=torch.complex64, device=gspec.device)
        _lib.call("b200sht_spec_unpack_ex", L, M, m_offset, dense, _ptr(gspec.contiguous()), _ptr(out), B, C, _stream(gspec.device))
        return out, None, None


def _as_bc(x, nd_tail=2):
    """(..., h, w) -> (B, C, h, w) view plus the leading shape to restore."""
    lead = x.shape[:-nd_tail]
    if x.dim() == nd_tail + 2:
        return x, lead
    n = 1
    for s in lead:
        n *= int(s)
    return x.reshape(1, n, *x.shape[-nd_tail:]), lead


class _TransformBase(nn.Module):
    def __init__(self, nlat, nlon, lmax=None, mmax=None, grid="equiangular", norm="ortho", csphase=True, precision="auto"):
        super().__init__()
        if norm != "ortho":
            raise NotImplementedError("makani_b200 implements norm='ortho' (the only normalisation makani requests)")
        if grid not in ("equiangular", "legendre-gauss"):
            raise ValueError(f"Unknown quadrature mode {grid}")
        self.nlat, self.nlon = int(nlat), int(nlon)
        self.grid, self.norm, self.csphase = grid, norm, csphase
        self.lmax = int(lmax or self.nlat)
        self.mmax = int(mmax or self.nlon // 2 + 1)
        self.precision = precision

    def plan(self, device):
        return get_plan(self.nlat, self.nlon, self.lmax, self.mmax, self.grid, self.csphase, device)

    def extra_repr(self):
        return f"nlat={self.nlat}, nlon={self.nlon}, lmax={self.lmax}, mmax={self.mmax}, grid={self.grid}, csphase={self.csphase}"


class RealSHT(_TransformBase):
    """Forward real spherical harmonic transform (drop-in for torch_harmonics.RealSHT)."""

    def forward_packed(self, x):
        """x (B, C, nlat, nlon) float32/bfloat16 -> packed spectrum (flat float32 tensor)."""
        if x.shape[-2] != self.nlat or x.shape[-1] != self.nlon:
            raise ValueError(f"RealSHT: expected (..., {self.nlat}, {self.nlon}), got {tuple(x.shape)}")
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.to(torch.float32)
        return _AnalysisPacked.apply(x.contiguous(), self.plan(x.device), resolve_precision(self.precision))

    def forward(self, x):
        x4, lead = _as_bc(x)
        spec = self.forward_packed(x4)
        out = _SpecUnpack.apply(spec, self.lmax, self.mmax, x4.shape[0], x4.shape[1])
        return out.reshape(*lead, self.lmax, self.mmax)


class InverseRealSHT(_TransformBase):
    """Inverse real spherical harmonic transform (drop-in for torch_harmonics.InverseRealSHT)."""

    def forward_packed(self, spec, B, C, dtype=torch.float32, bias=None):
        """packed spectrum -> (B, C, nlat, nlon) in `dtype`; `bias` ([1,C,1,1] or [C]) is added in the FFT epilogue."""
        return _SynthesisPacked.apply(spec, bias, self.plan(spec.device), resolve_precision(self.precision), B, C, dtype)

    def forward(self, x):
        if x.shape[-2] != self.lmax or x.shape[-1] != self.mmax:
            raise ValueError(f"InverseRealSHT: expected (..., {self.lmax}, {self.mmax}), got {tuple(x.shape)}")
        if x.dtype != torch.complex64:
            x = x.to(torch.complex64)
        x4, lead = _as_bc(x)
        spec = _SpecPack.apply(x4)
        y = self.forward_packed(spec, x4.shape[0], x4.shape[1], torch.float32)
        return y.reshape(*lead, self.nlat, self.nlon)

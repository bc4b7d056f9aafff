"""RealVectorSHT / InverseRealVectorSHT -- drop-in for `torch_harmonics.RealVectorSHT` / `InverseRealVectorSHT` as makani's vector losses
build them (makani/utils/losses/base_loss.py:427-469 VortDivBaseLoss, :518-565 GradientBaseLoss), computed by the sm_90a kernels through the
vector entry points of include/b200sht.h.

    RealVectorSHT(nlat, nlon, lmax=None, mmax=None, grid="equiangular", norm="ortho", csphase=True)(x: (..., 2, nlat, nlon)) -> complex (..., 2, lmax, mmax)
    InverseRealVectorSHT(...)(c: complex (..., 2, lmax, mmax)) -> float32 (..., 2, nlat, nlon)

Input component 0 is the colatitude (theta) component and 1 the longitude (phi) component; output 0 holds the spheroidal coefficients S and
1 the toroidal coefficients T.  ivsht([f_lm, 0]) is the surface gradient (df/dtheta, df/dphi / sin theta) and ivsht([0, g_lm]) = -r x grad g.
The (theta, phi) pair is read in place as two component rows of the longitude transform; the contraction runs on the vector plan's tables
D = dP/dtheta and Q = m P / sin(theta) (DESIGN.md section 3).
"""
import torch

from . import _lib
from ._lib import B200ShtError, dtype_code as _dtype_code, launch_stream as _stream, ptr as _ptr
from .sht import _TransformBase, get_plan, resolve_precision


def _vector_precision(precision):
    p = resolve_precision(precision)
    if p == _lib.PREC_FP32X3:
        raise B200ShtError("the vector transforms have no 'fp32x3' mode (use 'fp32' or 'tf32')")
    return p


def _workspace(plan, B, C, device):
    n = int(_lib.load().b200sht_vsht_workspace_bytes(plan.handle, B, C))
    return torch.empty(n, dtype=torch.uint8, device=device)


class _VectorAnalysis(torch.autograd.Function):
    """x (B, C, 2, nlat, nlon) -> complex64 (B, C, 2, lmax, mmax).  Backward: b200sht_vsht_forward_adjoint."""

    @staticmethod
    def forward(ctx, x, plan, precision):
        B, C = x.shape[0], x.shape[1]
        out = torch.empty((B, C, 2, plan.lmax, plan.mmax), dtype=torch.complex64, device=x.device)
        ws = _workspace(plan, B, C, x.device)
        _lib.call("b200sht_vsht_forward", plan.handle, _ptr(x), _dtype_code(x.dtype), B, C, _ptr(out), _ptr(ws), precision, _stream(x.device))
        ctx.plan, ctx.precision, ctx.shape, ctx.dtype = plan, precision, tuple(x.shape), x.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        plan, (B, C) = ctx.plan, ctx.shape[:2]
        g = g.to(torch.complex64).contiguous()
        gx = torch.empty(ctx.shape, dtype=ctx.dtype, device=g.device)
        ws = _workspace(plan, B, C, g.device)
        _lib.call("b200sht_vsht_forward_adjoint", plan.handle, _ptr(g), _ptr(gx), _dtype_code(ctx.dtype), B, C, _ptr(ws), ctx.precision,
                  _stream(g.device))
        return gx, None, None


class _VectorSynthesis(torch.autograd.Function):
    """complex64 (B, C, 2, lmax, mmax) -> float32 (B, C, 2, nlat, nlon).  Backward: b200sht_vsht_inverse_adjoint."""

    @staticmethod
    def forward(ctx, c, plan, precision):
        B, C = c.shape[0], c.shape[1]
        y = torch.empty((B, C, 2, plan.nlat, plan.nlon), dtype=torch.float32, device=c.device)
        ws = _workspace(plan, B, C, c.device)
        _lib.call("b200sht_vsht_inverse", plan.handle, _ptr(c), _ptr(y), _lib.F32, B, C, _ptr(ws), precision, _stream(c.device))
        ctx.plan, ctx.precision, ctx.BC = plan, precision, (B, C)
        return y

    @staticmethod
    def backward(ctx, gy):
        plan, (B, C) = ctx.plan, ctx.BC
        gy = gy.to(torch.float32).contiguous()
        gc = torch.empty((B, C, 2, plan.lmax, plan.mmax), dtype=torch.complex64, device=gy.device)
        ws = _workspace(plan, B, C, gy.device)
        _lib.call("b200sht_vsht_inverse_adjoint", plan.handle, _ptr(gy), _lib.F32, B, C, _ptr(gc), _ptr(ws), ctx.precision, _stream(gy.device))
        return gc, None, None


def _as_fields(x, tail):
    """(..., 2, a, b) -> contiguous (1, n, 2, a, b) plus the leading shape to restore."""
    if x.dim() < 3 or tuple(x.shape[-3:]) != tail:
        raise ValueError(f"expected (..., {tail[0]}, {tail[1]}, {tail[2]}), got {tuple(x.shape)}")
    lead = x.shape[:-3]
    n = 1
    for s in lead:
        n *= int(s)
    return x.reshape(1, n, *tail).contiguous(), lead


class RealVectorSHT(_TransformBase):
    """Forward real vector spherical harmonic transform (drop-in for torch_harmonics.RealVectorSHT)."""

    def plan(self, device):
        return get_plan(self.nlat, self.nlon, self.lmax, self.mmax, self.grid, self.csphase, device, vector=True)

    def forward(self, x):
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.to(torch.float32)
        x5, lead = _as_fields(x, (2, self.nlat, self.nlon))
        plan = self.plan(x.device)
        out = _VectorAnalysis.apply(x5, plan, _vector_precision(self.precision))
        return out.reshape(*lead, 2, self.lmax, self.mmax)


class InverseRealVectorSHT(_TransformBase):
    """Inverse real vector spherical harmonic transform (drop-in for torch_harmonics.InverseRealVectorSHT)."""

    def plan(self, device):
        return get_plan(self.nlat, self.nlon, self.lmax, self.mmax, self.grid, self.csphase, device, vector=True)

    def forward(self, x):
        if x.dtype != torch.complex64:
            x = x.to(torch.complex64)
        x5, lead = _as_fields(x, (2, self.lmax, self.mmax))
        plan = self.plan(x.device)
        y = _VectorSynthesis.apply(x5, plan, _vector_precision(self.precision))
        return y.reshape(*lead, 2, self.nlat, self.nlon)

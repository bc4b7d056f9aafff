"""Pointwise tail of the SFNO block on the CUDA library (SURVEY row N2): instance norm (+ GELU) and bias + GELU as single-pass kernels.

`InstanceNorm2d` is `torch.nn.InstanceNorm2d` (same constructor, parameter names `weight` / `bias`, state dict) as the reference builds it at
/root/reference/makani/models/networks/sfnonet.py:618-620 (`num_features=embed_dim, eps=1e-6, affine=True, track_running_stats=False`); on CUDA tensors
of dtype float32 / bfloat16 its forward runs `b200sht_instance_norm_forward` (csrc/norm.cu) and can fuse the GELU that follows it in
`NeuralOperatorBlock.forward` (sfnonet.py:387-392).  `bias_gelu(x, bias)` is the `+ bias -> GELU` of the 1x1-convolution stacks
(makani/models/common/layers.py:537-760).  `DistributedLayerNorm` is makani's channel layer norm (makani/mpu/layer_norm.py:256-290) on
`b200sht_layer_norm_forward` / `_backward`, also with GELU fused.  Tensors on the CPU (the oracle-backend reference arm of bench.py, the CPU golden tests) and configurations the
kernels do not cover (running statistics, other dtypes) take torch's own operators -- these layers are outside the spherical-harmonic hot path, whose
no-fallback rule (DESIGN.md section 1) is unchanged.  `B200SHT_FUSED_POINTWISE=0` switches the kernels off.
"""
import ctypes
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib

_VP = ctypes.c_void_p
_ENABLED = os.environ.get("B200SHT_FUSED_POINTWISE", "1") != "0"


def set_fused_pointwise(on):
    """switch the fused kernels on / off at run time (returns the previous setting)"""
    global _ENABLED
    old, _ENABLED = _ENABLED, bool(on)
    return old


def fused_pointwise_enabled():
    return _ENABLED


def _ptr(t):
    return _VP(t.data_ptr()) if t is not None else _VP(0)


def _dt(dtype):
    return _lib.BF16 if dtype == torch.bfloat16 else _lib.F32


def _usable(x):
    return _ENABLED and x.is_cuda and x.dim() == 4 and x.dtype in (torch.float32, torch.bfloat16) and x.shape[0] * x.shape[1] <= 65535 and x.numel() > 0


def _workspace(B, C, hw, device):
    n = int(_lib.load().b200sht_pointwise_workspace_floats(B, C, hw))
    return torch.empty(max(n, 2), dtype=torch.float32, device=device)


class _InstanceNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, gelu):
        x = x.contiguous()
        B, C, H, W = x.shape
        hw = H * W
        y = torch.empty_like(x)
        stats = torch.empty(B * C, 2, dtype=torch.float32, device=x.device)
        ws = _workspace(B, C, hw, x.device)
        w32 = weight.detach().to(torch.float32).contiguous() if weight is not None else None
        b32 = bias.detach().to(torch.float32).contiguous() if bias is not None else None
        _lib.call("b200sht_instance_norm_forward", _ptr(x), _ptr(y), _ptr(w32), _ptr(b32), _ptr(stats), _ptr(ws), _dt(x.dtype), B, C, hw, float(eps), int(gelu),
                  _lib.launch_stream(x.device))
        ctx.save_for_backward(x, w32, b32, stats)
        ctx.gelu, ctx.has_affine = int(gelu), (weight is not None, bias is not None)
        ctx.param_dtypes = (weight.dtype if weight is not None else None, bias.dtype if bias is not None else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w32, b32, stats = ctx.saved_tensors
        B, C, H, W = x.shape
        hw = H * W
        dy = dy.contiguous().to(x.dtype)
        dx = torch.empty_like(x)
        sums = torch.empty(B * C, 2, dtype=torch.float32, device=x.device)
        ws = _workspace(B, C, hw, x.device)
        _lib.call("b200sht_instance_norm_backward", _ptr(x), _ptr(dy), _ptr(dx), _ptr(w32), _ptr(b32), _ptr(stats), _ptr(sums), _ptr(ws), _dt(x.dtype), B, C, hw,
                  ctx.gelu, _lib.launch_stream(x.device))
        per_c = sums.view(B, C, 2).sum(dim=0)
        dw = per_c[:, 1].to(ctx.param_dtypes[0]) if (ctx.has_affine[0] and ctx.needs_input_grad[1]) else None
        db = per_c[:, 0].to(ctx.param_dtypes[1]) if (ctx.has_affine[1] and ctx.needs_input_grad[2]) else None
        return (dx if ctx.needs_input_grad[0] else None), dw, db, None, None


class _BiasGeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias):
        x = x.contiguous()
        B, C, H, W = x.shape
        y = torch.empty_like(x)
        b32 = bias.detach().to(torch.float32).contiguous() if bias is not None else None
        _lib.call("b200sht_bias_gelu_forward", _ptr(x), _ptr(b32), _ptr(y), _dt(x.dtype), B, C, H * W, _lib.launch_stream(x.device))
        ctx.save_for_backward(x, b32)
        ctx.bias_dtype = bias.dtype if bias is not None else None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, b32 = ctx.saved_tensors
        B, C, H, W = x.shape
        hw = H * W
        dy = dy.contiguous().to(x.dtype)
        dx = torch.empty_like(x)
        need_b = b32 is not None and ctx.needs_input_grad[1]
        sums = torch.empty(B * C, 2, dtype=torch.float32, device=x.device) if need_b else None
        ws = _workspace(B, C, hw, x.device)
        _lib.call("b200sht_bias_gelu_backward", _ptr(x), _ptr(b32), _ptr(dy), _ptr(dx), _ptr(sums), _ptr(ws), _dt(x.dtype), B, C, hw, _lib.launch_stream(x.device))
        db = sums.view(B, C, 2)[:, :, 0].sum(dim=0).to(ctx.bias_dtype) if need_b else None
        return dx, db


def bias_gelu(x, bias=None):
    """gelu(x + bias[None, :, None, None]) for x (B, C, H, W); exact (erf) GELU"""
    if _usable(x) and (bias is None or bias.is_cuda):
        return _BiasGeluFn.apply(x, bias)
    if bias is not None:
        x = x + bias.to(x.dtype).view(1, -1, 1, 1)
    return F.gelu(x)


class InstanceNorm2d(nn.InstanceNorm2d):
    """torch.nn.InstanceNorm2d whose CUDA forward / backward run on the library's kernels; `forward(x, gelu=True)` returns gelu(norm(x))."""

    def forward(self, x, gelu=False):
        if _usable(x) and not self.track_running_stats and (self.weight is None or self.weight.is_cuda):
            if x.shape[1] != self.num_features:
                raise ValueError(f"expected input with {self.num_features} channels, got {x.shape[1]}")
            return _InstanceNormFn.apply(x, self.weight, self.bias, self.eps, bool(gelu))
        y = super().forward(x)
        return F.gelu(y) if gelu else y


# ------------------------------------------------------------------------------------------------------------------------------------------------------
# Quadrature-weighted instance norm on the sphere (makani's GeometricInstanceNormS2 / DistributedGeometricInstanceNormS2).  One formula for both
# classes, on a (b, c) plane x of H x W (the local shard under h x w), latitude weights q[i], normaliser D:
#   mu = (1/D) sum q x,  var = (1/D) sum q (x - mu)^2,  r = (var + eps)^-1/2,  xhat = (x - mu) r,  y = [gelu](gamma xhat + beta)
#   dx = gamma r (g - (q/D) (S1 + xhat S2 - corr S2)),  corr = r mu (D - S) / D,  S1 = sum g, S2 = sum g xhat (unweighted, over the whole field)
# The serial class has D = 1 (its sums over the crop are not divided by the crop's weight S, as makani's `self.quadrature(xf)`), the distributed
# class D = S of the global crop.  The stages below are the kernels of csrc/norm.cu (`CudaGeometricNormStages`) or the same formula in torch ops
# (`TorchGeometricNormStages`: CPU tensors and inputs the kernels do not take); `_GeometricNormFn` strings them together with a `gather` between the
# per-shard reductions and their combination (the identity in the serial class).

def _gw_workspace(B, C, hw, device):
    n = int(_lib.load().b200sht_geometric_norm_workspace_floats(B, C, hw))
    return torch.empty(max(n, 2), dtype=torch.float32, device=device)


class CudaGeometricNormStages:
    """the stages on the library's kernels (x float32 / bfloat16, contiguous, on CUDA)"""

    def partials(self, x, q):
        B, C, H, W = x.shape
        out = torch.empty(B * C, 3, dtype=torch.float64, device=x.device)
        _lib.call("b200sht_geometric_norm_partials", _ptr(x), _ptr(q), _ptr(out), _ptr(_gw_workspace(B, C, H * W, x.device)), _dt(x.dtype), B, C, H, W,
                  _lib.launch_stream(x.device))
        return out

    def finalize(self, parts, D, eps):
        R, rows = parts.shape[:2]
        stats = torch.empty(rows, 3, dtype=torch.float32, device=parts.device)
        _lib.call("b200sht_geometric_norm_finalize", _ptr(parts.contiguous()), R, rows, float(D), float(eps), _ptr(stats), _lib.launch_stream(parts.device))
        return stats

    def apply(self, x, w32, b32, stats, gelu):
        B, C, H, W = x.shape
        y = torch.empty_like(x)
        _lib.call("b200sht_geometric_norm_apply", _ptr(x), _ptr(y), _ptr(w32), _ptr(b32), _ptr(stats), _dt(x.dtype), B, C, H, W, int(gelu),
                  _lib.launch_stream(x.device))
        return y

    def backward_sums(self, x, dy, w32, b32, stats, gelu):
        B, C, H, W = x.shape
        sums = torch.empty(B * C, 2, dtype=torch.float64, device=x.device)
        _lib.call("b200sht_geometric_norm_backward_sums", _ptr(x), _ptr(dy), _ptr(w32), _ptr(b32), _ptr(stats), _ptr(sums),
                  _ptr(_gw_workspace(B, C, H * W, x.device)), _dt(x.dtype), B, C, H, W, int(gelu), _lib.launch_stream(x.device))
        return sums

    def backward_apply(self, x, dy, w32, b32, stats, sums, q, D, gelu):
        B, C, H, W = x.shape
        dx = torch.empty_like(x)
        _lib.call("b200sht_geometric_norm_backward_apply", _ptr(x), _ptr(dy), _ptr(dx), _ptr(w32), _ptr(b32), _ptr(stats), _ptr(sums.contiguous()),
                  sums.shape[0], _ptr(q), float(D), _dt(x.dtype), B, C, H, W, int(gelu), _lib.launch_stream(x.device))
        return dx

    def param_grads(self, sums, B, C):
        dg = torch.empty(C, dtype=torch.float32, device=sums.device)
        db = torch.empty(C, dtype=torch.float32, device=sums.device)
        _lib.call("b200sht_geometric_norm_param_grads", _ptr(sums), _ptr(dg), _ptr(db), B, C, _lib.launch_stream(sums.device))
        return dg, db


def _affine(xh, w32, b32):
    C = xh.shape[1]
    z = xh * w32.view(1, C, 1, 1) if w32 is not None else xh
    return z + b32.view(1, C, 1, 1) if b32 is not None else z


class TorchGeometricNormStages:
    """the same stages in torch operators: reductions in fp64, normalisation and affine in fp32, output in the dtype of x"""

    def partials(self, x, q):
        B, C, H, W = x.shape
        xd = x.to(torch.float64).reshape(B * C, H, W)
        qd = q.to(device=x.device, dtype=torch.float64).view(1, H, 1)
        d = xd - xd[:, :1, :1]
        sq = (q.to(torch.float64).sum() * W).to(x.device).expand(B * C)
        s1 = (qd * d).sum(dim=(1, 2))
        s2 = (qd * d * d).sum(dim=(1, 2))
        pos = sq > 0
        md = torch.where(pos, s1 / torch.where(pos, sq, torch.ones_like(sq)), torch.zeros_like(s1))
        mean = torch.where(pos, xd[:, 0, 0] + md, torch.zeros_like(md))
        m2 = torch.where(pos, (s2 - s1 * md).clamp_min(0.0), torch.zeros_like(md))
        return torch.stack([sq, mean, m2], dim=1)

    def finalize(self, parts, D, eps):
        parts = parts.to(torch.float64)
        S = torch.zeros_like(parts[0, :, 0])
        m, M2 = torch.zeros_like(S), torch.zeros_like(S)
        for k in range(parts.shape[0]):      # Chan / Welford in rank order; a shard of zero weight adds nothing
            nb, mb, M2b = parts[k].unbind(1)
            n = S + nb
            safe = torch.where(nb > 0, n, torch.ones_like(n))
            delta = mb - m
            m = torch.where(nb > 0, m + delta * (nb / safe), m)
            M2 = torch.where(nb > 0, M2 + M2b + delta * delta * (S * nb / safe), M2)
            S = n
        mu = S * m / D
        var = ((M2 + S * (m - mu) ** 2) / D).clamp_min(0.0)
        r = 1.0 / torch.sqrt(var + eps)
        return torch.stack([mu, r, r * mu * (D - S) / D], dim=1).to(torch.float32)

    @staticmethod
    def _xhat(x, stats):
        B, C = x.shape[:2]
        st = stats.view(B, C, 3, 1, 1)
        return (x.to(torch.float32) - st[:, :, 0]) * st[:, :, 1]

    def apply(self, x, w32, b32, stats, gelu):
        z = _affine(self._xhat(x, stats), w32, b32)
        return (F.gelu(z) if gelu else z).to(x.dtype)

    def _g(self, x, dy, w32, b32, stats, gelu):
        xh = self._xhat(x, stats)
        g = dy.to(torch.float32)
        if gelu:
            z = _affine(xh, w32, b32)
            g = g * (0.5 * (1.0 + torch.erf(z * 0.7071067811865476)) + z * 0.3989422804014327 * torch.exp(-0.5 * z * z))
        return xh, g

    def backward_sums(self, x, dy, w32, b32, stats, gelu):
        B, C = x.shape[:2]
        xh, g = self._g(x, dy, w32, b32, stats, gelu)
        g64 = g.to(torch.float64)
        return torch.stack([g64.sum(dim=(2, 3)), (g64 * xh.to(torch.float64)).sum(dim=(2, 3))], dim=-1).reshape(B * C, 2)

    def backward_apply(self, x, dy, w32, b32, stats, sums, q, D, gelu):
        B, C, H, W = x.shape
        xh, g = self._g(x, dy, w32, b32, stats, gelu)
        tot = sums.to(torch.float64).sum(dim=0).view(B, C, 2, 1, 1)
        st = stats.view(B, C, 3, 1, 1)
        k0 = (tot[:, :, 0] - st[:, :, 2].to(torch.float64) * tot[:, :, 1]).to(torch.float32)
        s2 = tot[:, :, 1].to(torch.float32)
        qd = (q.to(device=x.device, dtype=torch.float32) * float(1.0 / D)).view(1, 1, H, 1)
        gs = st[:, :, 1] * (w32.view(1, C, 1, 1) if w32 is not None else 1.0)
        return (gs * (g - qd * (k0 + xh * s2))).to(x.dtype)

    def param_grads(self, sums, B, C):
        per_c = sums.to(torch.float64).view(B, C, 2).sum(dim=0)
        return per_c[:, 1].to(torch.float32), per_c[:, 0].to(torch.float32)


def _gather_none(t):
    return t.unsqueeze(0)


class _GeometricNormFn(torch.autograd.Function):
    """x -> y through `stages`; `gather(t)`: this shard's per-row tensor -> every shard's, stacked in a fixed rank order (the identity here on one GPU)"""

    @staticmethod
    def forward(ctx, x, weight, bias, q, D, eps, gelu, stages, gather):
        x = x.contiguous()
        w32 = weight.detach().to(torch.float32).contiguous() if weight is not None else None
        b32 = bias.detach().to(torch.float32).contiguous() if bias is not None else None
        stats = stages.finalize(gather(stages.partials(x, q)), D, eps)
        y = stages.apply(x, w32, b32, stats, gelu)
        ctx.save_for_backward(x, w32, b32, stats, q)
        ctx.D, ctx.gelu, ctx.stages, ctx.gather = D, bool(gelu), stages, gather
        ctx.param_dtypes = (weight.dtype if weight is not None else None, bias.dtype if bias is not None else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w32, b32, stats, q = ctx.saved_tensors
        B, C = x.shape[:2]
        dy = dy.contiguous().to(x.dtype)
        sums = ctx.stages.backward_sums(x, dy, w32, b32, stats, ctx.gelu)
        dx = ctx.stages.backward_apply(x, dy, w32, b32, stats, ctx.gather(sums), q, ctx.D, ctx.gelu)
        dw = db = None
        if (w32 is not None and ctx.needs_input_grad[1]) or (b32 is not None and ctx.needs_input_grad[2]):
            dg, dbt = ctx.stages.param_grads(sums, B, C)     # this shard's partial sums: dgamma = sum_b S2, dbeta = sum_b S1
            dw = dg.to(ctx.param_dtypes[0]) if (w32 is not None and ctx.needs_input_grad[1]) else None
            db = dbt.to(ctx.param_dtypes[1]) if (b32 is not None and ctx.needs_input_grad[2]) else None
        return (dx if ctx.needs_input_grad[0] else None), dw, db, None, None, None, None, None, None


_CUDA_STAGES = CudaGeometricNormStages()
_TORCH_STAGES = TorchGeometricNormStages()


class GeometricInstanceNormS2(nn.Module):
    """makani's GeometricInstanceNormS2 (same constructor, parameters `weight` / `bias`, state dict): instance norm whose statistics are sums of the
    quadrature weights of the grid over the crop.  CUDA float32 / bfloat16 inputs run on the kernels of csrc/norm.cu; `forward(x, gelu=True)` returns
    gelu(norm(x)) in the same passes."""

    def __init__(self, img_shape, crop_shape, crop_offset, grid_type, num_features, eps=1e-05, affine=False):
        super().__init__()
        from .quadrature import grid_to_quadrature_rule

        self.eps, self.affine = eps, affine
        if self.affine:
            self.weight = nn.Parameter(torch.ones(num_features))
            self.bias = nn.Parameter(torch.zeros(num_features))
        grid_to_quadrature_rule(grid_type)     # NotImplementedError for a grid without a rule, as makani
        self.img_shape, self.grid_type, self.num_features = tuple(img_shape), grid_type, num_features
        self.crop_shape = tuple(img_shape) if crop_shape is None else tuple(crop_shape)
        self.crop_offset = tuple(crop_offset)
        self._init_quadrature(None, 0, self.crop_shape[1])

    def _init_quadrature(self, h_shapes, h_rank, w_local):
        from .quadrature import crop_quadrature_np

        q64 = crop_quadrature_np(self.grid_type, self.img_shape, self.crop_shape, self.crop_offset, h_shapes, h_rank)
        self.local_shape = (len(q64), int(w_local))
        # [H_local] latitude weights, built in fp64 and held in fp32 whatever dtype the module is cast to (the kernels and the torch stages read it)
        self.register_buffer("quad_weight", torch.from_numpy(q64).to(torch.float32), persistent=False)
        self._q64 = q64

    def _apply(self, fn, recurse=True):
        super()._apply(fn, recurse)
        if self.quad_weight.dtype != torch.float32:     # module.to(dtype) / .half(): re-round the weights from fp64, keep them fp32
            self.quad_weight = torch.from_numpy(self._q64).to(device=self.quad_weight.device, dtype=torch.float32)
        return self

    def _normaliser(self):
        return 1.0

    def _gather(self):
        return _gather_none

    def _stages(self, x):
        return _CUDA_STAGES if _usable(x) and (self.weight.is_cuda if self.affine else True) else _TORCH_STAGES

    def _q(self, x):
        return self.quad_weight.to(device=x.device).contiguous()

    def forward(self, x, gelu=False):
        if x.dim() != 4 or x.shape[1] != self.num_features or tuple(x.shape[-2:]) != self.local_shape:
            raise ValueError(f"expected input of shape (B, {self.num_features}, {self.local_shape[0]}, {self.local_shape[1]}), got {tuple(x.shape)}")
        stages = self._stages(x)
        w, b = (self.weight, self.bias) if self.affine else (None, None)
        return _GeometricNormFn.apply(x, w, b, self._q(x), self._normaliser(), self.eps, bool(gelu), stages, self._gather())


# ------------------------------------------------------------------------------------------------------------------------------------------------------
# Channel layer norm (makani's DistributedLayerNorm): nn.LayerNorm(C) at every grid point of an NCHW activation, which makani computes as transpose ->
# layer_norm -> transpose -> .contiguous().  The kernels of csrc/norm.cu reduce over the strided channel axis in place: the forward reads x once and
# writes y once, the backward reads x and dy once and writes dx once, and dgamma / dbeta come from fixed-order per-CTA partials.  The layer is
# pointwise in space, so under h x w model parallelism the local shard is the whole problem and nothing is exchanged.

def _layer_norm_out_dtype(x):
    """the dtype makani's layer returns for a CUDA tensor x: layer_norm is on CUDA autocast's fp32 list, otherwise the output keeps the dtype of x"""
    return torch.float32 if torch.is_autocast_enabled("cuda") else x.dtype


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps, gelu, out_dtype):
        x = x.contiguous()
        B, C, H, W = x.shape
        y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
        stats = torch.empty(B * H * W, 2, dtype=torch.float32, device=x.device)
        w32 = weight.detach().to(torch.float32).contiguous() if weight is not None else None
        b32 = bias.detach().to(torch.float32).contiguous() if bias is not None else None
        _lib.call("b200sht_layer_norm_forward", _ptr(x), _ptr(y), _ptr(w32), _ptr(b32), _ptr(stats), _dt(x.dtype), _dt(out_dtype), B, C, H * W, float(eps),
                  int(gelu), _lib.launch_stream(x.device))
        ctx.save_for_backward(x, w32, b32, stats)
        ctx.gelu, ctx.out_dtype = int(gelu), out_dtype
        ctx.param_dtypes = (weight.dtype if weight is not None else None, bias.dtype if bias is not None else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w32, b32, stats = ctx.saved_tensors
        B, C, H, W = x.shape
        dy = dy.contiguous().to(ctx.out_dtype)
        dx = torch.empty_like(x)
        need_w = w32 is not None and ctx.needs_input_grad[1]
        need_b = b32 is not None and ctx.needs_input_grad[2]
        dw = torch.empty(C, dtype=torch.float32, device=x.device) if need_w else None
        db = torch.empty(C, dtype=torch.float32, device=x.device) if need_b else None
        ws = torch.empty(max(int(_lib.load().b200sht_layer_norm_workspace_floats(B, C, H * W)), 2), dtype=torch.float32, device=x.device)
        _lib.call("b200sht_layer_norm_backward", _ptr(x), _ptr(dy), _ptr(dx), _ptr(w32), _ptr(b32), _ptr(stats), _ptr(dw), _ptr(db), _ptr(ws), _dt(x.dtype),
                  _dt(ctx.out_dtype), B, C, H * W, ctx.gelu, _lib.launch_stream(x.device))
        dw = dw.to(ctx.param_dtypes[0]) if need_w else None
        db = db.to(ctx.param_dtypes[1]) if need_b else None
        return (dx if ctx.needs_input_grad[0] else None), dw, db, None, None, None


class DistributedLayerNorm(nn.Module):
    """makani's DistributedLayerNorm (same constructor, `.norm` submodule nn.LayerNorm, state-dict keys `norm.weight` / `norm.bias`, the same
    `is_shared_mp` / `sharded_dims_mp` tags): layer norm over the channels of an NCHW activation at every grid point, on one GPU and under h x w
    spatial model parallelism alike.  CUDA float32 / bfloat16 4-D inputs normalised over their channel axis run on the kernels of csrc/norm.cu, and
    `forward(x, gelu=True)` returns gelu(norm(x)) in the same passes; other inputs take makani's formula (transpose -> self.norm -> transpose)."""

    def __init__(self, normalized_shape, eps=1e-05, elementwise_affine=True, bias=True, device=None, dtype=None):
        super().__init__()
        self.norm = nn.LayerNorm(normalized_shape, eps=eps, elementwise_affine=elementwise_affine, bias=bias, device=device, dtype=dtype)
        if elementwise_affine:
            self.norm.weight.is_shared_mp = ["model"]
            self.norm.weight.sharded_dims_mp = [None]
            if bias:
                self.norm.bias.is_shared_mp = ["model"]
                self.norm.bias.sharded_dims_mp = [None]

    def _kernels_take(self, x):
        if not (_ENABLED and x.is_cuda and x.dim() == 4 and x.dtype in (torch.float32, torch.bfloat16) and x.numel() > 0):
            return False
        if tuple(self.norm.normalized_shape) != (x.shape[1],):
            return False
        return all(p is None or (p.is_cuda and p.dtype in (torch.float32, x.dtype)) for p in (self.norm.weight, self.norm.bias))

    def forward(self, x, gelu=False):
        if self._kernels_take(x):
            return _LayerNormFn.apply(x, self.norm.weight, self.norm.bias, self.norm.eps, bool(gelu), _layer_norm_out_dtype(x))
        y = torch.transpose(self.norm(torch.transpose(x, 1, 3)), 1, 3).contiguous()
        return F.gelu(y) if gelu else y

"""NeighborhoodAttentionS2 -- drop-in for `torch_harmonics.NeighborhoodAttentionS2`, the local attention of torch-harmonics' spherical
transformers, with the attention on the sm_90a kernels of csrc/attention.cu.  AttentionS2 -- drop-in for `torch_harmonics.AttentionS2`, the
global attention of the same family, on the wgmma flash-attention kernels of csrc/attention_global.cu (see its class docstring).

    NeighborhoodAttentionS2(in_channels, in_shape, out_shape, grid_in="equiangular", grid_out="equiangular", num_heads=1, scale=None, bias=True,
                            theta_cutoff=None, k_channels=None, out_channels=None, optimized_kernel=True)
    forward(query, key=None, value=None): query (B, C_in, *out_shape), key / value (B, C_in, *in_shape), fp32 / bf16 on a CUDA device
                                          -> float32 (B, C_v, *out_shape)

Each output point (t, p) attends to the input points within the DISCO convolution's support (`disco.support_search`: r <= (1 + 1e-3) theta_cutoff
at longitude 0, shifted by s p, s = nlon_in / nlon_out), with the quadrature-weighted softmax (DESIGN.md section 4.9, include/b200sht.h):

    q = W_q query + b_q,  k = W_k key + b_k,  v = W_v value + b_v         (1x1 projections; head h on channels [h E, (h + 1) E))
    l_n = scale <q_h(t, p), k_h(n)>,  w_i = 2 pi w_in[i] / nlon_in
    y_h(t, p) = sum_n w_i exp(l_n) v_h(n) / sum_n w_i exp(l_n),   out = W_proj y + b_proj

The neighbourhood is a K = 1 DISCO plan whose value at (t, i, j) is w_i.  The projections are cuBLAS GEMMs (torch.bmm / baddbmm; TF32 follows
torch.backends.cuda.matmul.allow_tf32) that write the point-major, channel-contiguous operands (B, H W, C) of the kernels directly.
"""
import math
import threading

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import B200ShtError, launch_stream as _stream, ptr as _ptr
from .disco import DiscoPlan, DiscoPsi, support_search
from .quadrature import _grid_np

MAX_HEAD_DIM = 64     # the kernels' largest head dimension (include/b200sht.h)


def neighbourhood(in_shape, out_shape, grid_in, grid_out, theta_cutoff):
    """The neighbourhood S(t) of every output latitude as a K = 1 DiscoPsi in (i, j) order, valued w_i = 2 pi w_in[i] / nlon_in.

    Raises ValueError when nlon_in is not a multiple of nlon_out or an output latitude has no input point within the cutoff.  Within each
    (t, i) the support must be the arc j in [-off, n - 1 - off] (mod nlon_in), off = (n - 1) / 2, or the whole ring: the kernels read it as such."""
    (nlat_in, nlon_in), (nlat_out, nlon_out) = in_shape, out_shape
    sup = support_search(in_shape, out_shape, grid_in, grid_out, theta_cutoff)
    _, w_in = _grid_np(nlat_in, grid_in)
    omega = 2.0 * np.pi * w_in / nlon_in
    row_ptr = np.zeros(nlat_out + 1, dtype=np.int64)
    cols, vals = [], []
    for t, (i, j, _, _) in enumerate(sup):
        if len(i) == 0:
            raise ValueError(f"output latitude {t} has no input point within theta_cutoff {theta_cutoff} (the cutoff is below the grid spacing)")
        starts = np.flatnonzero(np.r_[True, i[1:] != i[:-1]])
        for a, b in zip(starts, np.r_[starts[1:], len(i)]):
            n = b - a
            off = (n - 1) // 2
            if not np.array_equal(j[a:b], np.sort(np.mod(np.arange(-off, n - off), nlon_in))):
                raise ValueError(f"the support of output latitude {t} in input row {i[a]} is not a symmetric arc of longitudes")
        cols.append((i * nlon_in + j).astype(np.int32))
        vals.append(omega[i])
        row_ptr[t + 1] = row_ptr[t] + len(i)
    col = np.concatenate(cols)
    return DiscoPsi(row_ptr, np.zeros(len(col), np.int32), col, np.concatenate(vals), nlat_in, nlon_in, nlat_out, nlon_out, 1)


class AttentionPlan(DiscoPlan):
    """The K = 1 DISCO plan of a neighbourhood, with the two attention calls of the C ABI."""

    def forward_attention(self, q, k, v, heads, scale):
        """q (B, HW_out, H ek), k (B, HW_in, H ek), v (B, HW_in, H ev), fp32 contiguous -> y (B, HW_out, H ev), lse (B, H, HW_out)"""
        B = q.shape[0]
        y = torch.empty((B, q.shape[1], v.shape[2]), dtype=torch.float32, device=q.device)
        lse = torch.empty((B, heads, q.shape[1]), dtype=torch.float32, device=q.device)
        _lib.call("b200sht_attention_forward", self.handle, _ptr(q), _ptr(k), _ptr(v), _ptr(y), _ptr(lse), B, heads, q.shape[2] // heads,
                  v.shape[2] // heads, float(scale), _stream(q.device))
        return y, lse

    def backward_attention(self, q, k, v, y, lse, dy, heads, scale):
        """-> dq, dk, dv (shapes of q, k, v); dy (B, HW_out, H ev) fp32 contiguous"""
        B = q.shape[0]
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        D = torch.empty_like(lse)
        _lib.call("b200sht_attention_backward", self.handle, _ptr(q), _ptr(k), _ptr(v), _ptr(y), _ptr(lse), _ptr(dy), _ptr(dq), _ptr(dk),
                  _ptr(dv), _ptr(D), B, heads, q.shape[2] // heads, v.shape[2] // heads, float(scale), _stream(q.device))
        return dq, dk, dv


_psi_cache, _plan_cache, _cache_lock = {}, {}, threading.Lock()


def get_neighbourhood(*key):
    """neighbourhood(in_shape, out_shape, grid_in, grid_out, theta_cutoff), cached per key"""
    with _cache_lock:
        if key not in _psi_cache:
            _psi_cache[key] = neighbourhood(*key)
        return _psi_cache[key]


def get_plan(key, device):
    """the device plan of get_neighbourhood(*key), cached per key and device"""
    device = torch.device(device)
    if device.type != "cuda":
        raise B200ShtError(f"the neighbourhood attention runs on CUDA devices only (got {device}); makani_b200 has no CPU fallback")
    dkey = key + (device.index if device.index is not None else torch.cuda.current_device(),)
    with _cache_lock:
        plan = _plan_cache.get(dkey)
    if plan is None:
        plan = AttentionPlan(get_neighbourhood(*key), device)
        with _cache_lock:
            plan = _plan_cache.setdefault(dkey, plan)
    return plan


class _NeighborhoodAttention(torch.autograd.Function):
    """y = attention(q, k, v) on the plan's neighbourhood.  Saves q, k, v, y and lse."""

    @staticmethod
    def forward(ctx, q, k, v, plan, heads, scale):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        y, lse = plan.forward_attention(q, k, v, heads, scale)
        ctx.save_for_backward(q, k, v, y, lse)
        ctx.plan, ctx.heads, ctx.scale = plan, heads, scale
        return y

    @staticmethod
    def backward(ctx, dy):
        q, k, v, y, lse = ctx.saved_tensors
        dq, dk, dv = ctx.plan.backward_attention(q, k, v, y, lse, dy.to(torch.float32).contiguous(), ctx.heads, ctx.scale)
        return dq, dk, dv, None, None, None


def _project_points(x, weight, bias):
    """1x1 projection of x (B, C_in, H, W) into the point-major layout (B, H W, C_out), fp32, written by one GEMM"""
    B, C = x.shape[0], x.shape[1]
    xt = x.to(torch.float32).reshape(B, C, -1).transpose(1, 2)                     # (B, HW, C_in), a view
    wt = weight.to(torch.float32).reshape(weight.shape[0], C).t().expand(B, -1, -1)  # (B, C_in, C_out)
    if bias is None:
        return torch.bmm(xt, wt)
    return torch.baddbmm(bias.to(torch.float32).view(1, 1, -1).expand(B, xt.shape[1], -1), xt, wt)


def _project_out(y, weight, bias):
    """the output projection of the point-major y (B, HW, C_v) -> (B, C_out, HW) fp32, one GEMM"""
    B, C = y.shape[0], y.shape[2]
    wp = weight.to(torch.float32).reshape(weight.shape[0], C).expand(B, -1, -1)
    if bias is None:
        return torch.bmm(wp, y.transpose(1, 2))
    return torch.baddbmm(bias.to(torch.float32).view(1, -1, 1).expand(B, -1, y.shape[1]), wp, y.transpose(1, 2))


class NeighborhoodAttentionS2(nn.Module):
    """Neighbourhood attention on the sphere (drop-in for torch_harmonics.NeighborhoodAttentionS2).

    Parameters q_weights, k_weights (C_k, C_in, 1, 1), v_weights (C_v, C_in, 1, 1), proj_weights (C_v, C_v, 1, 1), all xavier-uniform; with
    bias=True zero q_bias, k_bias (C_k,) and v_bias, proj_bias (C_v,).  C_k = k_channels or in_channels, C_v = out_channels or in_channels, both
    divisible by num_heads; head dims up to 64.  scale defaults to 1 / sqrt(C_k / num_heads) and multiplies the logits.  The neighbourhood and
    the quadrature are non-persistent buffers (a state dict holds the parameters only).  optimized_kernel is accepted and has no effect."""

    def __init__(self, in_channels, in_shape, out_shape, grid_in="equiangular", grid_out="equiangular", num_heads=1, scale=None, bias=True,
                 theta_cutoff=None, k_channels=None, out_channels=None, optimized_kernel=True):
        super().__init__()
        if theta_cutoff is None:
            raise ValueError("NeighborhoodAttentionS2 needs an explicit theta_cutoff (the default cutoff is not implemented)")
        if theta_cutoff <= 0:
            raise ValueError(f"theta_cutoff must be positive, got {theta_cutoff}")
        self.in_channels = in_channels
        self.k_channels = k_channels if k_channels is not None else in_channels
        self.out_channels = out_channels if out_channels is not None else in_channels
        self.num_heads = num_heads
        if num_heads < 1 or self.k_channels % num_heads or self.out_channels % num_heads:
            raise ValueError(f"k_channels {self.k_channels} and out_channels {self.out_channels} must be divisible by num_heads {num_heads}")
        ek, ev = self.k_channels // num_heads, self.out_channels // num_heads
        if max(ek, ev) > MAX_HEAD_DIM:
            raise NotImplementedError(f"head dims {ek}, {ev}: the neighbourhood attention kernels serve head dims up to {MAX_HEAD_DIM}")
        self.nlat_in, self.nlon_in = in_shape
        self.nlat_out, self.nlon_out = out_shape
        if self.nlon_in % self.nlon_out:
            raise ValueError(f"nlon_in {self.nlon_in} must be a multiple of nlon_out {self.nlon_out}")
        self.grid_in, self.grid_out, self.theta_cutoff = grid_in, grid_out, float(theta_cutoff)
        self.scale = float(scale) if scale is not None else 1.0 / math.sqrt(ek)
        self.optimized_kernel = optimized_kernel
        self._key = (tuple(in_shape), tuple(out_shape), grid_in, grid_out, float(theta_cutoff))
        psi = get_neighbourhood(*self._key)
        self.register_buffer("psi_row_ptr", torch.from_numpy(psi.row_ptr), persistent=False)
        self.register_buffer("psi_col_idx", torch.from_numpy(psi.col), persistent=False)
        self.register_buffer("quad_weights", torch.from_numpy(2.0 * np.pi * _grid_np(self.nlat_in, grid_in)[1] / self.nlon_in), persistent=False)

        def xavier(co, ci):
            w = torch.empty(co, ci, 1, 1)
            nn.init.xavier_uniform_(w)
            return nn.Parameter(w)

        self.q_weights = xavier(self.k_channels, in_channels)
        self.k_weights = xavier(self.k_channels, in_channels)
        self.v_weights = xavier(self.out_channels, in_channels)
        self.proj_weights = xavier(self.out_channels, self.out_channels)
        if bias:
            self.q_bias = nn.Parameter(torch.zeros(self.k_channels))
            self.k_bias = nn.Parameter(torch.zeros(self.k_channels))
            self.v_bias = nn.Parameter(torch.zeros(self.out_channels))
            self.proj_bias = nn.Parameter(torch.zeros(self.out_channels))
        else:
            self.q_bias = self.k_bias = self.v_bias = self.proj_bias = None

    def extra_repr(self):
        return (f"in_channels={self.in_channels}, k_channels={self.k_channels}, out_channels={self.out_channels}, num_heads={self.num_heads}, "
                f"in_shape={(self.nlat_in, self.nlon_in)}, out_shape={(self.nlat_out, self.nlon_out)}, theta_cutoff={self.theta_cutoff}")

    def plan(self, device):
        return get_plan(self._key, device)

    def _check(self, x, shape, what):
        if not x.is_cuda:
            raise B200ShtError(f"{type(self).__name__} runs on CUDA devices only; makani_b200 has no CPU fallback")
        if x.dim() != 4 or x.shape[1] != self.in_channels or tuple(x.shape[2:]) != shape:
            raise ValueError(f"{what}: expected (B, {self.in_channels}, {shape[0]}, {shape[1]}), got {tuple(x.shape)}")

    def forward(self, query, key=None, value=None):
        if (key is None or value is None) and (self.nlat_in, self.nlon_in) != (self.nlat_out, self.nlon_out):
            raise ValueError("key and value default to query, which needs in_shape == out_shape")
        key = query if key is None else key
        value = query if value is None else value
        self._check(query, (self.nlat_out, self.nlon_out), "query")
        self._check(key, (self.nlat_in, self.nlon_in), "key")
        self._check(value, (self.nlat_in, self.nlon_in), "value")
        if key.shape[0] != query.shape[0] or value.shape[0] != query.shape[0]:
            raise ValueError("query, key and value must have the same batch size")
        B = query.shape[0]
        q = _project_points(query, self.q_weights, self.q_bias)
        k = _project_points(key, self.k_weights, self.k_bias)
        v = _project_points(value, self.v_weights, self.v_bias)
        y = _NeighborhoodAttention.apply(q, k, v, self.plan(query.device), self.num_heads, self.scale)   # (B, HW_out, C_v)
        return _project_out(y, self.proj_weights, self.proj_bias).view(B, self.out_channels, self.nlat_out, self.nlon_out)


# ------------------------------------------------------------------------------------------------------------------- global attention
GLOBAL_MAX_HEAD_DIM = 128   # head dims served by csrc/attention_global.cu: multiples of 8 up to this


def _global_precision():
    """TF32 wgmma when torch allows TF32 matmuls, otherwise 3 x TF32 operand splitting in the same kernels"""
    return _lib.PREC_TF32 if torch.backends.cuda.matmul.allow_tf32 else _lib.PREC_FP32X3


def _global_workspace(BH, nq, nk, dqk, dv, precision, backward, device):
    n = _lib.load().b200sht_attention_global_workspace_floats(BH, nq, nk, dqk, dv, precision, int(backward))
    if n < 0:
        raise B200ShtError(f"global attention: no workspace for head dims {dqk}, {dv}")
    return torch.empty(n, dtype=torch.float32, device=device)


def global_attention_forward(q, k, v, bias, scale, precision):
    """q (B, H, nq, dqk), k (B, H, nk, dqk), v (B, H, dv, nk), bias (nk,): fp32 contiguous CUDA tensors -> o (B, H, nq, dv), lse (B, H, nq)"""
    B, H, nq, dqk = q.shape
    dv, nk = v.shape[2], v.shape[3]
    o = torch.empty((B, H, nq, dv), dtype=torch.float32, device=q.device)
    lse = torch.empty((B, H, nq), dtype=torch.float32, device=q.device)
    ws = _global_workspace(B * H, nq, nk, dqk, dv, precision, False, q.device)
    _lib.call("b200sht_attention_global_forward", _ptr(q), _ptr(k), _ptr(v), _ptr(bias), _ptr(o), _ptr(lse), B * H, nq, nk, dqk, dv,
              float(scale), precision, _ptr(ws), _stream(q.device))
    return o, lse


def global_attention_backward(q, k, v, bias, o, lse, do, scale, precision):
    """-> dq, dk, dv (shapes of q, k, v); do (B, H, nq, dv) fp32 contiguous"""
    B, H, nq, dqk = q.shape
    dv, nk = v.shape[2], v.shape[3]
    dq, dk, dvt = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    ws = _global_workspace(B * H, nq, nk, dqk, dv, precision, True, q.device)
    _lib.call("b200sht_attention_global_backward", _ptr(q), _ptr(k), _ptr(v), _ptr(bias), _ptr(o), _ptr(lse), _ptr(do), _ptr(dq), _ptr(dk),
              _ptr(dvt), B * H, nq, nk, dqk, dv, float(scale), precision, _ptr(ws), _stream(q.device))
    return dq, dk, dvt


def global_attention_rowdot(o, do):
    """D = rowsum(do o): o, do (B, H, nq, dv) fp32 contiguous -> D (B, H, nq), the first stage of the backward"""
    D = torch.empty(o.shape[:3], dtype=torch.float32, device=o.device)
    _lib.call("b200sht_attention_global_rowdot", _ptr(o), _ptr(do), _ptr(D), D.numel(), o.shape[3], _stream(o.device))
    return D


def global_attention_backward_kv(q, k, v, bias, lse, D, do, scale, precision):
    """dk, dv of the given keys against the given queries: q, do (B, H, nq, .), lse, D (B, H, nq) of the queries; k (B, H, nk, dqk),
    v (B, H, dv, nk), bias (nk,) of the keys; fp32 contiguous -> dk, dv (shapes of k, v)"""
    B, H, nq, dqk = q.shape
    dv, nk = v.shape[2], v.shape[3]
    dk, dvt = torch.empty_like(k), torch.empty_like(v)
    ws = _global_workspace(B * H, nq, nk, dqk, dv, precision, True, q.device)
    _lib.call("b200sht_attention_global_backward_kv", _ptr(q), _ptr(k), _ptr(v), _ptr(bias), _ptr(lse), _ptr(D), _ptr(do), _ptr(dk), _ptr(dvt),
              B * H, nq, nk, dqk, dv, float(scale), precision, _ptr(ws), _stream(q.device))
    return dk, dvt


def global_attention_backward_q(q, k, v, bias, lse, D, do, scale, precision):
    """dq of the given queries against the given keys (operands as global_attention_backward_kv) -> dq (shape of q)"""
    B, H, nq, dqk = q.shape
    dv, nk = v.shape[2], v.shape[3]
    dq = torch.empty_like(q)
    ws = _global_workspace(B * H, nq, nk, dqk, dv, precision, True, q.device)
    _lib.call("b200sht_attention_global_backward_q", _ptr(q), _ptr(k), _ptr(v), _ptr(bias), _ptr(lse), _ptr(D), _ptr(do), _ptr(dq),
              B * H, nq, nk, dqk, dv, float(scale), precision, _ptr(ws), _stream(q.device))
    return dq


class _GlobalAttention(torch.autograd.Function):
    """o = softmax(scale q k^T + bias) v per head.  Saves q, k, v, o and lse."""

    @staticmethod
    def forward(ctx, q, k, v, bias, scale, precision):
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        o, lse = global_attention_forward(q, k, v, bias, scale, precision)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.bias, ctx.scale, ctx.precision = bias, scale, precision
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        dq, dk, dv = global_attention_backward(q, k, v, ctx.bias, o, lse, do.to(torch.float32).contiguous(), ctx.scale, ctx.precision)
        return dq, dk, dv, None, None, None


def _project_channels(x, weight, bias):
    """1x1 projection of x (B, C_in, H, W) into the channel-major (B, C_out, H W), fp32, one GEMM"""
    B, C = x.shape[0], x.shape[1]
    xf = x.to(torch.float32).reshape(B, C, -1)
    w = weight.to(torch.float32).reshape(weight.shape[0], C).expand(B, -1, -1)
    if bias is None:
        return torch.bmm(w, xf)
    return torch.baddbmm(bias.to(torch.float32).view(1, -1, 1).expand(B, -1, xf.shape[2]), w, xf)


class AttentionS2(nn.Module):
    """Global attention on the sphere (drop-in for torch_harmonics.AttentionS2).

    AttentionS2(in_channels, num_heads, in_shape, out_shape, grid_in="equiangular", grid_out="equiangular", scale=None, bias=True,
                k_channels=None, out_channels=None, drop_rate=0.0)
    forward(query, key=None, value=None): query (B, C_in, *out_shape), key / value (B, C_in, *in_shape), fp32 / bf16 on a CUDA device
                                          -> float32 (B, C_v, *out_shape)

    Every output point attends to every input point, with the quadrature weight of the key as a float mask (SDPA with attn_mask = log w):

        q = W_q query + b_q,  k = W_k key + b_k,  v = W_v value + b_v          (1x1 projections; head h on channels [h E, (h + 1) E))
        y_h(i) = softmax_j(scale <q_h(i), k_h(j)> + log w_j) v_h(j),  w_j = 2 pi w_in[lat(j)] / nlon_in,  out = W_proj y + b_proj

    A key of zero quadrature weight drops out (bias -inf).  Parameters as NeighborhoodAttentionS2's: q_weights, k_weights (C_k, C_in, 1, 1),
    v_weights (C_v, C_in, 1, 1), proj_weights (C_v, C_v, 1, 1), xavier-uniform; with bias=True zero q_bias, k_bias (C_k,), v_bias,
    proj_bias (C_v,).  Head dims C_k / num_heads and C_v / num_heads must be multiples of 8 up to 128.  scale defaults to
    1 / sqrt(C_k / num_heads).  The key bias is a non-persistent buffer (a state dict holds the parameters only).  drop_rate > 0 is accepted
    and raises NotImplementedError when it would drop (in training).  The projections are cuBLAS GEMMs; the attention runs on TF32 wgmma when
    torch.backends.cuda.matmul.allow_tf32, otherwise on 3 x TF32 in the same kernels (fp32 accuracy)."""

    def __init__(self, in_channels, num_heads, in_shape, out_shape, grid_in="equiangular", grid_out="equiangular", scale=None, bias=True,
                 k_channels=None, out_channels=None, drop_rate=0.0):
        super().__init__()
        self.in_channels = in_channels
        self.k_channels = k_channels if k_channels is not None else in_channels
        self.out_channels = out_channels if out_channels is not None else in_channels
        self.num_heads = num_heads
        if num_heads < 1 or self.k_channels % num_heads or self.out_channels % num_heads:
            raise ValueError(f"k_channels {self.k_channels} and out_channels {self.out_channels} must be divisible by num_heads {num_heads}")
        ek, ev = self.k_channels // num_heads, self.out_channels // num_heads
        for e in (ek, ev):
            if e % 8 or e > GLOBAL_MAX_HEAD_DIM:
                raise NotImplementedError(f"head dims {ek}, {ev}: the global attention kernels serve multiples of 8 up to {GLOBAL_MAX_HEAD_DIM}")
        self.nlat_in, self.nlon_in = in_shape
        self.nlat_out, self.nlon_out = out_shape
        self.grid_in, self.grid_out = grid_in, grid_out
        self.scale = float(scale) if scale is not None else 1.0 / math.sqrt(ek)
        self.drop_rate = float(drop_rate)
        _grid_np(self.nlat_out, grid_out)   # validates the output grid name
        omega = 2.0 * np.pi * _grid_np(self.nlat_in, grid_in)[1] / self.nlon_in
        if not np.any(omega > 0):
            raise ValueError(f"every key of the {grid_in} grid {tuple(in_shape)} has zero quadrature weight: no query has a key to attend to")
        with np.errstate(divide="ignore"):
            log_w = np.where(omega > 0, np.log(np.where(omega > 0, omega, 1.0)), -np.inf)
        self.register_buffer("key_bias", torch.from_numpy(np.repeat(log_w, self.nlon_in).astype(np.float32)), persistent=False)

        def xavier(co, ci):
            w = torch.empty(co, ci, 1, 1)
            nn.init.xavier_uniform_(w)
            return nn.Parameter(w)

        self.q_weights = xavier(self.k_channels, in_channels)
        self.k_weights = xavier(self.k_channels, in_channels)
        self.v_weights = xavier(self.out_channels, in_channels)
        self.proj_weights = xavier(self.out_channels, self.out_channels)
        if bias:
            self.q_bias = nn.Parameter(torch.zeros(self.k_channels))
            self.k_bias = nn.Parameter(torch.zeros(self.k_channels))
            self.v_bias = nn.Parameter(torch.zeros(self.out_channels))
            self.proj_bias = nn.Parameter(torch.zeros(self.out_channels))
        else:
            self.q_bias = self.k_bias = self.v_bias = self.proj_bias = None

    def extra_repr(self):
        return (f"in_channels={self.in_channels}, k_channels={self.k_channels}, out_channels={self.out_channels}, num_heads={self.num_heads}, "
                f"in_shape={(self.nlat_in, self.nlon_in)}, out_shape={(self.nlat_out, self.nlon_out)}, drop_rate={self.drop_rate}")

    def _check(self, x, shape, what):
        if not x.is_cuda:
            raise B200ShtError(f"{type(self).__name__} runs on CUDA devices only; makani_b200 has no CPU fallback")
        if x.dtype not in (torch.float32, torch.bfloat16):
            raise TypeError(f"{what}: float32 or bfloat16 inputs are served, got {x.dtype}")
        if x.dim() != 4 or x.shape[1] != self.in_channels or tuple(x.shape[2:]) != shape:
            raise ValueError(f"{what}: expected (B, {self.in_channels}, {shape[0]}, {shape[1]}), got {tuple(x.shape)}")

    def forward(self, query, key=None, value=None):
        if (key is None or value is None) and (self.nlat_in, self.nlon_in) != (self.nlat_out, self.nlon_out):
            raise ValueError("key and value default to query, which needs in_shape == out_shape")
        if self.training and self.drop_rate > 0.0:
            raise NotImplementedError("AttentionS2: attention dropout (drop_rate > 0 in training) is not implemented")
        key = query if key is None else key
        value = query if value is None else value
        self._check(query, (self.nlat_out, self.nlon_out), "query")
        self._check(key, (self.nlat_in, self.nlon_in), "key")
        self._check(value, (self.nlat_in, self.nlon_in), "value")
        if key.shape[0] != query.shape[0] or value.shape[0] != query.shape[0]:
            raise ValueError("query, key and value must have the same batch size")
        B, H = query.shape[0], self.num_heads
        ek, ev = self.k_channels // H, self.out_channels // H
        nq, nk = self.nlat_out * self.nlon_out, self.nlat_in * self.nlon_in
        q = _project_channels(query, self.q_weights, self.q_bias).view(B, H, ek, nq).transpose(2, 3)   # (B, H, nq, ek)
        k = _project_channels(key, self.k_weights, self.k_bias).view(B, H, ek, nk).transpose(2, 3)
        v = _project_channels(value, self.v_weights, self.v_bias).view(B, H, ev, nk)                    # NCHW order of each head
        o = _GlobalAttention.apply(q, k, v, self.key_bias.to(query.device), self.scale, _global_precision())   # (B, H, nq, ev)
        y = o.transpose(2, 3).reshape(B, self.out_channels, nq)
        wp = self.proj_weights.to(torch.float32).reshape(self.out_channels, self.out_channels).expand(B, -1, -1)
        out = torch.bmm(wp, y) if self.proj_bias is None else torch.baddbmm(self.proj_bias.to(torch.float32).view(1, -1, 1).expand(B, -1, nq), wp, y)
        return out.view(B, self.out_channels, self.nlat_out, self.nlon_out)

"""fp64 restatement of AttentionS2's contract (DESIGN.md section 4.10): dense scaled dot-product attention with the log quadrature weight of
each key as a float mask, in plain torch, differentiable by autograd.  Test and measurement infrastructure only; the product path does not
import it.

    l_ij = scale <q_i, k_j> + log w_j,   o_i = sum_j exp(l_ij) v_j / sum_j exp(l_ij),   lse_i = log sum_j exp(l_ij)
    w_j = 2 pi w_in[lat(j)] / nlon_in (makani_b200.quadrature), -inf bias for a zero weight

Per-head operands in the kernels' layouts: q (B, H, nq, dqk), k (B, H, nk, dqk), v (B, H, dv, nk) -> o (B, H, nq, dv), lse (B, H, nq).
"""
import numpy as np
import torch

from makani_b200.quadrature import _grid_np


def key_bias(nlat_in, nlon_in, grid_in):
    """log w_j per input point in row-major (lat, lon) order, float64, -inf where the weight is zero"""
    omega = 2.0 * np.pi * _grid_np(nlat_in, grid_in)[1] / nlon_in
    with np.errstate(divide="ignore"):
        return torch.from_numpy(np.repeat(np.log(np.maximum(omega, 0.0)), nlon_in))


def attention(q, k, v, bias, scale, rows=None):
    """o, lse of the contract (in the dtype of q), for the query indices `rows` (default: all)"""
    if rows is not None:
        q = q[:, :, rows]
    lg = scale * (q @ k.transpose(-1, -2)) + bias.to(q.dtype)
    m = lg.amax(-1, keepdim=True).detach()   # the softmax does not depend on m
    e = torch.exp(lg - m)
    s = e.sum(-1, keepdim=True)
    return (e @ v.transpose(-1, -2)) / s, (m + torch.log(s)).squeeze(-1)


def project(x, weight, bias):
    """1x1 projection of x (B, C_in, H, W) to the channel-major (B, C_out, H W)"""
    B, C = x.shape[0], x.shape[1]
    y = weight.reshape(weight.shape[0], C) @ x.reshape(B, C, -1)
    return y if bias is None else y + bias.view(1, -1, 1)


def module_forward(params, query, key, value, grid_in, heads, scale, rows=None):
    """AttentionS2.forward in the dtype of `params` (a dict with the module's parameter names) -> (B, C_v, nq) at the query indices `rows`
    (default: all, reshaped to (B, C_v, nlat_out, nlon_out))"""
    B = query.shape[0]
    nlat_in, nlon_in = key.shape[-2:]
    q = project(query, params["q_weights"], params.get("q_bias"))
    k = project(key, params["k_weights"], params.get("k_bias"))
    v = project(value, params["v_weights"], params.get("v_bias"))
    ek, ev = q.shape[1] // heads, v.shape[1] // heads
    q = q.view(B, heads, ek, -1).transpose(2, 3)
    k = k.view(B, heads, ek, -1).transpose(2, 3)
    v = v.view(B, heads, ev, -1)
    o, _ = attention(q, k, v, key_bias(nlat_in, nlon_in, grid_in).to(q.device), scale, rows)
    y = o.transpose(2, 3).reshape(B, heads * ev, -1)
    wp = params["proj_weights"]
    out = wp.reshape(wp.shape[0], -1) @ y
    if params.get("proj_bias") is not None:
        out = out + params["proj_bias"].view(1, -1, 1)
    return out if rows is not None else out.view(B, wp.shape[0], *query.shape[-2:])

"""fp64 restatement of NeighborhoodAttentionS2's contract (DESIGN.md section 4.9): a gather over the neighbourhood CSR and a segment softmax in
plain torch, differentiable by autograd.  Test and measurement infrastructure only; the product path does not import it.

    N(t, p) = { (i, (j + s p) mod nlon_in) : i * nlon_in + j in col[row_ptr[t] : row_ptr[t + 1]] },  s = nlon_in / nlon_out
    l_n = scale <q_h(t, p), k_h(n)>,  y_h(t, p) = sum_n w_i exp(l_n) v_h(n) / sum_n w_i exp(l_n),  lse_h(t, p) = log sum_n w_i exp(l_n)

Operands are point-major: q (B, nlat_out nlon_out, H E_k), k (B, nlat_in nlon_in, H E_k), v (B, nlat_in nlon_in, H E_v); y (B, P, H E_v) and
lse (B, H, P) for the P = len(rows) nlon_out output points of the requested output rows.
"""
import numpy as np
import torch


def pairs(row_ptr, col, nlon_in, nlon_out, t):
    """(p, n) index arrays of every (output longitude p, neighbour n = input point index) of output row t"""
    s = nlon_in // nlon_out
    c = np.asarray(col[row_ptr[t] : row_ptr[t + 1]], dtype=np.int64)
    i, j = c // nlon_in, c % nlon_in
    p = np.arange(nlon_out)
    n = i[None, :] * nlon_in + (j[None, :] + s * p[:, None]) % nlon_in
    return np.repeat(p, len(c)), n.reshape(-1)


def attention(q, k, v, row_ptr, col, omega, nlon_in, nlon_out, heads, scale, rows=None):
    """y, lse of the contract for output rows `rows` (default: all), one output row at a time.  omega: (nlat_in,) quadrature weights."""
    B = q.shape[0]
    ek, ev = q.shape[2] // heads, v.shape[2] // heads
    qh, kh, vh = q.view(B, -1, heads, ek), k.view(B, -1, heads, ek), v.view(B, -1, heads, ev)
    omega = torch.as_tensor(omega, dtype=q.dtype, device=q.device)
    nlat_out = len(row_ptr) - 1
    ys, lses = [], []
    for t in range(nlat_out) if rows is None else rows:
        p, n = pairs(row_ptr, col, nlon_in, nlon_out, t)
        seg = torch.from_numpy(p).to(q.device)
        n = torch.from_numpy(n).to(q.device)
        lg = scale * (qh[:, t * nlon_out + seg] * kh[:, n]).sum(-1)                            # (B, pairs, H)
        m = torch.full((B, nlon_out, heads), -torch.inf, dtype=q.dtype, device=q.device)
        m = m.scatter_reduce(1, seg.view(1, -1, 1).expand_as(lg), lg.detach(), "amax")         # the softmax does not depend on m
        e = omega[n // nlon_in].view(1, -1, 1) * torch.exp(lg - m[:, seg])
        s = torch.zeros(B, nlon_out, heads, dtype=q.dtype, device=q.device).index_add(1, seg, e)
        y = torch.zeros(B, nlon_out, heads, ev, dtype=q.dtype, device=q.device).index_add(1, seg, e[..., None] * vh[:, n])
        ys.append((y / s[..., None]).reshape(B, nlon_out, heads * ev))
        lses.append((m + torch.log(s)).permute(0, 2, 1))
    return torch.cat(ys, 1), torch.cat(lses, 2)


def project(x, weight, bias):
    """1x1 projection of x (B, C_in, H, W) to the point-major (B, H W, C_out)"""
    B, C = x.shape[0], x.shape[1]
    y = x.reshape(B, C, -1).transpose(1, 2) @ weight.reshape(weight.shape[0], C).t()
    return y if bias is None else y + bias


def module_forward(params, query, key, value, row_ptr, col, omega, heads, scale, rows=None):
    """NeighborhoodAttentionS2.forward in the dtype of `params` (a dict with the module's parameter names) -> (B, C_v, len(rows), nlon_out)"""
    nlon_out, nlon_in = query.shape[-1], key.shape[-1]
    q = project(query, params["q_weights"], params.get("q_bias"))
    k = project(key, params["k_weights"], params.get("k_bias"))
    v = project(value, params["v_weights"], params.get("v_bias"))
    y, _ = attention(q, k, v, row_ptr, col, omega, nlon_in, nlon_out, heads, scale, rows)
    wp = params["proj_weights"]
    out = y @ wp.reshape(wp.shape[0], -1).t()
    if params.get("proj_bias") is not None:
        out = out + params["proj_bias"]
    B = query.shape[0]
    return out.transpose(1, 2).reshape(B, wp.shape[0], -1, nlon_out)

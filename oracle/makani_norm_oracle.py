"""fp64 oracle of makani's quadrature-weighted instance norms on the sphere, restated from their formulas:
GeometricInstanceNormS2 (makani/models/common/layer_norm.py:30-152), DistributedGeometricInstanceNormS2 (makani/mpu/layer_norm.py:173-253) and the
weights of GridQuadrature (makani/utils/grids.py:97-191, normalize=True), as full H x W tensors with the crop and the per-rank slices.

    serial      : mu = sum q x,            var = sum q (x - mu)^2            (sums over the crop; not divided by its weight S)
    distributed : mu = (1/D) sum q x,      var = (1/D) sum q (x - mu)^2      (D = S, the weight of the whole global crop)
    y = (x - mu) / sqrt(var + eps) [* gamma + beta] [-> gelu]

`backward` is the closed form of dx, dgamma, dbeta (DESIGN.md section 4.6b) that the kernels implement; `OracleStages` are the per-rank stages of
makani_b200.norm in fp64, the stand-in for the kernels in the gloo tests of the distributed class.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

RULES = {"euclidean": "uniform", "equiangular": "naive", "legendre-gauss": "legendre-gauss", "clenshaw-curtiss": "clenshaw-curtiss",
         "weatherbench2": "weatherbench2"}


def split_shapes(n, k):
    """torch_harmonics' compute_split_shapes: ceil(n / k) for the first k - 1 ranks, the rest last (floor split if the last would be empty)"""
    if k == 1:
        return [n]
    c = -(-n // k)
    last = n - c * (k - 1)
    if last <= 0:
        c = n // k
        last = n - c * (k - 1)
    return [c] * (k - 1) + [last]


def _lat_weights(rule, H):
    """the unnormalised per-latitude factor of each rule (the longitude factor 2 pi / W is common to all and cancels or is applied below)"""
    if rule == "naive":
        return np.maximum(np.sin(np.linspace(0.0, math.pi, H)), 0.0)
    if rule == "legendre-gauss":
        return np.polynomial.legendre.leggauss(H)[1]
    if rule == "clenshaw-curtiss":
        # Clenshaw-Curtis on H points of [-1, 1]: w_k = c_k / (H - 1) (1 - sum_j b_j cos(2 pi j k / (H - 1)) / (4 j^2 - 1)) by direct summation
        n = H - 1
        w = np.empty(H)
        for k in range(H):
            s = 0.0
            for j in range(1, n // 2 + 1):
                b = 1.0 if 2 * j == n else 2.0
                s += b * math.cos(2.0 * math.pi * j * k / n) / (4.0 * j * j - 1.0)
            w[k] = (1.0 if k in (0, n) else 2.0) * (1.0 - s) / n
        return w
    if rule == "weatherbench2":
        lats = np.linspace(0.0, math.pi, H)
        edges = np.concatenate([[0.0], (lats[:-1] + lats[1:]) / 2.0, [math.pi]])
        return np.cos(edges[:-1]) - np.cos(edges[1:])
    if rule == "uniform":
        return np.ones(H)
    raise ValueError(rule)


def grid_quadrature(grid_type, img_shape, crop_shape=None, crop_offset=(0, 0), h=1, ih=0, w=1, iw=0):
    """fp64 (H_local, W_local) weights of one rank's slice (h x w grid, rank (ih, iw)) of the crop; the full H x W grid sums to 1"""
    if grid_type not in RULES:
        raise NotImplementedError(grid_type)
    H, W = img_shape
    crop_shape = img_shape if crop_shape is None else crop_shape
    q = np.tile(_lat_weights(RULES[grid_type], H)[:, None], (1, W))
    q = q / q.sum()
    hs, ws = split_shapes(crop_shape[0], h), split_shapes(crop_shape[1], w)
    h0, w0 = crop_offset[0] + sum(hs[:ih]), crop_offset[1] + sum(ws[:iw])
    return torch.from_numpy(np.ascontiguousarray(q[h0:h0 + hs[ih], w0:w0 + ws[iw]]))


def forward(x, q, eps, weight=None, bias=None, gelu=False, D=1.0):
    """x (B, C, H, W) fp64 (autograd-able), q (H, W): the restated formula with normaliser D"""
    q = q.to(x.dtype)
    mu = (q * x).sum(dim=(-2, -1), keepdim=True) / D
    var = (q * (x - mu) ** 2).sum(dim=(-2, -1), keepdim=True) / D
    y = (x - mu) / torch.sqrt(var + eps)
    if weight is not None:
        y = y * weight.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)
    return F.gelu(y) if gelu else y


def serial(x, q, eps, weight=None, bias=None, gelu=False):
    return forward(x, q, eps, weight, bias, gelu, D=1.0)


def distributed(x, q, eps, weight=None, bias=None, gelu=False):
    """the distributed class on the whole global crop: D = its weight"""
    return forward(x, q, eps, weight, bias, gelu, D=float(q.sum()))


def backward(x, dy, q, eps, weight=None, bias=None, gelu=False, D=1.0):
    """closed form: dx = gamma r (g - (q/D) (S1 + xhat S2 - r mu S2 (D - S) / D)), dgamma = sum_b S2, dbeta = sum_b S1 (S1, S2 unweighted)"""
    q = q.to(x.dtype)
    S = q.sum()
    mu = (q * x).sum(dim=(-2, -1), keepdim=True) / D
    var = (q * (x - mu) ** 2).sum(dim=(-2, -1), keepdim=True) / D
    r = 1.0 / torch.sqrt(var + eps)
    xh = (x - mu) * r
    C = x.shape[1]
    gam = weight.view(1, C, 1, 1) if weight is not None else torch.ones(1, C, 1, 1, dtype=x.dtype)
    g = dy
    if gelu:
        z = xh * gam + (bias.view(1, C, 1, 1) if bias is not None else 0.0)
        g = dy * (0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi))
    S1 = g.sum(dim=(-2, -1), keepdim=True)
    S2 = (g * xh).sum(dim=(-2, -1), keepdim=True)
    dx = gam * r * (g - (q / D) * (S1 + xh * S2 - r * mu * S2 * (D - S) / D))
    return dx, S2.sum(dim=0).flatten(), S1.sum(dim=0).flatten()


class OracleStages:
    """makani_b200.norm's per-rank stages in fp64 from the formulas (inputs of any float dtype; outputs in the dtype of x)"""

    def __init__(self):
        self.last_stats = None

    def partials(self, x, q):
        B, C, H, W = x.shape
        xd = x.double().reshape(B * C, H, W)
        qd = q.double().view(1, H, 1).expand(1, H, W)
        sq = qd.sum().expand(B * C)
        mean = (qd * xd).sum(dim=(1, 2)) / sq if float(qd.sum()) > 0 else torch.zeros(B * C, dtype=torch.float64)
        m2 = (qd * (xd - mean.view(-1, 1, 1)) ** 2).sum(dim=(1, 2))
        return torch.stack([sq, mean, m2], dim=1)

    def finalize(self, parts, D, eps):
        S = torch.zeros(parts.shape[1], dtype=torch.float64)
        m, M2 = torch.zeros_like(S), torch.zeros_like(S)
        for k in range(parts.shape[0]):
            nb, mb, M2b = parts[k].double().unbind(1)
            if float(nb.max()) <= 0.0:
                continue
            n = S + nb
            delta = mb - m
            m = m + delta * nb / n
            M2 = M2 + M2b + delta * delta * S * nb / n
            S = n
        mu = S * m / D
        var = (M2 + S * (m - mu) ** 2) / D
        r = 1.0 / torch.sqrt(var + eps)
        self.last_stats = torch.stack([mu, r, r * mu * (D - S) / D], dim=1)
        return self.last_stats

    def _xh_g(self, x, dy, w, b, stats, gelu):
        B, C = x.shape[:2]
        st = stats.double().view(B, C, 3, 1, 1)
        xh = (x.double() - st[:, :, 0]) * st[:, :, 1]
        gam = w.double().view(1, C, 1, 1) if w is not None else 1.0
        z = xh * gam + (b.double().view(1, C, 1, 1) if b is not None else 0.0)
        g = None
        if dy is not None:
            g = dy.double()
            if gelu:
                g = g * (0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi))
        return xh, z, g, st, gam

    def apply(self, x, w, b, stats, gelu):
        _, z, _, _, _ = self._xh_g(x, None, w, b, stats, gelu)
        return (F.gelu(z) if gelu else z).to(x.dtype)

    def backward_sums(self, x, dy, w, b, stats, gelu):
        B, C = x.shape[:2]
        xh, _, g, _, _ = self._xh_g(x, dy, w, b, stats, gelu)
        return torch.stack([g.sum(dim=(2, 3)), (g * xh).sum(dim=(2, 3))], dim=-1).reshape(B * C, 2)

    def param_grads(self, sums, B, C):
        per_c = sums.double().view(B, C, 2).sum(dim=0)
        return per_c[:, 1], per_c[:, 0]

    def backward_apply(self, x, dy, w, b, stats, sums, q, D, gelu):
        B, C, H, W = x.shape
        xh, _, g, st, gam = self._xh_g(x, dy, w, b, stats, gelu)
        tot = sums.double().sum(dim=0).view(B, C, 2, 1, 1)
        qd = q.double().view(1, 1, H, 1) / D
        dx = gam * st[:, :, 1] * (g - qd * (tot[:, :, 0] + xh * tot[:, :, 1] - st[:, :, 2] * tot[:, :, 1]))
        return dx.to(x.dtype)

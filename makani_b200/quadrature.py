"""Quadrature rules of the SHT grids -- host-side mirror of `torch_harmonics.quadrature`
(used by the reference at /root/reference/makani/utils/grids.py:67-68,120-129,225).  Returns torch tensors (float64).
"""
import numpy as np
import torch


def _to_t(*arrs):
    return tuple(torch.from_numpy(np.ascontiguousarray(a)) for a in arrs)


def _legendre_gauss_np(n, a=-1.0, b=1.0):
    x, w = np.polynomial.legendre.leggauss(n)
    return (b - a) * 0.5 * x + (b + a) * 0.5, w * (b - a) * 0.5


def _clenshaw_curtiss_np(n, a=-1.0, b=1.0):
    """Clenshaw-Curtis rule on cos(linspace(pi, 0, n)) via the DCT-I closed form of the weights."""
    if n < 2:
        raise ValueError("clenshaw_curtiss_weights needs n >= 2")
    t = np.cos(np.linspace(np.pi, 0.0, n))
    if n == 2:
        w = np.array([1.0, 1.0])
    else:
        n1 = n - 1
        j = np.arange(1, n1 // 2 + 1, dtype=np.float64)
        coef = np.where(2 * j == n1, 1.0, 2.0) / (4.0 * j * j - 1.0)
        k = np.arange(n, dtype=np.float64)
        w = 1.0 - (coef[None, :] * np.cos(2.0 * np.pi * np.outer(k, j) / n1)).sum(axis=1)
        c = np.full(n, 2.0)
        c[0] = c[-1] = 1.0
        w = c * w / n1
    return (b - a) * 0.5 * t + (b + a) * 0.5, w * (b - a) * 0.5


def legendre_gauss_weights(n, a=-1.0, b=1.0):
    return _to_t(*_legendre_gauss_np(n, a, b))


def clenshaw_curtiss_weights(n, a=-1.0, b=1.0):
    return _to_t(*_clenshaw_curtiss_np(n, a, b))


def _grid_np(nlat, grid):
    """cos(colatitude) in row order (row 0 = north, theta ascending) and the matching weights."""
    if grid == "legendre-gauss":
        cost, w = _legendre_gauss_np(nlat)
    elif grid == "equiangular":
        cost, w = _clenshaw_curtiss_np(nlat)
    else:
        raise ValueError(f"Unknown quadrature mode {grid}")
    return np.ascontiguousarray(cost[::-1]), np.ascontiguousarray(w[::-1])


def precompute_latitudes(nlat, grid="equiangular"):
    """Colatitudes (ascending) and quadrature weights, as torch_harmonics.quadrature.precompute_latitudes."""
    cost, w = _grid_np(nlat, grid)
    return _to_t(np.arccos(np.clip(cost, -1.0, 1.0)), w)


def precompute_longitudes(nlon):
    return torch.linspace(0, 2 * np.pi, nlon + 1, dtype=torch.float64)[:-1]


# ------------------------------------------------------------------------------------------- grid quadrature of the norm layers
# makani's GridQuadrature (makani/utils/grids.py:97-191) with normalize=True: weights of the whole sphere summing to 1, constant along longitude,
# so one weight per latitude row.  Built in fp64 (makani builds `naive`, `weatherbench2` and `uniform` in fp32: the two differ in the last bits).
_GRID_TO_RULE = {
    "euclidean": "uniform",
    "equiangular": "naive",
    "legendre-gauss": "legendre-gauss",
    "clenshaw-curtiss": "clenshaw-curtiss",
    "weatherbench2": "weatherbench2",
}


def grid_to_quadrature_rule(grid_type):
    if grid_type not in _GRID_TO_RULE:
        raise NotImplementedError(f"Grid type {grid_type} does not have a quadrature rule")
    return _GRID_TO_RULE[grid_type]


def latitude_quadrature_np(rule, img_shape):
    """fp64 weight of every latitude row of the full H x W grid (each of its W points carries it); the H x W weights sum to 1"""
    H, W = int(img_shape[0]), int(img_shape[1])
    if rule == "naive":
        jac = np.clip(np.sin(np.linspace(0.0, np.pi, H)), 0.0, None)
        q = jac / (W * jac.sum())
    elif rule == "clenshaw-curtiss":
        q = _clenshaw_curtiss_np(H)[1] / (2.0 * W)
    elif rule == "legendre-gauss":
        q = _legendre_gauss_np(H)[1] / (2.0 * W)
    elif rule == "weatherbench2":
        lats = np.linspace(0.0, np.pi, H)
        bounds = np.concatenate([[0.0], 0.5 * (lats[:-1] + lats[1:]), [np.pi]])
        q = (np.cos(bounds[:-1]) - np.cos(bounds[1:])) / (2.0 * W)
    elif rule == "uniform":
        q = np.full(H, 1.0 / (H * W))
    else:
        raise ValueError(f"Unknown quadrature rule {rule}")
    return np.ascontiguousarray(q, dtype=np.float64)


def crop_quadrature_np(grid_type, img_shape, crop_shape=None, crop_offset=(0, 0), h_shapes=None, h_rank=0):
    """the latitude weights of a crop, or of one polar rank's slice of it (`h_shapes`: the split of the crop's rows over the polar group)"""
    crop_shape = tuple(img_shape) if crop_shape is None else tuple(crop_shape)
    q = latitude_quadrature_np(grid_to_quadrature_rule(grid_type), img_shape)
    lo, n = int(crop_offset[0]), int(crop_shape[0])
    if h_shapes is not None:
        lo, n = lo + int(sum(h_shapes[:h_rank])), int(h_shapes[h_rank])
    return np.ascontiguousarray(q[lo:lo + n])

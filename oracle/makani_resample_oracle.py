"""
CPU ORACLE for the bilinear resampling on the sphere  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

torch_harmonics.ResampleS2(mode="bilinear") restated in torch, as the contract written out in include/b200sht.h and DESIGN.md section 4.8,
independently of the product's table builder in makani_b200/resample.py:
  - the tables come from torch.searchsorted / torch.diff on the fp64 colatitudes of oracle.makani_oracle and a torch.linspace longitude grid,
    with the weights rounded to fp32;
  - the forward is the composition torch-harmonics is built from: the pole pseudo-rows concatenated as longitude means, index gathers and
    torch.lerp, evaluated in fp64 whatever the input's dtype (makani's decoder casts its input to fp32 first) and returned in that dtype;
    its backward is torch autograd.
torch-harmonics' source is not available, so this restatement is pinned by identities (tests/test_resample_cpu.py): coincident nodes reproduce
the input, constants are preserved, fields linear in the colatitude are reproduced, pole rows are the longitude means; and makani's own FCN3 /
SNO decoders and the whole FCN3 network run on it (tests/reference_suites/run_reference_fcn3.py).

Only `tests/`, `scripts/resample_bench.py` and `__graft_entry__` import this module; nothing under `makani_b200/` does.
"""
import math

import torch
import torch.nn as nn

from oracle.makani_oracle import precompute_latitudes


def tables(nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out):
    """-> dict of lat_idx, lat_w (fp32), lon_left, lon_right, lon_w (fp32), expand_poles"""
    lats_in = torch.as_tensor(precompute_latitudes(nlat_in, grid_in)[0], dtype=torch.float64)
    lats_out = torch.as_tensor(precompute_latitudes(nlat_out, grid_out)[0], dtype=torch.float64)
    expand = bool((lats_out < lats_in[0]).any() or (lats_out > lats_in[-1]).any())
    if expand:
        lats_in = torch.cat([torch.zeros(1, dtype=torch.float64), lats_in, torch.full((1,), math.pi, dtype=torch.float64)])
    lat_idx = torch.searchsorted(lats_in, lats_out, right=True) - 1
    lat_idx = torch.where(lats_out == lats_in[-1], lat_idx - 1, lat_idx)
    lat_w = ((lats_out - lats_in[lat_idx]) / torch.diff(lats_in)[lat_idx]).to(torch.float32)
    lons_in = torch.linspace(0, 2 * math.pi, nlon_in + 1, dtype=torch.float64)[:-1]
    lons_out = torch.linspace(0, 2 * math.pi, nlon_out + 1, dtype=torch.float64)[:-1]
    left = torch.searchsorted(lons_in, lons_out, right=True) - 1
    right = torch.where(lons_out >= lons_in[-1], torch.zeros_like(left), left + 1)
    diff = lons_in[right] - lons_in[left]
    diff = torch.where(diff < 0, diff + 2 * math.pi, diff)
    lon_w = ((lons_out - lons_in[left]) / diff).to(torch.float32)
    return dict(lat_idx=lat_idx, lat_w=lat_w, lon_left=left, lon_right=right, lon_w=lon_w, expand_poles=expand)


def resample(x, tab):
    """x (..., nlat_in, nlon_in) -> (..., nlat_out, nlon_out) in x's dtype: pole concat, longitude lerp, latitude lerp"""
    if tab["expand_poles"]:
        north = x[..., :1, :].mean(dim=-1, keepdim=True).expand(*x.shape[:-2], 1, x.shape[-1])
        south = x[..., -1:, :].mean(dim=-1, keepdim=True).expand(*x.shape[:-2], 1, x.shape[-1])
        x = torch.cat([north, x, south], dim=-2)
    dev = x.device
    wl = tab["lon_w"].to(device=dev, dtype=x.dtype)
    x = torch.lerp(x[..., tab["lon_left"].to(dev)], x[..., tab["lon_right"].to(dev)], wl)
    idx = tab["lat_idx"].to(dev)
    wt = tab["lat_w"].to(device=dev, dtype=x.dtype)[:, None]
    return torch.lerp(x[..., idx, :], x[..., idx + 1, :], wt)


class ResampleS2(nn.Module):
    """oracle of torch_harmonics.ResampleS2 (mode "bilinear"): same constructor and attributes, tables in non-persistent buffers"""

    def __init__(self, nlat_in, nlon_in, nlat_out, nlon_out, grid_in="equiangular", grid_out="equiangular", mode="bilinear"):
        super().__init__()
        if mode != "bilinear":
            raise NotImplementedError(f"the oracle restates mode 'bilinear' only, not {mode!r}")
        self.nlat_in, self.nlon_in, self.nlat_out, self.nlon_out = nlat_in, nlon_in, nlat_out, nlon_out
        self.grid_in, self.grid_out, self.mode = grid_in, grid_out, mode
        self.tab = tables(nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out)
        self.expand_poles = self.tab["expand_poles"]
        self.skip_resampling = (nlat_in, nlon_in, grid_in) == (nlat_out, nlon_out, grid_out)
        for name in ("lat_idx", "lat_w", "lon_left", "lon_right", "lon_w"):
            self.register_buffer(name, self.tab[name], persistent=False)

    def forward(self, x):
        if self.skip_resampling:
            return x
        return resample(x.to(torch.float64), self.tab).to(x.dtype)

#!/usr/bin/env python
"""Golden vectors for FCN3's decoder with upsample_sht=False, produced by makani's own `DiscreteContinuousDecoder`
(makani/models/networks/fourcastnet3.py, unmodified) on the oracles posed as torch_harmonics: `ResampleS2` from
oracle/makani_resample_oracle.py and `DiscreteContinuousConvS2` from oracle/makani_disco_oracle.py, in the environment of
tests/reference_suites/run_reference_disco.py.  Settings as FCN3 ships them (config/fourcastnet3.yaml): morlet basis, kernel (3, 3), norm "mean",
groups = gcd(channels), no bias, no MLP, at a scaled geometry.  Stored per case (float32): x, the convolution weight, y = decoder(x),
g, dx = d(sum(y g))/dx and dW = d(sum(y g))/dweight, plus the decoder's theta_cutoff.

tests/test_gpu_resample.py composes makani_b200's ResampleS2 and DiscreteContinuousConvS2 with the stored weight and checks y, dx and dW, so the
GPU suite follows makani's decoder without a makani checkout.

    python tests/golden/make_fcn3_decoder_golden.py     # needs a makani checkout -> tests/golden/fcn3_decoder_golden.npz
"""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "reference_suites"))

# (name, model grid (nlat, nlon), grid_in, data grid, grid_out, inp_chans, out_chans): FCN3's 360 x 720 Legendre-Gauss -> 721 x 1440
# equiangular scaled by 1/15, and one equiangular -> equiangular case
CASES = [
    ("lg24x48_eq49x96", (24, 48), "legendre-gauss", (49, 96), "equiangular", 6, 3),
    ("eq25x48_eq49x96", (25, 48), "equiangular", (49, 96), "equiangular", 4, 2),
]


def main():
    import build_reference_sfno as S
    import run_reference_tests as base

    base.install_environment()
    S.stub_physicsnemo()
    from oracle import makani_disco_oracle as DO
    from oracle import makani_resample_oracle as RO

    import makani_b200.disco as mbdisco

    th = sys.modules["torch_harmonics"]
    th.filter_basis = mbdisco
    sys.modules["torch_harmonics.filter_basis"] = mbdisco
    th.DiscreteContinuousConvS2 = DO.DiscreteContinuousConvS2
    th.ResampleS2 = RO.ResampleS2
    import importlib

    M = importlib.import_module("makani.models.networks.fourcastnet3")
    out = {}
    for name, ish, gi, osh, go, cin, cout in CASES:
        torch.manual_seed(23)
        dec = M.DiscreteContinuousDecoder(inp_shape=ish, out_shape=osh, grid_in=gi, grid_out=go, inp_chans=cin, out_chans=cout, kernel_shape=(3, 3),
                                          basis_type="morlet", basis_norm_mode="mean", groups=math.gcd(cin, cout), bias=False, use_mlp=False,
                                          upsample_sht=False)
        assert isinstance(dec.upsample, RO.ResampleS2) and isinstance(dec.conv, DO.DiscreteContinuousConvS2)
        dec = dec.double()
        x = torch.randn(1, cin, *ish, dtype=torch.float64).float().double().requires_grad_(True)
        y = dec(x)
        g = torch.randn_like(y).float().double()
        (y * g).sum().backward()
        rec = dict(x=x.detach(), weight=dec.conv.weight.detach(), y=y.detach(), g=g, dx=x.grad, dW=dec.conv.weight.grad)
        for k, v in rec.items():
            out[f"{name}/{k}"] = v.numpy().astype(np.float32)
        out[f"{name}/theta_cutoff"] = np.float64(M._compute_cutoff_radius(nlat=osh[0], kernel_shape=(3, 3), basis_type="morlet"))
        print(name, {k: tuple(v.shape) for k, v in rec.items()})
    path = os.path.join(HERE, "fcn3_decoder_golden.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Golden vectors for the SFNO network's `normalization_layer="instance_norm_s2"` (makani_b200/sfno.py with makani_b200.norm.GeometricInstanceNormS2),
produced by the REFERENCE's own network class: makani/models/networks/sfnonet.py (SphericalFourierNeuralOperatorNet with makani's own
GeometricInstanceNormS2 and GridQuadrature, unmodified) on the CPU oracle posed as `torch_harmonics`, as tests/golden/make_sfno_golden.py does.
torch.compile is switched off: makani compiles its normalize kernels, and the golden run takes them eagerly.  One case on an equiangular model
grid (`naive` weights, zero-weight pole rows, different input and output grids), one on Legendre-Gauss.  Stored per case: the full state dict,
the input, the output, d(loss)/d(input) and the gradients of the norm parameters and a few others for loss = sum(out * g).

    python tests/golden/make_sfno_s2norm_golden.py     # needs a makani checkout -> tests/golden/sfno_s2norm_golden.npz
"""
import os
import sys

os.environ["TORCHDYNAMO_DISABLE"] = "1"

import numpy as np  # noqa: E402
import torch  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "reference_suites"))

SFNO_S2NORM_GOLDEN_CASES = {
    # equiangular model grid, output grid different from the input grid: the last block's norms run at out_shape
    "s2norm_eq": dict(inp_shape=(33, 64), out_shape=(17, 32), inp_chans=4, out_chans=3, embed_dim=8, num_layers=3, scale_factor=2,
                      model_grid_type="equiangular", sht_grid_type="legendre-gauss", normalization_layer="instance_norm_s2",
                      activation_function="gelu", use_mlp=True, pos_embed="none"),
    # Legendre-Gauss model grid, four blocks (first, two middle, last)
    "s2norm_lg": dict(inp_shape=(32, 64), out_shape=(32, 64), inp_chans=3, out_chans=3, embed_dim=6, num_layers=4, scale_factor=2,
                      model_grid_type="legendre-gauss", sht_grid_type="legendre-gauss", normalization_layer="instance_norm_s2",
                      activation_function="gelu", use_mlp=True, pos_embed="none"),
}
GRAD_KEYS = ["blocks.0.norm0.weight", "blocks.0.norm1.bias", "blocks.1.norm0.bias", "blocks.2.norm1.weight", "blocks.0.filter.filter.weight",
             "encoder.fwd.0.weight"]


def main():
    import run_reference_tests as R
    from build_reference_sfno import stub_physicsnemo

    R.install_environment()
    stub_physicsnemo()
    from makani.models.common.layer_norm import GeometricInstanceNormS2
    from makani.models.networks import sfnonet

    out = {}
    for name, cfg in SFNO_S2NORM_GOLDEN_CASES.items():
        torch.manual_seed(333)
        net = sfnonet.SphericalFourierNeuralOperatorNet(**cfg)
        assert all(isinstance(b.norm0, GeometricInstanceNormS2) and isinstance(b.norm1, GeometricInstanceNormS2) for b in net.blocks)
        with torch.no_grad():   # non-trivial values where the reference initialises with zeros / ones
            for k, p in net.named_parameters():
                if k.endswith(".bias") or "norm" in k:
                    p.add_(0.1 * torch.randn_like(p))
        x = torch.randn(2, cfg["inp_chans"], *cfg["inp_shape"], requires_grad=True)
        y = net(x)
        g = torch.randn_like(y)
        (y * g).sum().backward()
        for k, v in net.state_dict().items():
            v = v.detach()
            out[f"{name}/sd/{k}"] = torch.view_as_real(v).numpy() if v.is_complex() else v.numpy()
        out[f"{name}/x"], out[f"{name}/y"], out[f"{name}/g"], out[f"{name}/dx"] = x.detach().numpy(), y.detach().numpy(), g.numpy(), x.grad.numpy()
        params = dict(net.named_parameters())
        for k in GRAD_KEYS:
            gr = params[k].grad
            out[f"{name}/grad/{k}"] = torch.view_as_real(gr).numpy() if gr.is_complex() else gr.numpy()
        print(name, "params", sum(p.numel() for p in net.parameters()), "y", tuple(y.shape), "|y|", float(y.abs().mean()))
    path = os.path.join(HERE, "sfno_s2norm_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

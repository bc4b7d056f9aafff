#!/usr/bin/env python
"""Golden vectors for the FourCastNet 3 network restatement (makani_b200/fcn3.py), produced by the REFERENCE's own network class:
makani/models/networks/fourcastnet3.py (AtmoSphericNeuralOperatorNet, unmodified) with makani's own SpectralConv / MLP / EncoderDecoder /
LayerScale, on the CPU oracles posed as torch_harmonics (RealSHT / InverseRealSHT from oracle/makani_oracle.py, DiscreteContinuousConvS2 from
oracle/makani_disco_oracle.py, ResampleS2 from oracle/makani_resample_oracle.py), in the environment of make_sfno_golden.py and
make_fcn3_decoder_golden.py.  All cases at a scaled geometry, small enough to keep the file small: 17 x 32 equiangular data grid -> 8 x 16
Legendre-Gauss model grid (scale factor 2).

Stored per case, float32: the full state dict (complex weights as view_as_real), x, y = net(x), g, dx = d(sum(y g))/dx and the gradients of
GRAD_KEYS[case]; and `tags`, a JSON string of every parameter's is_shared_mp / sharded_dims_mp.

    python tests/golden/make_fcn3_golden.py        # needs a makani checkout -> tests/golden/fcn3_golden.npz
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "reference_suites"))

GEOMETRY = dict(model_grid_type="equiangular", sht_grid_type="legendre-gauss", inp_shape=(17, 32), out_shape=(17, 32), scale_factor=2,
                kernel_shape=[3, 3], filter_basis_type="morlet", filter_basis_norm_mode="mean")
# config/fourcastnet3.yaml's channel structure, scaled down: variables x pressure levels in variable-major order, then surface variables with tcwv
LEVELS = (500, 850)
SHIPPED_CHANNELS = ["u10m", "v10m", "t2m", "msl", "tcwv"] + [f"{v}{p}" for v in "uvztq" for p in LEVELS]
SHIPPED_AUX = ["xzen", "xnoise0", "xoro", "xlsml", "xlsms"]                  # makani's get_auxiliary_channels order: zenith, noise, orography, masks

FCN3_GOLDEN_CASES = {
    # the shipped architecture settings (morlet (3, 3) "mean", serial MLP of ratio 2, gelu, layer scale, no bias / norm / big skip, water clamp)
    # with sfno_block_frequency 2 over 4 layers: blocks 0 and 2 global, 1 and 3 local
    "shipped": dict(GEOMETRY, channel_names=SHIPPED_CHANNELS, aux_channel_names=SHIPPED_AUX, atmo_embed_dim=4, surf_embed_dim=5, aux_embed_dim=3,
                    num_layers=4, num_groups=1, sfno_block_frequency=2, encoder_mlp=False, use_mlp=True, mlp_mode="serial", mlp_ratio=2,
                    activation_function="gelu", layer_scale=True, normalization_layer="none", hard_thresholding_fraction=1.0, pos_embed=False,
                    big_skip=False, bias=False, clamp_water=True),
    # everything the shipped config turns off: bias, encoder / decoder MLPs, big skip, layer norm, SHT upsampling, silu, no layer scale, fewer modes
    "variant": dict(GEOMETRY, channel_names=["sp", "tcwv", "u10m", "u300", "v300", "q300", "u700", "v700", "q700"], aux_channel_names=["xzen", "xoro"],
                    atmo_embed_dim=4, surf_embed_dim=5, aux_embed_dim=3, num_layers=3, sfno_block_frequency=2, encoder_mlp=True, upsample_sht=True,
                    use_mlp=True, mlp_ratio=1.5, activation_function="silu", layer_scale=False, normalization_layer="layer_norm", max_modes=(6, 7),
                    big_skip=True, bias=True, clamp_water=True),
    # pressure-level variables only and no auxiliary channels: no surface encoder / decoder, no aux encoder (surf_embed_dim 0, as the reference needs
    # then); instance norm, global every 3rd block
    "no_surf_no_aux": dict(GEOMETRY, channel_names=[f"{v}{p}" for v in "zt" for p in (500, 850)], atmo_embed_dim=4, surf_embed_dim=0, num_layers=3,
                           sfno_block_frequency=3, use_mlp=True, mlp_ratio=2, activation_function="gelu", layer_scale=True,
                           normalization_layer="instance_norm", hard_thresholding_fraction=0.75, big_skip=False, bias=False),
}
# both encoders, a global block, a local block, an MLP, the layer scale and both decoders, where the case has them
GRAD_KEYS = {
    "shipped": ["atmo_encoder.conv.weight", "surf_encoder.conv.weight", "aux_encoder.conv.weight", "blocks.0.global_conv.weight",
                "blocks.1.local_conv.weight", "blocks.1.mlp.fwd.0.weight", "blocks.2.mlp.fwd.3.weight", "blocks.3.layer_scale.weight",
                "atmo_decoder.conv.weight", "surf_decoder.conv.weight"],
    "variant": ["atmo_encoder.conv.bias", "atmo_encoder.mlp.fwd.0.weight", "surf_encoder.conv.weight", "aux_encoder.conv.weight",
                "blocks.0.global_conv.weight", "blocks.0.global_conv.bias", "blocks.1.local_conv.weight", "blocks.1.norm1.norm.weight",
                "blocks.2.mlp.fwd.0.bias", "atmo_decoder.mlp.fwd.2.weight", "atmo_decoder.conv.weight", "surf_decoder.conv.weight",
                "residual_transform.weight"],
    "no_surf_no_aux": ["atmo_encoder.conv.weight", "blocks.0.global_conv.weight", "blocks.1.local_conv.weight", "blocks.1.norm2.weight",
                       "blocks.2.mlp.fwd.0.weight", "blocks.2.layer_scale.weight", "atmo_decoder.conv.weight"],
}


def n_inputs(cfg):
    return len(cfg["channel_names"]) + len(cfg.get("aux_channel_names", []))


def tags(net):
    return json.dumps({k: [getattr(p, "is_shared_mp", None), getattr(p, "sharded_dims_mp", None)] for k, p in net.named_parameters()}, sort_keys=True)


def reference_module():
    """makani's fourcastnet3 module on the oracles posed as torch_harmonics"""
    import importlib

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
    return importlib.import_module("makani.models.networks.fourcastnet3")


def main():
    M = reference_module()
    out = {}
    for name, cfg in FCN3_GOLDEN_CASES.items():
        torch.manual_seed(333)
        net = M.AtmoSphericNeuralOperatorNet(**cfg)
        with torch.no_grad():   # non-trivial values where the reference initialises with zeros / ones / constants
            for k, p in net.named_parameters():
                if k.endswith(".bias") or "norm" in k or "layer_scale" in k:
                    p.add_(0.1 * torch.randn_like(p))
        x = torch.randn(1, n_inputs(cfg), *cfg["inp_shape"], requires_grad=True)
        y = net(x)
        g = torch.randn_like(y)
        (y * g).sum().backward()
        for k, v in net.state_dict().items():
            v = v.detach()
            out[f"{name}/sd/{k}"] = torch.view_as_real(v).numpy() if v.is_complex() else v.numpy()
        out[f"{name}/x"], out[f"{name}/y"], out[f"{name}/g"], out[f"{name}/dx"] = x.detach().numpy(), y.detach().numpy(), g.numpy(), x.grad.numpy()
        params = dict(net.named_parameters())
        for k in GRAD_KEYS[name]:
            gr = params[k].grad
            out[f"{name}/grad/{k}"] = torch.view_as_real(gr).numpy() if gr.is_complex() else gr.numpy()
        out[f"{name}/tags"] = np.array(tags(net))
        print(name, "params", sum(p.numel() for p in net.parameters()), "x", tuple(x.shape), "y", tuple(y.shape), "|y|", float(y.detach().abs().mean()))
    path = os.path.join(HERE, "fcn3_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

"""FourCastNet 3 network on the CUDA kernels of this package: makani's AtmoSphericNeuralOperatorNet without a makani checkout.

Restates, with the same constructor arguments, module tree, parameter names, shapes, initialisation scales and model-parallel tags, the reference's
  DiscreteContinuousEncoder / Decoder    makani/models/networks/fourcastnet3.py:117-418   (DISCO convolution; bilinear or SHT upsampling in fp32)
  NeuralOperatorBlock                    makani/models/networks/fourcastnet3.py:421-638   (norm1 -> local DISCO or global dhconv -> norm2 -> MLP -> layer scale + skip)
  AtmoSphericNeuralOperatorNet           makani/models/networks/fourcastnet3.py:641-1135  (channel groups, encoders, processor, decoders, big skip, water clamp)
  _compute_cutoff_radius, _soft_clamp, _get_norm_layer_handle    fourcastnet3.py:47-114
  get_channel_groups, get_water_channels makani/utils/features.py:69-140
  LayerScale                             makani/models/common/layers.py:154-197
so that a checkpoint of the reference network loads with `load_state_dict(strict=True)` and gives the same outputs (tests/golden/fcn3_golden.npz is
produced by the REFERENCE class, tests/golden/make_fcn3_golden.py).

Under h x w spatial model parallelism (the process grid of makani_b200.distributed.init(polar_group, azimuth_group) has more than one rank, read
where makani reads comm.get_size("spatial")), the network builds what makani builds there (fourcastnet3.py:63-114, 190, 340-366, 519, 927-936):
DistributedDiscreteContinuousConvS2 in the encoders, local blocks and decoders, DistributedResampleS2 (or the DistributedRealSHT /
DistributedInverseRealSHT pair with `upsample_sht`), the distributed SHT pair for the processor, DistributedInstanceNorm2d /
DistributedGeometricInstanceNormS2, and it tags the convolution weights and biases is_shared_mp = ["spatial"].  Module tree, parameter names and
state-dict keys stay those of the serial network; inputs and outputs are this rank's (lat, lon) shard of the data grid (`compute_split_shapes`).
Every other operation (MLPs, layer scale, skips, big skip, water clamp, the scatter of `decode`) acts on local pixels.  Loading a global
checkpoint, keeping the shared parameters in step and reducing their gradients: makani_b200.distributed.scatter_state_dict, gather_state_dict,
sync_shared_params and reduce_shared_gradients.  makani's `matmul` feature parallelism (DistributedMLP) is not built.

On the CUDA backend every FLOP-heavy operation runs on this library's sm_90a kernels or a cuBLAS GEMM: the DISCO convolutions (csrc/disco.cu), the
bilinear resampling (csrc/resample.cu), the SHT pair and the dhconv SpectralConv (tensor-core engine), the 1x1 convolutions as GEMMs on the NCHW tensor
with the bias + GELU kernel of csrc/norm.cu (sfno.Conv1x1 / MLP / EncoderDecoder), the norms on csrc/norm.cu.  LayerScale, which makani computes as a
grouped conv2d with one group per channel, is the per-channel multiply it equals.

`backend` lets the same network be built on other transform / convolution / norm classes (the CPU tests pass the oracle's).
"""
import math
import re
from collections import OrderedDict
from functools import partial

import torch
import torch.nn as nn
from torch import amp
from torch.utils.checkpoint import checkpoint

from .sfno import _ACTS, MLP, Conv1x1, DropPath, EncoderDecoder
from .sfno import _Backend as _SpectralBackend


class _Backend(_SpectralBackend):
    """default classes: the CUDA path of this package (SHT pair and SpectralConv at `precision`, DISCO, resampling, norms)"""

    def __init__(self, precision="auto"):
        super().__init__(precision)
        import makani_b200 as mb
        from . import norm

        self.DiscreteContinuousConvS2 = mb.DiscreteContinuousConvS2
        self.ResampleS2 = mb.ResampleS2
        self.InstanceNorm2d = norm.InstanceNorm2d
        self.LayerNorm = norm.DistributedLayerNorm
        self.GeometricInstanceNormS2 = norm.GeometricInstanceNormS2


class _DistributedBackend(_Backend):
    """the classes makani builds at spatial model parallelism > 1, on the process grid of makani_b200.distributed"""

    def __init__(self, precision="auto"):
        super().__init__(precision)
        from . import distributed as mbd

        self.RealSHT = partial(mbd.DistributedRealSHT, precision=precision)
        self.InverseRealSHT = partial(mbd.DistributedInverseRealSHT, precision=precision)
        self.DiscreteContinuousConvS2 = mbd.DistributedDiscreteContinuousConvS2
        self.ResampleS2 = mbd.DistributedResampleS2
        self.InstanceNorm2d = mbd.DistributedInstanceNorm2d
        self.GeometricInstanceNormS2 = mbd.DistributedGeometricInstanceNormS2


def _spatial_size():
    """makani's comm.get_size("spatial"): the ranks of the h x w grid set by makani_b200.distributed.init (1 without one)"""
    from . import distributed as mbd

    return mbd.polar_group_size() * mbd.azimuth_group_size()


def _default_backend(precision="auto"):
    return _DistributedBackend(precision) if _spatial_size() > 1 else _Backend(precision)


def _tag_spatial_conv(conv):
    """makani's tags of a DISCO convolution under spatial model parallelism: weight and bias replicated on every spatial rank"""
    if _spatial_size() > 1:
        conv.weight.is_shared_mp = ["spatial"]
        conv.weight.sharded_dims_mp = [None, None, None]
        if conv.bias is not None:
            conv.bias.is_shared_mp = ["spatial"]
            conv.bias.sharded_dims_mp = [None]


def _refuse_oversplit(lat_sizes, lon_sizes):
    """each latitude-like size split over the polar group and each longitude-like size over the azimuth group must leave every rank at least
    one point; a module would otherwise fail deep inside its forward"""
    from . import distributed as mbd

    for sizes, n_ranks, what in ((lat_sizes, mbd.polar_group_size(), "polar (h)"), (lon_sizes, mbd.azimuth_group_size(), "azimuth (w)")):
        for name, n in sizes.items():
            if n_ranks > 1 and min(mbd.compute_split_shapes(n, n_ranks)) < 1:
                raise ValueError(f"{name} = {n} cannot be split over the {n_ranks} ranks of the {what} group: every rank needs at least one point")


def _compute_cutoff_radius(nlat, kernel_shape, basis_type):
    """heuristic DISCO cutoff: (kernel_shape[0] + 1) * factor * pi / (nlat - 1)"""
    theta_cutoff_factor = {"piecewise linear": 0.5, "morlet": 0.5, "harmonic": 0.5, "zernike": math.sqrt(2.0)}
    return (kernel_shape[0] + 1) * theta_cutoff_factor[basis_type] * math.pi / float(nlat - 1)


def _soft_clamp(x, offset=0.0):
    """0 below 0, x^2 on [0, 0.5), x - 1/4 from 0.5 on: positive and continuously differentiable"""
    x = x + offset
    y = torch.where(x > 0.0, x**2, 0.0)
    y = torch.where(x >= 0.5, x - 0.25, y)
    return y


def get_water_channels(channel_names):
    """indices of specific / relative humidity channels (q*, r*) and of tcwv"""
    return [c for c, ch in enumerate(channel_names) if ch[0] in {"q", "r"} or ch == "tcwv"]


def get_channel_groups(channel_names, aux_channel_names=()):
    """-> (atmo_chans, surf_chans, dyn_aux_chans, stat_aux_chans, pressure levels): a name ending in 1-4 digits after 1-3 lower-case letters (other
    than d2) is an atmospheric variable on that pressure level, grouped level by level in order of first appearance; everything else is a surface
    variable.  Auxiliary channels are numbered after the channel names; orography and the land-sea masks are static."""
    atmo_groups = OrderedDict()
    surf_chans, dyn_aux_chans, stat_aux_chans = [], [], []
    for idx, chn in enumerate(channel_names):
        if (re.search("[a-z]{1,3}[0-9]{1,4}$", chn) is not None) and (chn != "d2"):
            atmo_groups.setdefault(int(re.search("[0-9]{1,4}$", chn).group()), []).append(idx)
        else:
            surf_chans.append(idx)
    atmo_chans, n_atmo_chans = [], None
    for idx in atmo_groups.values():
        if n_atmo_chans is None:
            n_atmo_chans = len(idx)
        elif n_atmo_chans != len(idx):
            raise ValueError(f"expected all atmospheric pressure level groups to have the same number of channels ({n_atmo_chans}), but got {len(idx)}")
        atmo_chans += idx
    for idx, chn in enumerate(aux_channel_names):
        (stat_aux_chans if chn in ["xoro", "xlsml", "xlsms"] else dyn_aux_chans).append(idx + len(channel_names))
    return atmo_chans, surf_chans, dyn_aux_chans, stat_aux_chans, atmo_groups.keys()


class LayerScale(nn.Module):
    """learned per-channel scale of a residual branch, weight (C, 1, 1, 1) initialised to `init_value`.  makani applies it as a grouped conv2d with
    one group per channel; here it is the multiply that equals, in the dtype the convolution would return (the autocast dtype under autocast)."""

    def __init__(self, num_chans=3, init_value=0.1):
        super().__init__()
        self.num_chans = num_chans
        self.weight = nn.Parameter(torch.randn(self.num_chans, 1, 1, 1))     # drawn, then overwritten, as the reference: same RNG stream
        torch.nn.init.constant_(self.weight, val=init_value)

    def forward(self, x):
        dtype = torch.get_autocast_dtype(x.device.type) if torch.is_autocast_enabled(x.device.type) else x.dtype
        return x.to(dtype) * self.weight.to(dtype).view(1, -1, 1, 1)


def _get_norm_layer_handle(h, w, embed_dim, normalization_layer="none", sht_grid_type="legendre-gauss", backend=None):
    """the norm constructor of fourcastnet3.py:63-114 on the backend's classes.  "instance_norm_s2": makani's handle also passes `pole_mask=0`, which
    its GeometricInstanceNormS2 does not take (so makani's class cannot be built with this setting); pole_mask 0 masks nothing and is not passed."""
    backend = backend or _default_backend()
    if normalization_layer == "layer_norm":
        return partial(backend.LayerNorm, normalized_shape=(embed_dim), elementwise_affine=True, eps=1e-6)
    if normalization_layer == "instance_norm":
        if _spatial_size() > 1:         # makani's DistributedInstanceNorm2d keeps no running statistics to switch off
            return partial(backend.InstanceNorm2d, num_features=embed_dim, eps=1e-6, affine=True)
        return partial(backend.InstanceNorm2d, num_features=embed_dim, eps=1e-6, affine=True, track_running_stats=False)
    if normalization_layer == "instance_norm_s2":
        return partial(backend.GeometricInstanceNormS2, img_shape=(h, w), crop_shape=(h, w), crop_offset=(0, 0), grid_type=sht_grid_type,
                       num_features=embed_dim, eps=1e-6, affine=True)
    if normalization_layer == "none":
        return nn.Identity
    raise NotImplementedError(f"Error, normalization {normalization_layer} not implemented.")


class DiscreteContinuousEncoder(nn.Module):
    """DISCO convolution from the data grid onto the model grid (+ activation and a 1x1 MLP with `use_mlp`, the convolution weight scaled by sqrt 2)"""

    def __init__(self, inp_shape=(721, 1440), out_shape=(480, 960), grid_in="equiangular", grid_out="equiangular", inp_chans=2, out_chans=2,
                 kernel_shape=(3, 3), basis_type="harmonic", basis_norm_mode="mean", use_mlp=False, mlp_ratio=2.0, activation_function=nn.GELU, groups=1,
                 bias=False, backend=None):
        super().__init__()
        backend = backend or _default_backend()
        theta_cutoff = _compute_cutoff_radius(nlat=inp_shape[0], kernel_shape=kernel_shape, basis_type=basis_type)
        self.conv = backend.DiscreteContinuousConvS2(inp_chans, out_chans, in_shape=inp_shape, out_shape=out_shape, kernel_shape=kernel_shape,
                                                     basis_type=basis_type, basis_norm_mode=basis_norm_mode, grid_in=grid_in, grid_out=grid_out,
                                                     groups=groups, bias=bias, theta_cutoff=theta_cutoff)
        _tag_spatial_conv(self.conv)
        if use_mlp:
            with torch.no_grad():
                self.conv.weight *= math.sqrt(2.0)
            self.act = activation_function()
            self.mlp = EncoderDecoder(num_layers=1, input_dim=out_chans, output_dim=out_chans, hidden_dim=int(mlp_ratio * out_chans),
                                      act_layer=activation_function, input_format="nchw")

    def forward(self, x):
        x = self.conv(x)
        if hasattr(self, "act"):
            x = self.act(x)
        if hasattr(self, "mlp"):
            x = self.mlp(x)
        return x


class DiscreteContinuousDecoder(nn.Module):
    """[activation, 1x1 MLP] -> upsampling to the data grid (bilinear ResampleS2, or SHT -> inverse SHT with `upsample_sht`) -> DISCO convolution on
    the data grid; upsampling and convolution in fp32 with autocast off, the output cast back to the input's dtype"""

    def __init__(self, inp_shape=(480, 960), out_shape=(721, 1440), grid_in="equiangular", grid_out="equiangular", inp_chans=2, out_chans=2,
                 kernel_shape=(3, 3), basis_type="harmonic", basis_norm_mode="mean", use_mlp=False, mlp_ratio=2.0, activation_function=nn.GELU, groups=1,
                 bias=False, upsample_sht=False, backend=None):
        super().__init__()
        backend = backend or _default_backend()
        if use_mlp:
            self.mlp = EncoderDecoder(num_layers=1, input_dim=inp_chans, output_dim=inp_chans, hidden_dim=int(mlp_ratio * inp_chans),
                                      act_layer=activation_function, input_format="nchw", gain=2.0)
            self.act = activation_function()
        if upsample_sht:
            self.sht = backend.RealSHT(*inp_shape, grid=grid_in).float()
            self.isht = backend.InverseRealSHT(*out_shape, lmax=self.sht.lmax, mmax=self.sht.mmax, grid=grid_out).float()
            self.upsample = nn.Sequential(self.sht, self.isht)
        else:
            self.upsample = backend.ResampleS2(*inp_shape, *out_shape, grid_in=grid_in, grid_out=grid_out, mode="bilinear")
        theta_cutoff = _compute_cutoff_radius(nlat=out_shape[0], kernel_shape=kernel_shape, basis_type=basis_type)
        self.conv = backend.DiscreteContinuousConvS2(inp_chans, out_chans, in_shape=out_shape, out_shape=out_shape, kernel_shape=kernel_shape,
                                                     basis_type=basis_type, basis_norm_mode=basis_norm_mode, grid_in=grid_out, grid_out=grid_out,
                                                     groups=groups, bias=False, theta_cutoff=theta_cutoff)
        _tag_spatial_conv(self.conv)

    def forward(self, x):
        dtype = x.dtype
        if hasattr(self, "act"):        # the reference applies the activation before the MLP here (fourcastnet3.py:406-410)
            x = self.act(x)
        if hasattr(self, "mlp"):
            x = self.mlp(x)
        with amp.autocast(device_type=x.device.type, enabled=False):
            x = self.conv(self.upsample(x.to(torch.float32)))
        return x.to(dtype=dtype)


class NeuralOperatorBlock(nn.Module):
    """norm1 -> local DISCO convolution or global dhconv SpectralConv -> norm2 -> [MLP] -> drop path -> skip(x[:, :out_chans]) + layer_scale(dx)"""

    def __init__(self, forward_transform, inverse_transform, inp_chans, out_chans, conv_type="local", mlp_ratio=2.0, mlp_drop_rate=0.0,
                 path_drop_rate=0.0, act_layer=nn.GELU, normalization_layer="none", num_groups=1, skip="identity", layer_scale=True, use_mlp=False,
                 kernel_shape=(3, 3), basis_type="harmonic", basis_norm_mode="mean", checkpointing_level=0, bias=False, backend=None):
        super().__init__()
        backend = backend or _default_backend()
        self.inp_shape = (forward_transform.nlat, forward_transform.nlon)
        self.out_shape = (inverse_transform.nlat, inverse_transform.nlon)
        self.out_chans = out_chans
        if conv_type == "local":
            theta_cutoff = 2 * _compute_cutoff_radius(nlat=self.inp_shape[0], kernel_shape=kernel_shape, basis_type=basis_type)
            self.local_conv = backend.DiscreteContinuousConvS2(inp_chans, inp_chans, in_shape=self.inp_shape, out_shape=self.out_shape,
                                                               kernel_shape=kernel_shape, basis_type=basis_type, basis_norm_mode=basis_norm_mode,
                                                               groups=num_groups, grid_in=forward_transform.grid, grid_out=inverse_transform.grid,
                                                               bias=False, theta_cutoff=theta_cutoff)
            _tag_spatial_conv(self.local_conv)
        elif conv_type == "global":
            self.global_conv = backend.SpectralConv(forward_transform, inverse_transform, inp_chans, inp_chans, operator_type="dhconv",
                                                    num_groups=num_groups, bias=bias, gain=1.0)
        else:
            raise ValueError(f"Unknown convolution type {conv_type}")
        norm_layer_handle = _get_norm_layer_handle(self.inp_shape[0], self.inp_shape[1], inp_chans, normalization_layer=normalization_layer,
                                                   sht_grid_type=forward_transform.grid, backend=backend)
        self.norm1 = norm_layer_handle()
        self.norm2 = norm_layer_handle()
        self.checkpoint_mlp = checkpointing_level >= 2     # makani's MLP(checkpointing=...) recomputes fc1 -> act -> fc2 in the backward
        if use_mlp:
            self.mlp = MLP(in_features=inp_chans, out_features=out_chans, hidden_features=int(inp_chans * mlp_ratio), act_layer=act_layer,
                           drop_rate=mlp_drop_rate, drop_type="features", gain=1.0)
        self.drop_path = DropPath(path_drop_rate) if path_drop_rate > 0.0 else nn.Identity()
        if layer_scale:
            self.layer_scale = LayerScale(out_chans)
            self.layer_scale.weight.is_shared_mp = ["spatial"]
            self.layer_scale.weight.sharded_dims_mp = [None, None, None, None]
        else:
            self.layer_scale = nn.Identity()
        if skip == "linear":
            self.skip = Conv1x1(inp_chans, out_chans, 1, 1, bias=False)
            torch.nn.init.normal_(self.skip.weight, std=math.sqrt(1.0 / inp_chans))
            self.skip.weight.is_shared_mp = ["spatial"]
            self.skip.weight.sharded_dims_mp = [None, None, None, None]
        elif skip == "identity":
            self.skip = nn.Identity()
        elif skip != "none":
            raise ValueError(f"Unknown skip connection type {skip}")

    def forward(self, x):
        x = self.norm1(x)
        if hasattr(self, "global_conv"):
            dx, _ = self.global_conv(x)
        else:
            dx = self.local_conv(x)
        dx = self.norm2(dx)
        if hasattr(self, "mlp"):
            dx = checkpoint(self.mlp, dx, use_reentrant=False) if self.checkpoint_mlp else self.mlp(dx)
        dx = self.drop_path(dx)
        if hasattr(self, "skip"):
            return self.skip(x[..., : self.out_chans, :, :]) + self.layer_scale(dx)
        return dx


class AtmoSphericNeuralOperatorNet(nn.Module):
    """FourCastNet 3: atmospheric channels encoded level by level with one shared DISCO encoder, surface and auxiliary channels with their own; a
    processor of NeuralOperatorBlocks on the (h, w) = inp_shape // scale_factor Legendre-Gauss grid, global (dhconv) every `sfno_block_frequency`
    blocks and local (DISCO) otherwise, the embedded auxiliary channels appended to every block's input; decoders back to the data grid, an optional
    linear big skip and a soft clamp of the water channels.  Constructor as makani's (config keys it does not use, such as pos_embed or mlp_mode, are
    accepted and ignored), plus `precision` for the CUDA SHT / SpectralConv and `backend`."""

    def __init__(self, model_grid_type="equiangular", sht_grid_type="legendre-gauss", inp_shape=(721, 1440), out_shape=(721, 1440), kernel_shape=(3, 3),
                 filter_basis_type="harmonic", filter_basis_norm_mode="mean", scale_factor=8, encoder_mlp=False, upsample_sht=False,
                 channel_names=("u500", "v500"), aux_channel_names=(), n_history=0, atmo_embed_dim=8, surf_embed_dim=8, aux_embed_dim=8, num_layers=4,
                 num_groups=1, use_mlp=True, mlp_ratio=2.0, activation_function="gelu", layer_scale=True, pos_drop_rate=0.0, path_drop_rate=0.0,
                 mlp_drop_rate=0.0, normalization_layer="none", max_modes=None, hard_thresholding_fraction=1.0, sfno_block_frequency=2, big_skip=False,
                 clamp_water=False, bias=False, checkpointing_level=0, freeze_encoder=False, freeze_processor=False, precision="auto", backend=None,
                 **kwargs):
        super().__init__()
        backend = backend or _default_backend(precision)
        self.inp_shape, self.out_shape = inp_shape, out_shape
        self.atmo_embed_dim, self.surf_embed_dim, self.aux_embed_dim = atmo_embed_dim, surf_embed_dim, aux_embed_dim
        self.big_skip, self.checkpointing_level = big_skip, checkpointing_level
        if n_history != 0:
            raise ValueError(f"this model currently does not support history, expected n_history == 0 but got {n_history}")
        self.h, self.w = int(self.inp_shape[0] // scale_factor), int(self.inp_shape[1] // scale_factor)
        if _spatial_size() > 1:
            modes_lat, modes_lon = self._modes(hard_thresholding_fraction, max_modes)
            _refuse_oversplit({"inp_shape[0]": inp_shape[0], "out_shape[0]": out_shape[0], "model grid h": self.h, "modes_lat": modes_lat},
                              {"inp_shape[1]": inp_shape[1], "out_shape[1]": out_shape[1], "model grid w": self.w, "modes_lon": modes_lon,
                               "decoder SHT modes w // 2 + 1": self.w // 2 + 1})
        self._init_spectral_transforms(backend, sht_grid_type, hard_thresholding_fraction, max_modes)
        self._precompute_channel_groups(channel_names, aux_channel_names)
        self.n_out_chans = self.n_atmo_groups * self.n_atmo_chans + self.n_surf_chans
        self.total_embed_dim = self.n_atmo_groups * self.atmo_embed_dim + self.surf_embed_dim
        kernel_shape = tuple(kernel_shape)
        if activation_function not in _ACTS:
            raise ValueError(f"Unknown activation function {activation_function}")
        act = _ACTS[activation_function]

        common = dict(kernel_shape=kernel_shape, basis_type=filter_basis_type, basis_norm_mode=filter_basis_norm_mode, activation_function=act, bias=bias,
                      use_mlp=encoder_mlp, backend=backend)
        enc = partial(DiscreteContinuousEncoder, inp_shape=inp_shape, out_shape=(self.h, self.w), grid_in=model_grid_type, grid_out=sht_grid_type, **common)
        dec = partial(DiscreteContinuousDecoder, inp_shape=(self.h, self.w), out_shape=out_shape, grid_in=sht_grid_type, grid_out=model_grid_type,
                      upsample_sht=upsample_sht, **common)
        # construction order as the reference's (the parameters draw the same random numbers from the same seed)
        self.atmo_encoder = enc(inp_chans=self.n_atmo_chans, out_chans=self.atmo_embed_dim, groups=math.gcd(self.n_atmo_chans, self.atmo_embed_dim))
        if self.n_surf_chans > 0:
            self.surf_encoder = enc(inp_chans=self.n_surf_chans, out_chans=self.surf_embed_dim, groups=math.gcd(self.n_surf_chans, self.surf_embed_dim))
        self.atmo_decoder = dec(inp_chans=self.atmo_embed_dim, out_chans=self.n_atmo_chans, groups=math.gcd(self.n_atmo_chans, self.atmo_embed_dim))
        if self.n_surf_chans > 0:
            self.surf_decoder = dec(inp_chans=self.surf_embed_dim, out_chans=self.n_surf_chans, groups=math.gcd(self.n_surf_chans, self.surf_embed_dim))
        if self.n_aux_chans > 0:
            self.aux_encoder = enc(inp_chans=self.n_aux_chans, out_chans=self.aux_embed_dim, groups=math.gcd(self.n_aux_chans, self.aux_embed_dim))

        self.pos_drop = nn.Dropout(p=pos_drop_rate) if pos_drop_rate > 0.0 else nn.Identity()
        dpr = [v.item() for v in torch.linspace(0, path_drop_rate, num_layers)]
        self.blocks = nn.ModuleList()
        for i in range(num_layers):
            self.blocks.append(NeuralOperatorBlock(self.sht, self.isht, self.total_embed_dim + (self.n_aux_chans > 0) * self.aux_embed_dim, self.total_embed_dim,
                                                   conv_type="global" if i % sfno_block_frequency == 0 else "local", mlp_ratio=mlp_ratio,
                                                   mlp_drop_rate=mlp_drop_rate, path_drop_rate=dpr[i], act_layer=act, normalization_layer=normalization_layer,
                                                   skip="identity", layer_scale=layer_scale, use_mlp=use_mlp, kernel_shape=kernel_shape,
                                                   basis_type=filter_basis_type, basis_norm_mode=filter_basis_norm_mode, bias=bias,
                                                   checkpointing_level=checkpointing_level, backend=backend))

        if self.big_skip:
            self.residual_transform = Conv1x1(self.n_out_chans, self.n_out_chans, 1, bias=False)
            self.residual_transform.weight.is_shared_mp = ["spatial"]
            self.residual_transform.weight.sharded_dims_mp = [None, None, None, None]
            nn.init.normal_(self.residual_transform.weight, mean=0.0, std=math.sqrt(0.5 / self.n_out_chans))

        if clamp_water:
            water_chans = get_water_channels(channel_names)
            if len(water_chans) > 0:
                self.register_buffer("water_channels", torch.tensor(water_chans, dtype=torch.long), persistent=False)
                mask = torch.zeros(self.n_out_chans, dtype=torch.bool)
                mask[water_chans] = True
                self.register_buffer("water_channel_mask", mask.view(1, -1, 1, 1), persistent=False)

        if freeze_encoder:
            frozen = list(self.atmo_encoder.parameters()) + list(self.atmo_decoder.parameters())
            if hasattr(self, "surf_encoder"):
                frozen += list(self.surf_encoder.parameters()) + list(self.surf_decoder.parameters())
            if hasattr(self, "aux_encoder"):
                frozen += list(self.aux_encoder.parameters())
            if self.big_skip:
                frozen += list(self.residual_transform.parameters())
            for p in frozen:
                p.requires_grad = False
        if freeze_processor:
            for p in self.blocks.parameters():
                p.requires_grad = False

    def _init_spectral_transforms(self, backend, sht_grid_type, hard_thresholding_fraction, max_modes):
        """the processor's SHT pair on the (h, w) grid"""
        modes_lat, modes_lon = self._modes(hard_thresholding_fraction, max_modes)
        self.sht = backend.RealSHT(self.h, self.w, lmax=modes_lat, mmax=modes_lon, grid=sht_grid_type).float()
        self.isht = backend.InverseRealSHT(self.h, self.w, lmax=modes_lat, mmax=modes_lon, grid=sht_grid_type).float()

    def _modes(self, hard_thresholding_fraction, max_modes):
        """modes = max_modes, else int(h * frac), int((w // 2 + 1) * frac)"""
        if max_modes is not None:
            return tuple(max_modes)
        return int(self.h * hard_thresholding_fraction), int((self.w // 2 + 1) * hard_thresholding_fraction)

    def _precompute_channel_groups(self, channel_names, aux_channel_names):
        atmo_chans, surf_chans, dyn_aux_chans, stat_aux_chans, pressure_lvls = get_channel_groups(channel_names, aux_channel_names)
        self.n_atmo_groups = len(pressure_lvls)
        self.n_atmo_chans = len(atmo_chans) // self.n_atmo_groups
        if len(atmo_chans) % self.n_atmo_groups:
            raise ValueError(f"Expected number of atmospheric variables to be divisible by number of atmospheric groups but got {len(atmo_chans)} and "
                             f"{self.n_atmo_groups}")
        self.register_buffer("atmo_channels", torch.LongTensor(atmo_chans), persistent=False)
        self.register_buffer("surf_channels", torch.LongTensor(surf_chans), persistent=False)
        self.register_buffer("aux_channels", torch.LongTensor(dyn_aux_chans + stat_aux_chans), persistent=False)
        self.n_surf_chans = self.surf_channels.shape[0]
        self.n_aux_chans = self.aux_channels.shape[0]

    def encode(self, x):
        """atmospheric levels through the shared encoder (levels folded into the batch), surface channels through theirs, concatenated"""
        batchdims = x.shape[:-3]
        x_atmo = x[..., self.atmo_channels, :, :].contiguous().reshape(-1, self.n_atmo_chans, *x.shape[-2:])
        x_out = self.atmo_encoder(x_atmo)
        x_out = x_out.reshape(*batchdims, self.n_atmo_groups * self.atmo_embed_dim, *x_out.shape[-2:])
        if hasattr(self, "surf_encoder"):
            x_out = torch.cat((x_out, self.surf_encoder(x[..., self.surf_channels, :, :].contiguous())), dim=-3)
        return x_out.reshape(*batchdims, self.total_embed_dim, *x_out.shape[-2:])

    def encode_auxiliary_channels(self, x):
        if not hasattr(self, "aux_encoder"):
            return None
        x_aux = self.aux_encoder(x[..., self.aux_channels, :, :])
        return x_aux.reshape(*x.shape[:-3], self.aux_embed_dim, *x_aux.shape[-2:])

    def decode(self, x):
        batchdims = x.shape[:-3]
        x_atmo = self.atmo_decoder(x[..., : (self.n_atmo_groups * self.atmo_embed_dim), :, :].reshape(-1, self.atmo_embed_dim, *x.shape[-2:]))
        x_out = torch.zeros(*batchdims, self.n_out_chans, *x_atmo.shape[-2:], dtype=x.dtype, device=x.device)
        x_out[..., self.atmo_channels, :, :] = x_atmo.reshape(*batchdims, -1, *x_atmo.shape[-2:])
        if hasattr(self, "surf_decoder"):
            x_surf = self.surf_decoder(x[..., -self.surf_embed_dim :, :, :])
            x_out[..., self.surf_channels, :, :] = x_surf.reshape(*batchdims, -1, *x_surf.shape[-2:])
        return x_out

    def process(self, x, x_aux=None):
        """the processor blocks, the embedded auxiliary channels appended to every block's input"""
        x = self.pos_drop(x)
        for blk in self.blocks:
            if x_aux is not None:
                x = torch.cat([x, x_aux], dim=-3)
            x = checkpoint(blk, x, use_reentrant=False) if self.checkpointing_level >= 3 else blk(x)
        return x

    def processor_blocks(self, x, x_aux=None):
        return self.process(x, x_aux)

    def encode_process(self, x):
        x_aux = self.encode_auxiliary_channels(x)
        x = checkpoint(self.encode, x, use_reentrant=False) if self.checkpointing_level >= 1 else self.encode(x)
        return self.process(x, x_aux)

    def clamp_water_channels(self, x):
        """water channels through the soft clamp (shifted by means / stds where the model carries its normalisation), others unchanged"""
        if hasattr(self, "water_channels"):
            if hasattr(self, "normalization_means") and hasattr(self, "normalization_stds"):
                means = self.normalization_means[self.water_channels].view(1, -1, 1, 1)
                stds = self.normalization_stds[self.water_channels].view(1, -1, 1, 1)
                offset = (means / stds).to(x.dtype)
                w = _soft_clamp(x[..., self.water_channels, :, :], offset=offset) - offset
            else:
                w = _soft_clamp(x[..., self.water_channels, :, :])
            w_full = torch.zeros_like(x)
            w_full.index_copy_(-3, self.water_channels, w.to(x.dtype))
            x = torch.where(self.water_channel_mask, w_full, x)
        return x

    def forward(self, x):
        if self.big_skip:
            residual = x[..., : self.n_out_chans, :, :].contiguous()
        x = self.encode_process(x)
        x = checkpoint(self.decode, x, use_reentrant=False) if self.checkpointing_level >= 1 else self.decode(x)
        if self.big_skip:
            x = x + self.residual_transform(residual)
        return self.clamp_water_channels(x)

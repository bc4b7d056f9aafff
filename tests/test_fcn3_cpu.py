"""makani_b200/fcn3.py (FourCastNet 3's AtmoSphericNeuralOperatorNet restated) against golden vectors produced by the REFERENCE's own network class
(tests/golden/make_fcn3_golden.py: makani/models/networks/fourcastnet3.py on the CPU oracles).  CPU: the network logic on the oracle backend (same
arithmetic as the golden run), the constructor surface and refusals of the CUDA-backed network."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

import makani_b200
from makani_b200 import fcn3, norm
from makani_b200.fcn3 import AtmoSphericNeuralOperatorNet
from oracle import makani_disco_oracle, makani_resample_oracle
from oracle.sfno_backend import OracleBackend

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_fcn3_golden import FCN3_GOLDEN_CASES, GRAD_KEYS, SHIPPED_AUX, n_inputs, tags  # noqa: E402

GOLD = os.path.join(os.path.dirname(__file__), "golden", "fcn3_golden.npz")

# config/fourcastnet3.yaml's 72 channel names
SHIPPED_72 = (["u10m", "v10m", "u100m", "v100m", "t2m", "msl", "tcwv"]
              + [f"{v}{p}" for v in "uvztq" for p in (50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925, 1000)])


class OracleFCN3Backend(OracleBackend):
    """the oracle transforms / SpectralConv / DISCO convolution / resampling; the instance norm is torch's nn.InstanceNorm2d, as makani builds it,
    and the layer norm and the spherical instance norm are the package's, whose CPU paths compute makani's formulas"""

    DiscreteContinuousConvS2 = makani_disco_oracle.DiscreteContinuousConvS2
    ResampleS2 = makani_resample_oracle.ResampleS2
    InstanceNorm2d = nn.InstanceNorm2d

    def __init__(self):
        super().__init__()
        self.LayerNorm = norm.DistributedLayerNorm
        self.GeometricInstanceNormS2 = norm.GeometricInstanceNormS2


def golden_state_dict(g, name):
    sd = {}
    for k in g.files:
        if k.startswith(f"{name}/sd/"):
            key = k[len(f"{name}/sd/"):]
            v = torch.from_numpy(g[k])
            sd[key] = torch.view_as_complex(v.contiguous()) if key.endswith("global_conv.weight") else v
    return sd


def _real(t):
    return torch.view_as_real(t) if t.is_complex() else t


@pytest.mark.parametrize("name", sorted(FCN3_GOLDEN_CASES))
def test_network_on_oracle_backend_matches_reference_network(name):
    g = np.load(GOLD)
    torch.manual_seed(0)
    net = AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], backend=OracleFCN3Backend())
    sd = golden_state_dict(g, name)
    assert sorted(net.state_dict().keys()) == sorted(sd.keys())
    net.load_state_dict(sd, strict=True)
    x = torch.from_numpy(g[f"{name}/x"]).requires_grad_(True)
    y = net(x)
    yref = torch.from_numpy(g[f"{name}/y"])
    assert torch.allclose(y, yref, rtol=1e-4, atol=1e-5), (y - yref).abs().max()
    (y * torch.from_numpy(g[f"{name}/g"])).sum().backward()
    assert torch.allclose(x.grad, torch.from_numpy(g[f"{name}/dx"]), rtol=1e-3, atol=1e-4)
    params = dict(net.named_parameters())
    for k in GRAD_KEYS[name]:
        ref = torch.from_numpy(g[f"{name}/grad/{k}"])
        assert torch.allclose(_real(params[k].grad), ref, rtol=1e-3, atol=1e-4 * ref.abs().max().item() + 1e-6), k


@pytest.mark.parametrize("name", sorted(FCN3_GOLDEN_CASES))
def test_batch_of_two_is_two_batches_of_one(name):
    """the encoders fold pressure levels into the batch and the decoders unfold them: a batch of two samples gives each sample's own output and
    input gradient (the golden vectors hold one sample)"""
    g = np.load(GOLD)
    net = AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], backend=OracleFCN3Backend())
    net.load_state_dict(golden_state_dict(g, name), strict=True)
    torch.manual_seed(1)
    x = torch.cat([torch.from_numpy(g[f"{name}/x"]), torch.randn_like(torch.from_numpy(g[f"{name}/x"]))]).requires_grad_(True)
    y = net(x)
    y.square().sum().backward()
    for b in range(2):
        xb = x[b : b + 1].detach().clone().requires_grad_(True)
        yb = net(xb)
        yb.square().sum().backward()
        assert torch.allclose(y[b : b + 1], yb, rtol=1e-5, atol=1e-6) and torch.allclose(x.grad[b : b + 1], xb.grad, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("name", sorted(FCN3_GOLDEN_CASES))
def test_cuda_backed_network_has_the_reference_parameter_surface(name):
    """constructed on the CPU (plans are created lazily on the device): names, shapes and dtypes of every state-dict entry, the model-parallel tags
    of every parameter, and the reference's checkpoint loads with strict=True"""
    g = np.load(GOLD)
    net = AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], precision="fp32")
    sd = golden_state_dict(g, name)
    mine = net.state_dict()
    assert list(mine.keys()) == [k[len(f"{name}/sd/"):] for k in g.files if k.startswith(f"{name}/sd/")]
    for k, v in sd.items():
        assert tuple(mine[k].shape) == tuple(v.shape) and mine[k].dtype == v.dtype, k
    assert json.loads(tags(net)) == json.loads(str(g[f"{name}/tags"]))
    net.load_state_dict(sd, strict=True)


@pytest.mark.parametrize("name", sorted(FCN3_GOLDEN_CASES))
def test_same_seed_draws_the_reference_parameters(name):
    """construction order and initialisation as the reference's: from the golden run's seed, every parameter the golden run did not perturb
    (weights other than norms and layer scales) comes out equal to the stored one"""
    g = np.load(GOLD)
    torch.manual_seed(333)
    net = AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], backend=OracleFCN3Backend())
    sd = golden_state_dict(g, name)
    for k, p in net.named_parameters():
        if not (k.endswith(".bias") or "norm" in k or "layer_scale" in k):
            assert torch.equal(p.detach(), sd[k]), k


def test_buffers_are_the_reference_channel_groups():
    cfg = FCN3_GOLDEN_CASES["shipped"]
    net = AtmoSphericNeuralOperatorNet(**cfg, backend=OracleFCN3Backend())
    names = cfg["channel_names"]
    assert [names[i] for i in net.atmo_channels] == [f"{v}{p}" for p in (500, 850) for v in "uvztq"]
    assert [names[i] for i in net.surf_channels] == ["u10m", "v10m", "t2m", "msl", "tcwv"]
    assert net.aux_channels.tolist() == list(range(len(names), len(names) + len(SHIPPED_AUX)))
    assert [names[i] for i in net.water_channels] == ["tcwv", "q500", "q850"]
    assert net.water_channel_mask.view(-1).nonzero().view(-1).tolist() == net.water_channels.tolist()
    assert not any(k in net.state_dict() for k in ("atmo_channels", "surf_channels", "aux_channels", "water_channels", "water_channel_mask"))


def test_channel_groups_of_the_shipped_config():
    """makani's get_channel_groups on config/fourcastnet3.yaml's 72 names and the aux names of its preprocessor: 13 levels of u, v, z, t, q and 7
    surface variables; orography and the land-sea masks static, zenith and noise dynamic"""
    aux = ["xzen"] + [f"xnoise{i}" for i in range(8)] + ["xoro", "xlsml", "xlsms"]
    atmo, surf, dyn_aux, stat_aux, levels = fcn3.get_channel_groups(SHIPPED_72, aux)
    assert list(levels) == [50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925, 1000]
    assert atmo == [v * 13 + lvl + 7 for lvl in range(13) for v in range(5)]
    assert surf == list(range(7))
    assert dyn_aux == list(range(72, 81)) and stat_aux == [81, 82, 83]
    assert fcn3.get_water_channels(SHIPPED_72) == [6] + list(range(7 + 4 * 13, 72))
    # "d2" is a surface variable; "u10m" does not end in digits
    assert fcn3.get_channel_groups(["d2", "t850", "u10m"])[:2] == ([1], [0, 2])


def test_shipped_processor_width():
    """the shipped configuration (13 levels x 45 + 56 surface + 36 aux = 677 processor channels) constructs on the CUDA backend on the CPU"""
    aux = ["xzen"] + [f"xnoise{i}" for i in range(8)] + ["xoro", "xlsml", "xlsms"]
    net = AtmoSphericNeuralOperatorNet(inp_shape=(721, 1440), out_shape=(721, 1440), scale_factor=2, atmo_embed_dim=45, surf_embed_dim=56,
                                       aux_embed_dim=36, num_layers=2, sfno_block_frequency=5, filter_basis_type="morlet", kernel_shape=[3, 3],
                                       channel_names=SHIPPED_72, aux_channel_names=aux, mlp_ratio=2, clamp_water=True)
    assert (net.h, net.w) == (360, 720) and net.n_out_chans == 72 and net.total_embed_dim == 641 and net.n_aux_chans == 12
    assert net.blocks[0].global_conv.weight.shape == (1, 677, 677, 360)
    assert net.blocks[1].local_conv.weight.shape == (677, 677, 9)
    assert net.blocks[1].mlp.fwd[3].weight.shape == (641, 1354, 1, 1)


def test_cutoff_and_soft_clamp():
    import math

    assert fcn3._compute_cutoff_radius(721, (3, 3), "morlet") == 4 * 0.5 * math.pi / 720
    assert fcn3._compute_cutoff_radius(10, (3, 3), "zernike") == 4 * math.sqrt(2.0) * math.pi / 9
    x = torch.tensor([-1.0, 0.0, 0.25, 0.5, 2.0])
    assert fcn3._soft_clamp(x).tolist() == [0.0, 0.0, 0.0625, 0.25, 1.75]
    assert fcn3._soft_clamp(x, offset=0.5).tolist() == [0.0, 0.25, 0.5, 0.75, 2.25]


def test_layer_scale_is_the_grouped_convolution():
    ls = fcn3.LayerScale(5)
    with torch.no_grad():
        ls.weight.copy_(torch.randn(5, 1, 1, 1))
    x = torch.randn(2, 5, 3, 4)
    assert torch.allclose(ls(x), nn.functional.conv2d(x, ls.weight, groups=5), rtol=1e-6, atol=1e-7)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        assert ls(x).dtype == nn.functional.conv2d(x, ls.weight, groups=5).dtype == torch.bfloat16


@pytest.mark.parametrize("level", [1, 2, 3])
def test_checkpointing_levels_give_the_same_result_on_the_oracle(level):
    name = "variant"
    g = np.load(GOLD)
    sd = golden_state_dict(g, name)
    out = []
    for lvl in (0, level):
        net = AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], checkpointing_level=lvl, backend=OracleFCN3Backend())
        net.load_state_dict(sd, strict=True)
        x = torch.from_numpy(g[f"{name}/x"]).requires_grad_(True)
        y = net(x)
        y.square().sum().backward()
        out.append((y.detach(), x.grad, [p.grad for p in net.parameters()]))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    assert all(torch.equal(a, b) for a, b in zip(out[0][2], out[1][2]))


def test_freeze_encoder_and_processor():
    cfg = FCN3_GOLDEN_CASES["variant"]
    net = AtmoSphericNeuralOperatorNet(**cfg, freeze_encoder=True, backend=OracleFCN3Backend())
    frozen = {k for k, p in net.named_parameters() if not p.requires_grad}
    assert frozen == {k for k, _ in net.named_parameters() if not k.startswith("blocks.")}
    net = AtmoSphericNeuralOperatorNet(**cfg, freeze_processor=True, backend=OracleFCN3Backend())
    frozen = {k for k, p in net.named_parameters() if not p.requires_grad}
    assert frozen == {k for k, _ in net.named_parameters() if k.startswith("blocks.")}


def test_normalization_layers():
    cfg = dict(FCN3_GOLDEN_CASES["no_surf_no_aux"])
    for kind, cls in (("instance_norm", norm.InstanceNorm2d), ("layer_norm", norm.DistributedLayerNorm),
                      ("instance_norm_s2", norm.GeometricInstanceNormS2), ("none", nn.Identity)):
        cfg["normalization_layer"] = kind
        net = AtmoSphericNeuralOperatorNet(**cfg)
        assert type(net.blocks[0].norm1) is cls and type(net.blocks[1].norm2) is cls
    cfg["normalization_layer"] = "instance_norm_s2"
    net = AtmoSphericNeuralOperatorNet(**cfg)
    assert net.blocks[0].norm1.grid_type == "legendre-gauss" and net.blocks[0].norm1.local_shape == (8, 16)
    cfg["normalization_layer"] = "batch_norm"
    with pytest.raises(NotImplementedError):
        AtmoSphericNeuralOperatorNet(**cfg)


def test_refusals():
    cfg = FCN3_GOLDEN_CASES["shipped"]
    with pytest.raises(ValueError, match="history"):
        AtmoSphericNeuralOperatorNet(**cfg | dict(n_history=1))
    with pytest.raises(ValueError, match="Unknown activation"):
        AtmoSphericNeuralOperatorNet(**cfg | dict(activation_function="tanh"))
    with pytest.raises(ValueError, match="same number of channels"):
        AtmoSphericNeuralOperatorNet(**cfg | dict(channel_names=["u500", "v500", "u850"]))
    with pytest.raises(NotImplementedError):     # the reference's default basis, as makani's class raises on this library's DISCO
        AtmoSphericNeuralOperatorNet(**{k: v for k, v in cfg.items() if k != "filter_basis_type"})
    with pytest.raises(ValueError, match="convolution type"):
        fcn3.NeuralOperatorBlock(makani_b200.RealSHT(16, 32, grid="legendre-gauss"), makani_b200.InverseRealSHT(16, 32, grid="legendre-gauss"), 4, 4,
                                 conv_type="spectral")


def test_cpu_tensors_on_the_cuda_backend_raise():
    name = "shipped"
    net = AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], precision="fp32")
    with pytest.raises(makani_b200.B200ShtError):
        net(torch.randn(1, n_inputs(FCN3_GOLDEN_CASES[name]), *FCN3_GOLDEN_CASES[name]["inp_shape"]))

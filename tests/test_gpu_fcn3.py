"""FourCastNet 3 on the GPU: makani_b200/fcn3.py's AtmoSphericNeuralOperatorNet on the CUDA kernels (DISCO, bilinear resampling, SHT pair and
dhconv SpectralConv, 1x1 GEMMs with the fused bias + GELU, norms), loaded with the REFERENCE network's state dict and compared with the REFERENCE
network's output and gradients (tests/golden/fcn3_golden.npz, produced by makani's fourcastnet3.py on the CPU oracles,
tests/golden/make_fcn3_golden.py); checkpointing, an autoregressive rollout and one step at the shipped geometry."""
import os
import sys

import numpy as np
import pytest
import torch

from makani_b200.fcn3 import AtmoSphericNeuralOperatorNet
from test_gpu_parity import close

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_fcn3_golden import FCN3_GOLDEN_CASES, GRAD_KEYS  # noqa: E402
from test_fcn3_cpu import GOLD, SHIPPED_72, golden_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
SHIPPED_AUX_12 = ["xzen"] + [f"xnoise{i}" for i in range(8)] + ["xoro", "xlsml", "xlsms"]


@pytest.fixture
def torch_tf32():
    """the DISCO channel GEMMs and the 1x1 convolutions run on cuBLAS and follow torch.backends.cuda.matmul.allow_tf32; the strict-fp32
    comparison switches it off"""
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


def _net(name, g, **kw):
    net = AtmoSphericNeuralOperatorNet(**(FCN3_GOLDEN_CASES[name] | kw))
    net.load_state_dict(golden_state_dict(g, name), strict=True)
    return net.to(DEV)


@pytest.mark.parametrize("name", sorted(FCN3_GOLDEN_CASES))
@pytest.mark.parametrize("precision,rtol,grtol", [("fp32", 1e-5, 1e-5), ("tf32", 2e-3, 8e-3)])
def test_fcn3_network_matches_reference_network(name, precision, rtol, grtol, torch_tf32):
    """bound: |err| <= rtol * (max|ref| + |ref|) per element (test_gpu_parity.close), rtol for y and grtol for dx and the parameter gradients.
    fp32: the golden run is itself fp32, so the difference is fp32 rounding in a different order.  On an H100 80GB HBM3 the largest err / bound
    was 0.037 for y and 0.27 for the gradients (the "variant" case's encoder MLP weight; relative L2 <= 2.7e-6).
    TF32: the SHT pair, the spectral mix, the DISCO channel GEMMs and the 1x1 GEMMs round their operands to 10 mantissa bits.  The largest
    err / bound was 0.51 for y and, at grtol 6e-3, 0.67 for the gradients, i.e. 0.51 of the 8e-3 here; both in the "variant" case (encoder /
    decoder MLPs, SHT upsampling, layer norm; relative L2 <= 3.6e-3).  Both TF32 bounds are below test_gpu_sfno.py's (4e-3, 1.5e-2)."""
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = (precision == "tf32")
    g = np.load(GOLD)
    net = _net(name, g, precision=precision)
    x = torch.from_numpy(g[f"{name}/x"]).to(DEV).requires_grad_(True)
    y = net(x)
    close(y, torch.from_numpy(g[f"{name}/y"]), rtol, f"FCN3[{name},{precision}] y")
    (y * torch.from_numpy(g[f"{name}/g"]).to(DEV)).sum().backward()
    close(x.grad, torch.from_numpy(g[f"{name}/dx"]), grtol, f"FCN3[{name},{precision}] dx")
    params = dict(net.named_parameters())
    for k in GRAD_KEYS[name]:
        ref = torch.from_numpy(g[f"{name}/grad/{k}"])
        got = params[k].grad
        close(torch.view_as_real(got) if got.is_complex() else got, ref, grtol, f"FCN3[{name},{precision}] d{k}")


def test_fcn3_network_bf16_autocast_runs_and_is_close():
    """the way makani trains (bf16 autocast around the network; transforms, DISCO contractions and decoders in fp32 / TF32): loose agreement with
    the fp32 golden output"""
    name = "shipped"
    g = np.load(GOLD)
    net = _net(name, g, precision="tf32")
    x = torch.from_numpy(g[f"{name}/x"]).to(DEV).requires_grad_(True)
    with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
        y = net(x)
    yref = torch.from_numpy(g[f"{name}/y"])
    rel = ((y.float().cpu() - yref).norm() / yref.norm()).item()
    print(f"[parity] FCN3[{name}] bf16 autocast rel_l2={rel:.3e}")
    assert torch.isfinite(y).all() and rel < 5e-2
    y.float().square().mean().backward()
    assert torch.isfinite(x.grad).all()


@pytest.mark.parametrize("level", [1, 2, 3])
def test_checkpointing_levels_are_bit_identical(level):
    """checkpointing recomputes the same deterministic kernels on the same inputs: outputs and every gradient equal level 0 bit for bit"""
    name = "variant"
    g = np.load(GOLD)
    res = []
    for lvl in (0, level):
        net = _net(name, g, precision="tf32", checkpointing_level=lvl)
        x = torch.from_numpy(g[f"{name}/x"]).to(DEV).requires_grad_(True)
        with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
            y = net(x)
        (y.float() * torch.from_numpy(g[f"{name}/g"]).to(DEV)).sum().backward()
        res.append([y.detach(), x.grad] + [p.grad for p in net.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*res))


def test_two_step_rollout_trains():
    """multistep 2 as makani trains it: the prediction, with the auxiliary channels appended, is the next input; the loss sums both steps"""
    name = "shipped"
    cfg = FCN3_GOLDEN_CASES[name]
    g = np.load(GOLD)
    net = _net(name, g, precision="tf32")
    x = torch.from_numpy(g[f"{name}/x"]).to(DEV).requires_grad_(True)
    n_out = len(cfg["channel_names"])
    targets = torch.randn(2, *g[f"{name}/y"].shape, device=DEV)
    loss, inp = 0.0, x
    with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
        for step in range(2):
            y = net(inp)
            loss = loss + (y.float() - targets[step]).square().mean()
            inp = torch.cat([y.float(), x[:, n_out:]], dim=1)
    loss.backward()
    assert torch.isfinite(loss)
    assert torch.isfinite(x.grad).all() and x.grad.abs().sum() > 0
    for k, p in net.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), k


def test_shipped_geometry_forward_backward():
    """config/fourcastnet3.yaml at full size: 721 x 1440 equiangular -> 360 x 720 Legendre-Gauss, 72 channels + 12 auxiliary (zenith, 8 noise,
    orography, 2 land-sea masks), 677 processor channels, 10 blocks, batch 1, bf16 autocast; one forward and backward, finite.  Without
    checkpointing the peak was 54.9 GiB on an H100 80GB HBM3, most of it the decoders' 20.4 GiB DISCO filter tensor on top of the saved activations."""
    torch.manual_seed(0)
    net = AtmoSphericNeuralOperatorNet(inp_shape=(721, 1440), out_shape=(721, 1440), scale_factor=2, kernel_shape=[3, 3], filter_basis_type="morlet",
                                       channel_names=SHIPPED_72, aux_channel_names=SHIPPED_AUX_12, atmo_embed_dim=45, surf_embed_dim=56,
                                       aux_embed_dim=36, num_layers=10, sfno_block_frequency=5, mlp_ratio=2, clamp_water=True).to(DEV)
    x = torch.randn(1, 84, 721, 1440, device=DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
        y = net(x)
    y.float().square().mean().backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2**30
    print(f"[fcn3] shipped geometry fwd+bwd, batch 1, bf16 autocast: peak memory {peak:.1f} GiB on {torch.cuda.get_device_name()}")
    assert y.shape == (1, 72, 721, 1440) and torch.isfinite(y).all()
    for k, p in net.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), k

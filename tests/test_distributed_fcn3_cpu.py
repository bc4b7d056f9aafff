"""FourCastNet 3 under h x w spatial model parallelism on CPU / gloo (makani_b200/fcn3.py on the grid of makani_b200.distributed, with
makani_b200/distributed/helpers.py), against the golden vectors of makani's own class (tests/golden/fcn3_golden.npz):

* for every FCN3_GOLDEN_CASES case on 2 x 1, 1 x 2 and 2 x 2: the golden state dict loaded through scatter_state_dict, forward and backward on
  this rank's shard of the 17 x 32 data grid (uneven latitude splits on the data grid; the 8 x 16 model grid and the modes split too), and the
  gathered output, input gradient and reduce_shared_gradients-reduced GRAD_KEYS gradients compared with makani's at test_fcn3_cpu.py's tolerance;
* gather_state_dict gives back the golden state dict bit for bit;
* after reduce_shared_gradients every replicated parameter's gradient is bit-identical on the ranks that share it, and sync_shared_params makes
  perturbed replicas equal again;
* the default backend builds the distributed classes, and every parameter carries the tags makani's class carries on the same grid;
* a grid that splits a dimension into more parts than it has points is refused at construction.

The per-rank stages are the oracle stand-ins of the other CPU distributed tests (SHT, DISCO window contraction, resampling, norm statistics) and
the dhconv spectral mix on this rank's (l, m) block; the CUDA stages are covered by tests/test_gpu_distributed_fcn3.py.  4 x 2 is not run: the
golden cases' surface decoder resamples five planes, fewer than DistributedResampleS2 spreads over 4 x 2 ranks."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn

import makani_b200.distributed as mbd
from makani_b200 import fcn3, norm
from makani_b200.distributed import helpers
from oracle import makani_norm_oracle as NO
from oracle import makani_oracle as O
from test_distributed_cpu import OracleLocalOps, _free_port
from test_distributed_disco_cpu import OracleDiscoLocalOps, OracleResampleLocalOps

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_fcn3_golden import FCN3_GOLDEN_CASES, GRAD_KEYS, tags  # noqa: E402
from test_fcn3_cpu import GOLD, golden_state_dict  # noqa: E402

# The tags that makani's AtmoSphericNeuralOperatorNet carries on an h x w grid where they differ from its serial ones (the `tags` of the golden
# file), read once from makani's class built on a 2 x 2 gloo grid in the environment of tests/reference_suites/run_reference_distributed_fcn3.py.
# The tags are the same on every rank and every grid of more than one rank (fourcastnet3.py:206-210, 382-386, 535-540; mpu/layer_norm.py).
_CONV = [["spatial"], [None, None, None]]
_BIAS = [["spatial"], [None]]
_NORM = [["spatial"], None]
DISTRIBUTED_TAGS = {
    "shipped": {k: _CONV for k in ("atmo_encoder.conv.weight", "surf_encoder.conv.weight", "aux_encoder.conv.weight", "blocks.1.local_conv.weight",
                                   "blocks.3.local_conv.weight", "atmo_decoder.conv.weight", "surf_decoder.conv.weight")},
    "variant": {**{k: _CONV for k in ("atmo_encoder.conv.weight", "surf_encoder.conv.weight", "aux_encoder.conv.weight", "blocks.1.local_conv.weight",
                                      "atmo_decoder.conv.weight", "surf_decoder.conv.weight")},
                **{k: _BIAS for k in ("atmo_encoder.conv.bias", "surf_encoder.conv.bias", "aux_encoder.conv.bias")}},
    "no_surf_no_aux": {**{k: _CONV for k in ("atmo_encoder.conv.weight", "blocks.1.local_conv.weight", "blocks.2.local_conv.weight",
                                             "atmo_decoder.conv.weight")},
                       **{f"blocks.{b}.norm{n}.{p}": _NORM for b in range(3) for n in (1, 2) for p in ("weight", "bias")}},
}


class OracleDistributedSpectralConv(nn.Module):
    """the dhconv SpectralConv on this rank's (l, m) block: the weight (G, C_in / G, C_out / G, l_local) is the "h" slice of makani's, the mix
    is local to every (l, m), the transforms are the distributed pair (oracle stages)"""

    def __init__(self, forward_transform, inverse_transform, in_channels, out_channels, num_groups=1, operator_type="dhconv", bias=False, gain=1.0):
        super().__init__()
        assert operator_type == "dhconv"
        self.forward_transform, self.inverse_transform, self.num_groups = forward_transform, inverse_transform, num_groups
        self.weight = nn.Parameter(torch.zeros(num_groups, in_channels // num_groups, out_channels // num_groups, inverse_transform.lmax_local,
                                               dtype=torch.complex64))
        self.weight.is_shared_mp = ["matmul", "w"]
        self.weight.sharded_dims_mp = [None, None, None, "h"]
        if bias:
            self.bias = nn.Parameter(torch.zeros(1, out_channels, 1, 1))
            self.bias.is_shared_mp = ["model"]
            self.bias.sharded_dims_mp = [None, None, None, None]

    def forward(self, x):
        with torch.autocast(device_type=x.device.type, enabled=False):
            xs = self.forward_transform(x.float())
            B, C, L, M = xs.shape
            ys = O.contract_dense(xs.reshape(B, self.num_groups, C // self.num_groups, L, M), self.weight.to(xs.dtype), operator_type="dhconv")
            y = self.inverse_transform(ys.reshape(B, -1, L, M)).float()
            if hasattr(self, "bias"):
                y = y + self.bias
        return y.to(x.dtype), x


class OracleDistributedBackend(fcn3._DistributedBackend):
    SpectralConv = OracleDistributedSpectralConv

    def __init__(self):
        super().__init__("fp32")
        self.SpectralConv = OracleDistributedSpectralConv


def _grid(rank, h, w):
    h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
    w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
    ih, iw = rank // w, rank % w
    mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
    return ih, iw


def _shard(t, ih, iw, h, w):
    t = torch.split(t, mbd.compute_split_shapes(t.shape[-2], h), dim=-2)[ih]
    return torch.split(t, mbd.compute_split_shapes(t.shape[-1], w), dim=-1)[iw].contiguous()


def _gather_grid(t):
    """this rank's (lat, lon) shard -> the whole field"""
    if mbd.azimuth_group_size() > 1:
        t = helpers._gather_uneven(t, t.dim() - 1, mbd.azimuth_group())
    if mbd.polar_group_size() > 1:
        t = helpers._gather_uneven(t, t.dim() - 2, mbd.polar_group())
    return t


def _gather_param(p, t):
    """a tensor shaped as this rank's shard of parameter `p` -> the global tensor (its "h" / "w" dimensions gathered)"""
    for d, tag in helpers._sharded_dims(p):
        t = helpers._gather_uneven(t, d, helpers._group_of(tag))
    return t


def _identical_over(t, group):
    """True where every rank of `group` holds the same bits"""
    if group is None:
        return True
    parts = [torch.empty_like(t) for _ in range(dist.get_world_size(group))]
    dist.all_gather(parts, t.contiguous(), group=group)
    return all(torch.equal(parts[0], p) for p in parts)


def _close(a, b, rtol, atol):
    return bool(torch.allclose(a, b, rtol=rtol, atol=atol)), float((a - b).abs().max())


def _worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        ih, iw = _grid(rank, h, w)
        mbd.set_local_ops(OracleLocalOps)
        mbd.set_disco_local_ops(OracleDiscoLocalOps)
        mbd.set_resample_local_ops(OracleResampleLocalOps)
        mbd.set_norm_local_ops(lambda layer: NO.OracleStages())
        g = np.load(GOLD)
        res = {}
        for name in sorted(FCN3_GOLDEN_CASES):
            cfg = FCN3_GOLDEN_CASES[name]
            # the default backend on the grid: the distributed classes and makani's tags
            default = fcn3.AtmoSphericNeuralOperatorNet(**cfg, precision="fp32")
            types = {type(m).__name__ for m in default.modules()}
            expected = {"DistributedDiscreteContinuousConvS2", "DistributedRealSHT", "DistributedInverseRealSHT"}
            expected |= {"DistributedResampleS2"} if not cfg.get("upsample_sht") else set()
            expected |= {"DistributedInstanceNorm2d"} if cfg.get("normalization_layer") == "instance_norm" else set()
            res[f"{name}/classes"] = expected <= types and not types & {"DiscreteContinuousConvS2", "RealSHT", "ResampleS2", "InstanceNorm2d"}
            want = json.loads(str(g[f"{name}/tags"])) | DISTRIBUTED_TAGS[name]
            res[f"{name}/tags default"] = json.loads(tags(default)) == want

            net = fcn3.AtmoSphericNeuralOperatorNet(**cfg, backend=OracleDistributedBackend())
            res[f"{name}/tags"] = json.loads(tags(net)) == want
            sd = golden_state_dict(g, name)
            net.load_state_dict(mbd.scatter_state_dict(net, sd), strict=True)
            back = mbd.gather_state_dict(net)
            res[f"{name}/gather_state_dict"] = list(back) == list(sd) and all(torch.equal(back[k], sd[k]) for k in sd)

            x = _shard(torch.from_numpy(g[f"{name}/x"]), ih, iw, h, w).requires_grad_(True)
            y = net(x)
            (y * _shard(torch.from_numpy(g[f"{name}/g"]), ih, iw, h, w)).sum().backward()
            mbd.reduce_shared_gradients(net)
            res[f"{name}/y"] = _close(_gather_grid(y.detach()), torch.from_numpy(g[f"{name}/y"]), 1e-4, 1e-5)
            res[f"{name}/dx"] = _close(_gather_grid(x.grad), torch.from_numpy(g[f"{name}/dx"]), 1e-3, 1e-4)
            params = dict(net.named_parameters())
            for k in GRAD_KEYS[name]:
                ref = torch.from_numpy(g[f"{name}/grad/{k}"])
                got = _gather_param(params[k], params[k].grad)
                got = torch.view_as_real(got) if got.is_complex() else got
                res[f"{name}/d{k}"] = _close(got, ref, 1e-3, 1e-4 * ref.abs().max().item() + 1e-6)
            # replicated gradients bit-identical on the ranks that share them: the whole grid, or the azimuth group of the dhconv weight
            same = True
            for k, p in params.items():
                grad = torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad
                for grp in helpers._shared_groups(p):
                    same = same and _identical_over(grad, grp)
            res[f"{name}/shared grads identical"] = same
            # sync_shared_params: replicas perturbed on every rank but the first of their groups take the first rank's values again
            with torch.no_grad():
                for p in params.values():
                    p.add_(sum(dist.get_rank(grp) for grp in helpers._shared_groups(p)))
            mbd.sync_shared_params(net)
            synced = mbd.gather_state_dict(net)
            res[f"{name}/sync_shared_params"] = all(torch.equal(synced[k], sd[k]) for k in sd)
        # over-split grids are refused at construction, naming the dimension
        over = dict(FCN3_GOLDEN_CASES["shipped"], max_modes=(1, 1))
        try:
            fcn3.AtmoSphericNeuralOperatorNet(**over, backend=OracleDistributedBackend())
            res["refusal"] = "constructed"
        except ValueError as e:
            res["refusal"] = str(e)
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", [(2, 1), (1, 2), (2, 2)])
def test_distributed_fcn3_matches_reference_network(h, w):
    world = h * w
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, h, w, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in out:
        assert err is None, f"rank {rank}:\n{err}"
        for k, v in res.items():
            if k == "refusal":
                group = "modes_lat = 1 cannot be split over the 2 ranks of the polar" if h > 1 else "modes_lon = 1 cannot be split over the 2 ranks"
                assert group in v, (rank, v)
            elif isinstance(v, tuple):
                assert v[0], (rank, k, v[1])
            else:
                assert v, (rank, k)


def test_serial_network_keeps_the_serial_classes_and_tags():
    """without a grid (or on a grid of one rank) nothing changes: the default backend is the single-GPU one and no spatial tags are added"""
    name = "no_surf_no_aux"
    net = fcn3.AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], precision="fp32")
    assert type(fcn3._default_backend()) is fcn3._Backend
    assert type(net.blocks[1].norm1) is norm.InstanceNorm2d and not any("Distributed" in type(m).__name__ for m in net.modules()
                                                                        if type(m).__name__ != "DistributedLayerNorm")
    assert json.loads(tags(net)) == json.loads(str(np.load(GOLD)[f"{name}/tags"]))


def test_helpers_reject_unknown_groups():
    p = nn.Parameter(torch.zeros(2))
    p.is_shared_mp = ["fin"]
    with pytest.raises(ValueError, match="fin"):
        helpers._shared_groups(p)
    p.sharded_dims_mp = ["spatial"]
    with pytest.raises(ValueError, match="spatial"):
        helpers._sharded_dims(p)

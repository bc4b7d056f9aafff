"""FourCastNet 3 under h x w spatial model parallelism on the CUDA kernels: makani_b200/fcn3.py on the grid of makani_b200.distributed, gloo ranks
sharing one GPU (as tests/test_gpu_distributed_attention_global.py), on 2 x 1, 1 x 2 and 2 x 2.  Every per-rank stage runs on the CUDA kernels;
the all-to-all exchanges between the ranks go through host copies, since gloo's point-to-point transport takes host tensors only.

For every FCN3_GOLDEN_CASES case, at fp32 and TF32, the golden state dict goes in through scatter_state_dict, forward and backward run on the
shards, and the gathered output, input gradient and reduce_shared_gradients-reduced GRAD_KEYS gradients are compared
* with makani's own class (tests/golden/fcn3_golden.npz) at tests/test_gpu_fcn3.py's bounds: fp32 rtol 1e-5; TF32 2e-3 for y, 8e-3 for gradients;
* with the single-GPU network of this package in the same process, at the same bounds.
Bound: |err| <= rtol * (max|ref| + |ref|) per element (test_gpu_parity.close).  The ranks run the single-GPU kernels on their shards; what the grid
changes is the order of a few sums (the norm statistics over ranks, the DISCO halo adjoint, the weight gradients summed over ranks), so the
serial bounds hold.  Each comparison prints its need (max err / bound).  On an H100 80GB HBM3 (700 W power limit) the largest need over the three
grids against the golden vectors was 0.034 for y and 0.21 for the gradients at fp32, 0.23 and 0.50 at TF32; against the single-GPU network 0.015
and 0.14 at fp32, 0.39 and 0.52 at TF32 (the "variant" case: encoder MLP weight, dhconv bias, 2 x 2 output).
Also: checkpointing levels 1-3 bit-identical to level 0 on the same grid, a two-step rollout and bf16 autocast with finite outputs and gradients."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import makani_b200.distributed as mbd
from makani_b200.distributed import disco as DD
from makani_b200.distributed import primitives
from makani_b200.fcn3 import AtmoSphericNeuralOperatorNet
from test_distributed_cpu import _free_port
from test_distributed_fcn3_cpu import _gather_grid, _gather_param, _grid, _shard

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
from make_fcn3_golden import FCN3_GOLDEN_CASES, GRAD_KEYS  # noqa: E402
from test_fcn3_cpu import GOLD, golden_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
BOUNDS = {"fp32": (1e-5, 1e-5), "tf32": (2e-3, 8e-3)}


def _need(a, b, rtol):
    """max |a - b| / (rtol (max|b| + |b|)); inf where a is not finite"""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    if not torch.isfinite(a).all():
        return float("inf")
    return ((a - b).abs() / (rtol * (b.abs().max() + b.abs())).clamp_min(1e-300)).max().item()


def _real(t):
    return torch.view_as_real(t) if t.is_complex() else t


def _run(net, x, gy, keys):
    """forward + backward of sum(y gy); -> y, dx and the gradients of `keys`, gathered to the global tensors"""
    x = x.clone().requires_grad_(True)
    y = net(x)
    (y * gy).sum().backward()
    if mbd.polar_group_size() * mbd.azimuth_group_size() > 1:
        mbd.reduce_shared_gradients(net)
    params = dict(net.named_parameters())
    grads = {k: _real(_gather_param(params[k], params[k].grad)).cpu() for k in keys}
    return _gather_grid(y.detach()).cpu(), _gather_grid(x.grad).cpu(), grads


def _stage_all_to_all_through_host():
    """gloo's send / recv take host tensors only: the ranks' exchanges of CUDA shards (the transposes and the DISCO halo) go through host copies
    here; with NCCL the same choreography is one dist.all_to_all of the device tensors"""
    real = primitives._all_to_all

    def staged(recv, send, group):
        host = [torch.empty(r.shape, dtype=r.dtype) for r in recv]
        real(host, [s.cpu() for s in send], group)
        for r, t in zip(recv, host):
            r.copy_(t)

    primitives._all_to_all = DD._all_to_all = staged


def _worker(rank, world, port, h, w, q):
    try:
        torch.cuda.set_device(0)
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        _stage_all_to_all_through_host()
        g = np.load(GOLD)
        res = {}
        # the single-GPU network first, before the grid exists
        serial = {}
        for name in sorted(FCN3_GOLDEN_CASES):
            for prec in BOUNDS:
                torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = prec == "tf32"
                net = AtmoSphericNeuralOperatorNet(**FCN3_GOLDEN_CASES[name], precision=prec)
                net.load_state_dict(golden_state_dict(g, name), strict=True)
                serial[name, prec] = _run(net.to(DEV), torch.from_numpy(g[f"{name}/x"]).to(DEV), torch.from_numpy(g[f"{name}/g"]).to(DEV),
                                          GRAD_KEYS[name])
        ih, iw = _grid(rank, h, w)

        def sharded(name, prec, **kw):
            torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = prec == "tf32"
            net = AtmoSphericNeuralOperatorNet(**(FCN3_GOLDEN_CASES[name] | kw), precision=prec)
            net.load_state_dict(mbd.scatter_state_dict(net, golden_state_dict(g, name)), strict=True)
            return net.to(DEV)

        def inputs(name):
            return tuple(_shard(torch.from_numpy(g[f"{name}/{k}"]), ih, iw, h, w).to(DEV) for k in ("x", "g"))

        for name in sorted(FCN3_GOLDEN_CASES):
            for prec, (rtol, grtol) in BOUNDS.items():
                y, dx, grads = _run(sharded(name, prec), *inputs(name), GRAD_KEYS[name])
                sy, sdx, sgrads = serial[name, prec]
                for ref_name, ref in (("golden", (torch.from_numpy(g[f"{name}/y"]), torch.from_numpy(g[f"{name}/dx"]),
                                                  {k: torch.from_numpy(g[f"{name}/grad/{k}"]) for k in GRAD_KEYS[name]})),
                                      ("serial", (sy, sdx, sgrads))):
                    res[f"{name}/{prec}/{ref_name}/y"] = (_need(y, ref[0], rtol), 1.0)
                    res[f"{name}/{prec}/{ref_name}/dx"] = (_need(dx, ref[1], grtol), 1.0)
                    for k in GRAD_KEYS[name]:
                        res[f"{name}/{prec}/{ref_name}/d{k}"] = (_need(grads[k], ref[2][k], grtol), 1.0)

        # checkpointing levels 1-3 against level 0 on the same grid, bit for bit (bf16 autocast, TF32)
        name = "variant"
        x, gy = inputs(name)
        runs = []
        for lvl in (0, 1, 2, 3):
            net = sharded(name, "tf32", checkpointing_level=lvl)
            xl = x.clone().requires_grad_(True)
            with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
                yl = net(xl)
            (yl.float() * gy).sum().backward()
            mbd.reduce_shared_gradients(net)
            runs.append([yl.detach(), xl.grad] + [p.grad for p in net.parameters()])
        for lvl in (1, 2, 3):
            res[f"checkpointing {lvl}"] = (0.0 if all(torch.equal(a, b) for a, b in zip(runs[0], runs[lvl])) else float("inf"), 0.0)

        # a two-step rollout under bf16 autocast: finite loss and gradients, every parameter reached
        name = "shipped"
        n_out = len(FCN3_GOLDEN_CASES[name]["channel_names"])
        net = sharded(name, "tf32")
        x, _ = inputs(name)
        x = x.clone().requires_grad_(True)
        torch.manual_seed(11)
        targets = _shard(torch.randn(2, 1, n_out, *FCN3_GOLDEN_CASES[name]["out_shape"]), ih, iw, h, w).to(DEV)
        loss, inp = 0.0, x
        with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
            for step in range(2):
                y = net(inp)
                loss = loss + (y.float() - targets[step]).square().mean()
                inp = torch.cat([y.float(), x[:, n_out:]], dim=1)
        loss.backward()
        mbd.reduce_shared_gradients(net)
        finite = bool(torch.isfinite(loss)) and bool(torch.isfinite(x.grad).all()) and all(
            p.grad is not None and bool(torch.isfinite(p.grad).all()) for p in net.parameters())
        res["rollout finite"] = (0.0 if finite else float("inf"), 0.0)
        res["bf16 autocast y finite"] = (0.0 if bool(torch.isfinite(y).all()) else float("inf"), 0.0)
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", [(2, 1), (1, 2), (2, 2)])
def test_distributed_fcn3_on_one_gpu(h, w):
    world = h * w
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, h, w, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = sorted([q.get(timeout=1200) for _ in range(world)], key=lambda o: o[0])
    for p in procs:
        p.join(timeout=60)
    errs = [f"rank {rank}:\n{err}" for rank, _, err in out if err is not None]
    assert not errs, "\n".join(errs)
    worst = {}
    for rank, res, _ in out:
        for k, (need, limit) in res.items():
            worst[k] = max(worst.get(k, 0.0), need)
    for k, need in sorted(worst.items()):
        print(f"[parity] FCN3 {h}x{w} {k}: max err/bound over ranks {need:.3f}")
    bad = {k: v for k, v in worst.items() if v > out[0][1][k][1]}
    assert not bad, bad

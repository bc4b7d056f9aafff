"""gloo tests (CPU) of DistributedInstanceNorm2d (makani_b200/distributed/norm.py, makani's DistributedInstanceNorm2d) at h x w = 1 x 2, 2 x 1,
2 x 2 and 4 x 2, with uneven splits (181 x 360, 17 x 33), against fp64 `F.instance_norm` of the whole field:

* the output and the input gradient of every shard, and the parameter gradients summed over the ranks (makani's gradient hooks add the local
  partials), affine and not, B = 2;
* the statistics (mu, r, corr) identical bit for bit on every rank, and the normaliser D = the global point count, cached per local shape;
* both per-rank stages: the oracle's fp64 stages with q = 1 (`set_norm_local_ops`) and the module's own torch-operator stages that CPU tensors take;
* the constructor contract of makani's class, a 1 x 1 grid, and `compat.patch_makani_instance_norm()`.
The CUDA stages are covered by tests/test_gpu_distributed_instance_norm.py."""
import inspect
import os
import sys
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F

import makani_b200.distributed as mbd
from makani_b200 import norm as N
from oracle import makani_norm_oracle as O
from test_distributed_cpu import _free_port

# H, W, affine, B, C
CASES = [(181, 360, True, 2, 3), (17, 33, False, 2, 4), (181, 360, False, 2, 2), (17, 33, True, 2, 5)]
GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
EPS = 1e-5


class _Recording:
    """the stages, keeping the statistics of the last finalize"""

    def __init__(self, inner):
        self.inner, self.last_stats = inner, None

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def finalize(self, parts, D, eps):
        self.last_stats = self.inner.finalize(parts, D, eps)
        return self.last_stats


def _reference(x, dy, weight, bias):
    """fp64 F.instance_norm of the whole field: y, dx, dweight, dbias"""
    xr = x.clone().requires_grad_(True)
    pr = [p.detach().double().requires_grad_(True) for p in (weight, bias)] if weight is not None else [None, None]
    yr = F.instance_norm(xr, weight=pr[0], bias=pr[1], eps=EPS)
    yr.backward(dy)
    return yr.detach(), xr.grad, pr[0].grad if weight is not None else None, pr[1].grad if weight is not None else None


def _worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
        w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
        ih, iw = rank // w, rank % w
        mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
        res = {}
        for stage_kind in ("oracle", "torch"):
            for n, (H, W, affine, B, C) in enumerate(CASES):
                rec = _Recording(O.OracleStages() if stage_kind == "oracle" else N.TorchGeometricNormStages())
                mbd.set_norm_local_ops(lambda layer: rec)
                mod = mbd.DistributedInstanceNorm2d(C, eps=EPS, affine=affine)
                mbd.set_norm_local_ops(None)
                plain = mbd.DistributedInstanceNorm2d(C, eps=EPS, affine=affine)    # no replacement: CPU tensors take the torch stages
                hs, ws = O.split_shapes(H, h), O.split_shapes(W, w)
                g = torch.Generator().manual_seed(60 + n)
                if affine:
                    with torch.no_grad():
                        for m in (mod, plain):
                            m.weight.copy_(1.0 + 0.3 * torch.randn(C, generator=torch.Generator().manual_seed(n)))
                            m.bias.copy_(0.2 * torch.randn(C, generator=torch.Generator().manual_seed(n + 100)))
                x = 2.0 + torch.randn(B, C, H, W, dtype=torch.float64, generator=g)
                dy = torch.randn(B, C, H, W, dtype=torch.float64, generator=g)

                def shard(t):
                    t = torch.split(t, hs, dim=-2)[ih]
                    return torch.split(t, ws, dim=-1)[iw].contiguous()

                dt = torch.float64 if stage_kind == "oracle" else torch.float32
                xl = shard(x).to(dt).requires_grad_(True)
                y = mod(xl)
                y.backward(shard(dy).to(dt))
                assert y.dtype == dt and y.shape == xl.shape
                yr, dxr, dwr, dbr = _reference(x, dy, mod.weight if affine else None, mod.bias if affine else None)
                rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
                key = f"{stage_kind}{n}"
                res[f"{key}/y"] = rel(y.detach(), shard(yr))
                res[f"{key}/dx"] = rel(xl.grad, shard(dxr))
                if affine:
                    for name, r in (("weight", dwr), ("bias", dbr)):
                        tot = getattr(mod, name).grad.clone()
                        dist.all_reduce(tot)
                        res[f"{key}/d{name}"] = rel(tot, r)
                res[f"{key}/D"] = float(mod._points != {(hs[ih], ws[iw]): float(H * W)})
                st = rec.last_stats.double().contiguous()
                every = [torch.empty_like(st) for _ in range(world)]
                dist.all_gather(every, st)
                res[f"{key}/stats_identical"] = float(not all(torch.equal(e, every[0]) for e in every))
                if stage_kind == "torch":
                    xp = shard(x).float().requires_grad_(True)
                    yp = plain(xp)
                    yp.backward(shard(dy).float())
                    res[f"{key}/default_stages_equal"] = float(not (torch.equal(yp, y.detach()) and torch.equal(xp.grad, xl.grad)))
        # one module, two local shapes: D is exchanged once per shape and cached
        mod = mbd.DistributedInstanceNorm2d(3)
        for H, W in ((181, 360), (17, 33), (181, 360)):
            hs, ws = O.split_shapes(H, h), O.split_shapes(W, w)
            mod(torch.randn(1, 3, hs[ih], ws[iw]))
        res["cache/D"] = float(mod._points != {(O.split_shapes(181, h)[ih], O.split_shapes(360, w)[iw]): 181.0 * 360,
                                              (O.split_shapes(17, h)[ih], O.split_shapes(33, w)[iw]): 17.0 * 33})
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", GRIDS)
def test_distributed_instance_norm_matches_fp64_instance_norm(h, w):
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
        for kind in ("oracle", "torch"):
            for n, case in enumerate(CASES):
                want = {"y", "dx", "D", "stats_identical"} | ({"dweight", "dbias"} if case[2] else set()) | ({"default_stages_equal"} if kind == "torch" else set())
                assert {k.split("/")[1] for k in res if k.startswith(f"{kind}{n}/")} == want
        for k, v in res.items():
            # flags must be 0; the oracle's stages run in fp64 (parameter gradients returned in fp32), the torch stages normalise in fp32
            tol = 0.0 if k.split("/")[1] in ("D", "stats_identical", "default_stages_equal") else (1e-6 if k.startswith("oracle") else 2e-5)
            assert v <= tol, (rank, k, v)


def test_constructor_contract():
    sig = inspect.signature(mbd.DistributedInstanceNorm2d.__init__)
    assert [(p.name, p.default) for p in list(sig.parameters.values())[1:]] == [
        ("num_features", inspect.Parameter.empty), ("eps", 1e-05), ("affine", False)]
    assert mbd.DistributedInstanceNorm2d.__name__ == "DistributedInstanceNorm2d"
    m = mbd.DistributedInstanceNorm2d(6, eps=1e-6, affine=True)
    assert m.eps == 1e-6 and m.affine
    assert [(n, tuple(p.shape)) for n, p in m.named_parameters()] == [("weight", (6,)), ("bias", (6,))]
    assert torch.equal(m.weight, torch.ones(6)) and torch.equal(m.bias, torch.zeros(6))
    assert m.weight.is_shared_mp == ["spatial"] and m.bias.is_shared_mp == ["spatial"]
    assert list(m.state_dict().keys()) == ["weight", "bias"]
    m(torch.randn(2, 6, 5, 7))
    assert list(m.state_dict().keys()) == ["weight", "bias"]      # the cached weights and point counts are not state
    sd = {"weight": torch.randn(6), "bias": torch.randn(6)}
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.weight, sd["weight"])
    na = mbd.DistributedInstanceNorm2d(6)
    assert list(na.parameters()) == [] and list(na.state_dict().keys()) == [] and not na.affine
    assert na(torch.randn(1, 11, 4, 5)).shape == (1, 11, 4, 5)     # without affine, any channel count (as makani's layer)
    with pytest.raises(ValueError):
        m(torch.randn(2, 5, 4, 4))
    with pytest.raises(ValueError):
        m(torch.randn(6, 4, 4))


@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.bfloat16])
def test_one_rank_grid_matches_instance_norm(affine, dtype):
    """on a 1 x 1 grid the class is nn.InstanceNorm2d; the output keeps the input's dtype, computed in fp32 as makani's layer (also under autocast)"""
    mbd.init(None, None)
    try:
        torch.manual_seed(5)
        mod = mbd.DistributedInstanceNorm2d(4, affine=affine)
        if affine:
            with torch.no_grad():
                mod.weight.add_(0.3 * torch.randn(4))
                mod.bias.add_(0.2 * torch.randn(4))
        x = (3.0 + torch.randn(2, 4, 17, 33, dtype=torch.float64)).to(dtype).requires_grad_(True)
        dy = torch.randn(2, 4, 17, 33, dtype=torch.float64)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            y = mod(x)
        y.backward(dy.to(dtype))
        assert y.dtype == dtype
        yr, dxr, dwr, dbr = _reference(x.detach().double(), dy, mod.weight if affine else None, mod.bias if affine else None)
        tol = 1e-2 if dtype == torch.bfloat16 else 1e-5
        rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
        assert rel(y.detach(), yr) < tol and rel(x.grad, dxr) < (2e-2 if dtype == torch.bfloat16 else 1e-5)
        if affine:
            assert rel(mod.weight.grad, dwr) < tol and rel(mod.bias.grad, dbr) < tol
        assert mod._points == {(17, 33): 17.0 * 33}
    finally:
        mbd.finalize()


def test_compat_patch_points_makani_names_at_the_class(monkeypatch):
    from makani_b200 import compat

    class Theirs(nn.Module):
        pass

    class TheirLayerNorm(nn.Module):
        pass

    mods = {}
    for name in ("makani", "makani.mpu", "makani.mpu.layer_norm", "makani.models", "makani.models.networks", "makani.models.networks.sfnonet",
                 "makani.models.networks.snonet"):
        mods[name] = types.ModuleType(name)
        monkeypatch.setitem(sys.modules, name, mods[name])
    for name in ("makani.mpu.layer_norm", "makani.models.networks.sfnonet", "makani.models.networks.snonet"):
        mods[name].DistributedInstanceNorm2d = Theirs
        mods[name].DistributedLayerNorm = TheirLayerNorm
    compat.patch_makani_instance_norm()
    for name in ("makani.mpu.layer_norm", "makani.models.networks.sfnonet", "makani.models.networks.snonet"):
        assert mods[name].DistributedInstanceNorm2d is mbd.DistributedInstanceNorm2d, name
        assert mods[name].DistributedLayerNorm is TheirLayerNorm, name      # the layer norm has its own patch

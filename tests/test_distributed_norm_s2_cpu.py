"""gloo tests (CPU) of DistributedGeometricInstanceNormS2 (makani_b200/distributed/norm.py) at h x w = 2 x 1, 1 x 2, 2 x 2 and 4 x 2, with uneven
splits (181 x 360 equiangular, 180 x 360 Legendre-Gauss, 49 x 97 Clenshaw-Curtis, a partial crop of a weatherbench2 grid), against the SERIAL
fp64 oracle of the class on the whole global crop (oracle/makani_norm_oracle.py, normaliser D = the crop's weight):

* the output, the input gradient and the parameter gradients summed over the ranks (makani's gradient hooks add the local partials), with and
  without GELU, affine and not;
* the statistics (mu, r, corr) identical bit for bit on every rank;
* both per-rank stages: the oracle's fp64 stand-in for the kernels (`set_norm_local_ops`) and the module's own torch-operator stages that CPU
  tensors take.
The CUDA stages are covered by tests/test_gpu_norm_s2.py."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import makani_b200.distributed as mbd
from makani_b200 import norm as N
from oracle import makani_norm_oracle as O
from test_distributed_cpu import _free_port

# img_shape, crop_shape, crop_offset, grid, affine, gelu, B, C
CASES = [
    ((181, 360), (181, 360), (0, 0), "equiangular", True, True, 1, 3),
    ((180, 360), (180, 360), (0, 0), "legendre-gauss", True, False, 2, 2),
    ((49, 97), (49, 97), (0, 0), "clenshaw-curtiss", False, False, 2, 3),
    ((60, 120), (37, 75), (11, 20), "weatherbench2", True, True, 2, 2),
]
GRIDS = [(2, 1), (1, 2), (2, 2), (4, 2)]


class _Recording:
    """the stages, keeping the statistics of the last finalize"""

    def __init__(self, inner):
        self.inner, self.last_stats = inner, None

    def __getattr__(self, name):
        return getattr(self.inner, name)

    def finalize(self, parts, D, eps):
        self.last_stats = self.inner.finalize(parts, D, eps)
        return self.last_stats


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
            for n, (img, cs, co, grid, affine, gelu, B, C) in enumerate(CASES):
                rec = {}
                if stage_kind == "oracle":
                    mbd.set_norm_local_ops(lambda layer: rec.setdefault("s", _Recording(O.OracleStages())))
                else:
                    stages = _Recording(N.TorchGeometricNormStages())
                    rec["s"] = stages
                    mbd.set_norm_local_ops(lambda layer: stages)
                mod = mbd.DistributedGeometricInstanceNormS2(img, cs, co, grid, C, eps=1e-5, affine=affine)
                mbd.set_norm_local_ops(None)
                hs, ws = O.split_shapes(cs[0], h), O.split_shapes(cs[1], w)
                assert mod.local_shape == (hs[ih], ws[iw])
                g = torch.Generator().manual_seed(40 + n)
                if affine:
                    with torch.no_grad():
                        mod.weight.copy_(1.0 + 0.3 * torch.randn(C, generator=g))
                        mod.bias.copy_(0.2 * torch.randn(C, generator=g))
                x = 2.0 + torch.randn(B, C, *cs, dtype=torch.float64, generator=g)
                dy = torch.randn(B, C, *cs, dtype=torch.float64, generator=g)

                def shard(t):
                    t = torch.split(t, hs, dim=-2)[ih]
                    return torch.split(t, ws, dim=-1)[iw].contiguous()

                dt = torch.float64 if stage_kind == "oracle" else torch.float32
                xl = shard(x).to(dt).requires_grad_(True)
                y = mod(xl, gelu=gelu)
                y.backward(shard(dy).to(dt))
                qg = O.grid_quadrature(grid, img, cs, co)
                xr = x.clone().requires_grad_(True)
                pr = [p.detach().double().requires_grad_(True) for p in mod.parameters()]
                yr = O.distributed(xr, qg, 1e-5, *(pr if affine else (None, None)), gelu=gelu)
                yr.backward(dy)
                rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
                key = f"{stage_kind}{n}"
                res[f"{key}/y"] = rel(y.detach(), shard(yr.detach()))
                res[f"{key}/dx"] = rel(xl.grad, shard(xr.grad))
                for (name, p), r in zip(mod.named_parameters(), pr):
                    tot = p.grad.clone()
                    dist.all_reduce(tot)
                    res[f"{key}/d{name}"] = rel(tot, r.grad)
                st = rec["s"].last_stats.double().contiguous()
                every = [torch.empty_like(st) for _ in range(world)]
                dist.all_gather(every, st)
                res[f"{key}/stats_identical"] = float(not all(torch.equal(e, every[0]) for e in every))
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", GRIDS)
def test_distributed_geometric_norm_matches_serial_oracle(h, w):
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
                want = {"y", "dx", "stats_identical"} | ({"dweight", "dbias"} if case[4] else set())
                assert {k.split("/")[1] for k in res if k.startswith(f"{kind}{n}/")} == want
        for k, v in res.items():
            # the oracle stand-in runs in fp64 on float32-rounded weights; the torch stages normalise in fp32
            tol = 0.0 if k.endswith("stats_identical") else (1e-6 if k.startswith("oracle") else 2e-5)
            assert v <= tol, (rank, k, v)


def test_one_rank_grid_matches_serial_class():
    """on a 1 x 1 grid the distributed class is the serial formula with D = the crop's weight"""
    mbd.init(None, None)
    try:
        mod = mbd.DistributedGeometricInstanceNormS2((24, 48), (20, 40), (2, 4), "legendre-gauss", 3, affine=True)
        x = torch.randn(2, 3, 20, 40, dtype=torch.float64).requires_grad_(True)
        y = mod(x.float())
        qg = O.grid_quadrature("legendre-gauss", (24, 48), (20, 40), (2, 4))
        yr = O.distributed(x, qg, 1e-5, torch.ones(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64))
        assert ((y.double() - yr).abs().max() / yr.abs().max()).item() < 1e-5
    finally:
        mbd.finalize()


def test_shim_names_the_class():
    import importlib
    import sys

    import makani_b200.compat as compat

    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        compat.install_torch_harmonics_shim()
        assert importlib.import_module("torch_harmonics.distributed").DistributedGeometricInstanceNormS2 is mbd.DistributedGeometricInstanceNormS2
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)

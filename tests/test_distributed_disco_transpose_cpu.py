"""CPU tests of DistributedDiscreteContinuousConvTransposeS2 (makani_b200/distributed/disco.py) on gloo, world sizes 2 to 8: the whole
choreography (local GEMM, azimuth all-to-all, window adjoint, halo adjoint, and the mirror image in the backward) with the per-rank stages on
the oracle's dense psi_T, against the SERIAL fp64 oracle: the gathered y, dx, dW and dbias, on uneven latitude splits; and the refusals at
B * C_out < w and at a grid of one rank.  The CUDA stages are covered by tests/test_gpu_disco_transpose.py."""
import math
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import disco_transpose_oracle as TO
import makani_b200.distributed as mbd
from oracle import makani_disco_oracle as DO
from test_distributed_cpu import _free_port


class OracleTransposeLocalOps:
    """the window contraction and its adjoint on the oracle's dense psi_T, restricted to this rank's window: plan output rows t0 .. t1 are
    in-grid latitudes, the window lo .. hi out-grid latitudes"""

    def __init__(self, layer):
        w = layer.window
        psi = TO.dense_psi_T(layer.kernel_shape, layer.basis_norm_mode, (layer.nlat_in, layer.nlon_in), (layer.nlat_out, layer.nlon_out),
                             layer.grid_in, layer.grid_out, layer.theta_cutoff)
        outside = psi[:, w.t0 : w.t1].clone()
        outside[:, :, w.lo : w.hi] = 0
        assert not outside.any(), "oracle psi_T reaches outside the window"
        self.K, self.nt, self.nwin = layer.kernel_size, w.t1 - w.t0, w.hi - w.lo
        self.nlon_in, self.nlon_out = layer.nlon_in, layer.nlon_out
        self.psi = psi[:, w.t0 : w.t1, w.lo : w.hi].reshape(self.K * self.nt, -1)

    def contract(self, gwin):
        return DO.contraction(gwin.double().unsqueeze(1), self.psi, self.K, self.nt, self.nlon_in)[:, 0].float()

    def adjoint(self, Y):
        return TO.transpose_contraction(Y.double().unsqueeze(1), self.psi, self.nwin, self.nlon_out)[:, 0].float()


# (C_in, C_out, in_shape, out_shape, kernel_shape, groups, bias, grid_in, grid_out, norm, cutoff in out-grid spacings)
CASES = [(4, 6, (17, 32), (33, 64), (3, 3), 2, True, "equiangular", "equiangular", "mean", 3.0),
         (6, 4, (19, 30), (19, 30), (2, 3), 2, False, "legendre-gauss", "legendre-gauss", "support", 2.5),
         (3, 3, (16, 32), (31, 64), (3, 3), 3, True, "legendre-gauss", "equiangular", "individual", 4.0),
         (2, 1, (17, 32), (17, 32), (3, 3), 1, True, "equiangular", "equiangular", "none", 6.0)]   # C_out = 1 < w: B*C_out rows are split


def _worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
        w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
        ih, iw = rank // w, rank % w
        mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
        mbd.set_disco_local_ops(OracleTransposeLocalOps)
        res = {}

        def shard(t, hs, ws):
            return torch.split(torch.split(t, hs, dim=-2)[ih], ws, dim=-1)[iw].contiguous()

        def allsum(t):
            t = t.clone()
            dist.all_reduce(t)
            return t

        for n, (cin, cout, ish, osh, ks, G, bias, gi, go, norm, u) in enumerate(CASES):
            kw = dict(basis_type="morlet", basis_norm_mode=norm, groups=G, grid_in=gi, grid_out=go, bias=bias,
                      theta_cutoff=u * math.pi / (osh[0] - 1))
            torch.manual_seed(17)
            ref = TO.DiscreteContinuousConvTransposeS2(cin, cout, ish, osh, ks, **kw).double()
            mod = mbd.DistributedDiscreteContinuousConvTransposeS2(cin, cout, ish, osh, ks, **kw)
            with torch.no_grad():
                mod.weight.copy_(ref.weight)
                if bias:
                    ref.bias.normal_()
                    mod.bias.copy_(ref.bias)
            x = torch.randn(2, cin, *ish, dtype=torch.float64)
            gy = torch.randn(2, cout, *osh, dtype=torch.float64)
            xs = x.clone().requires_grad_(True)
            ys = ref(xs)
            ys.backward(gy)
            xd = shard(x, mod.lat_in_shapes, mod.lon_in_shapes).float().requires_grad_(True)
            yd = mod(xd)
            assert yd.shape == (2, cout, mod.nlat_out_local, mod.nlon_out_local) and yd.dtype == torch.float32
            yd.backward(shard(gy, mod.lat_out_shapes, mod.lon_out_shapes).float())
            rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
            res[f"disco{n}/y"] = rel(yd.detach(), shard(ys.detach(), mod.lat_out_shapes, mod.lon_out_shapes))
            res[f"disco{n}/dx"] = rel(xd.grad, shard(xs.grad, mod.lat_in_shapes, mod.lon_in_shapes))
            res[f"disco{n}/dw"] = rel(allsum(mod.weight.grad), ref.weight.grad)
            if bias:
                res[f"disco{n}/db"] = rel(allsum(mod.bias.grad), ref.bias.grad)
            if w > 1 and cout == 1:
                try:
                    mod(shard(x[:1], mod.lat_in_shapes, mod.lon_in_shapes).float())
                    res[f"disco{n}/few_rows"] = 1.0
                except ValueError:
                    res[f"disco{n}/few_rows"] = 0.0
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", [(2, 1), (1, 2), (2, 2), (4, 2)])
def test_distributed_transpose_matches_serial_oracle(h, w):
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
        assert len(res) == 4 * len(CASES) - 1 + (w > 1), sorted(res)
        for k, v in res.items():
            assert v <= 2e-6, (rank, k, v)     # the GEMMs run in fp32, as on one GPU


def test_grid_of_one_rank_is_refused():
    mbd.init(None, None)
    try:
        with pytest.raises(NotImplementedError, match="distributed DISCO.*DiscreteContinuousConvTransposeS2"):
            mbd.DistributedDiscreteContinuousConvTransposeS2(4, 4, (17, 32), (33, 64), (3, 3), basis_type="morlet", theta_cutoff=0.3)
    finally:
        mbd.finalize()

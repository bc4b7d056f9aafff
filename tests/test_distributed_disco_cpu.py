"""CPU tests of DistributedDiscreteContinuousConvS2 and DistributedResampleS2 (makani_b200/distributed/disco.py, resample.py):

* the window psi_hat of every polar rank: the windows of all ranks together are exactly the global psi_hat, each window is the minimal range of
  input rows and equals the dense global psi_hat restricted to it; the halo's send / receive lists agree between every pair of ranks;
* on gloo (world sizes 2 to 8): the halo exchange equals slicing the gathered tensor and its adjoint satisfies <Hx, y> = <x, H^T y>;
  the whole choreography of both modules with the per-rank stages on the oracle, against the SERIAL fp64 oracle: y, dx, dW and dbias of the
  convolution, the forward and input gradient of the resampling.
The CUDA stages are covered by tests/test_gpu_distributed_disco.py."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import makani_b200.distributed as mbd
from makani_b200 import disco as D
from makani_b200.distributed import disco as DD
from oracle import makani_disco_oracle as DO
from oracle import makani_resample_oracle as RO
from test_distributed_cpu import _free_port


class OracleDiscoLocalOps:
    """the window contraction and its adjoint on the oracle's dense fp64 psi_hat, restricted to this rank's output rows and input window"""

    def __init__(self, layer):
        w = layer.window
        psi, _ = DO.dense_psi(layer.kernel_shape, layer.basis_norm_mode, (layer.nlat_in, layer.nlon_in), (layer.nlat_out, layer.nlon_out),
                              layer.grid_in, layer.grid_out, layer.theta_cutoff)
        outside = psi[:, w.t0 : w.t1].clone()
        outside[:, :, w.lo : w.hi] = 0
        assert not outside.any(), "oracle psi_hat reaches outside the window"
        self.K, self.nt, self.nlon_out, self.nlon_in = layer.kernel_size, w.t1 - w.t0, layer.nlon_out, layer.nlon_in
        self.nwin = w.hi - w.lo
        self.psi = psi[:, w.t0 : w.t1, w.lo : w.hi].reshape(self.K * self.nt, -1)

    def contract(self, xwin):
        return DO.contraction(xwin.double().unsqueeze(1), self.psi, self.K, self.nt, self.nlon_out)[:, 0].float()

    def adjoint(self, dX):
        return DO.adjoint(dX.double().unsqueeze(1), self.psi, self.nwin, self.nlon_in)[:, 0].float()


class OracleResampleLocalOps:
    """the oracle's forward and (autograd) adjoint on whole spheres"""

    def __init__(self, layer):
        self.tab = RO.tables(layer.nlat_in, layer.nlon_in, layer.nlat_out, layer.nlon_out, layer.grid_in, layer.grid_out)
        self.in_shape = (layer.nlat_in, layer.nlon_in)

    def forward(self, x):
        return RO.resample(x.double(), self.tab).float()

    def adjoint(self, dy):
        with torch.enable_grad():   # called from inside a backward
            x = torch.zeros(dy.shape[0], *self.in_shape, dtype=torch.float64, requires_grad=True)
            return torch.autograd.grad(RO.resample(x, self.tab), x, dy.double())[0].float()


# ------------------------------------------------------------------------------------------------------------- windows
# (in_shape, out_shape, grid_in, grid_out, cutoff in input spacings): pscale 1 and 2, equiangular (pole rows) and Legendre-Gauss grids, odd sizes
WINDOW_GEOMS = [((17, 32), (17, 32), "equiangular", "equiangular", 6.0), ((33, 64), (17, 32), "equiangular", "legendre-gauss", 2.0),
                ((19, 30), (19, 30), "legendre-gauss", "legendre-gauss", 2.5), ((24, 48), (24, 24), "legendre-gauss", "equiangular", 4.0)]


def _psi(geom, norm="mean", kernel_shape=(3, 3)):
    ish, osh, gi, go, u = geom
    return D.get_psi(kernel_shape, "morlet", norm, ish, osh, gi, go, u * np.pi / (ish[0] - 1))


@pytest.mark.parametrize("norm", ["mean", "individual", "support"])
@pytest.mark.parametrize("geom", WINDOW_GEOMS)
def test_windows_partition_global_psi(geom, norm):
    psi = _psi(geom, norm)
    dense = D.psi_dense(psi)
    lat_out = D.psi_lat_out(psi)
    for h in (1, 2, 3, 4):
        shapes = mbd.compute_split_shapes(psi.nlat_out, h)
        wins = DD.disco_windows(psi, shapes)
        ker, t, col, val = [], [], [], []
        for win in wins:
            sub = win.psi
            assert (sub.nlat_out, sub.nlat_in, sub.nlon_in, sub.nlon_out) == (win.t1 - win.t0, win.hi - win.lo, psi.nlon_in, psi.nlon_out)
            ker.append(sub.ker)
            t.append(D.psi_lat_out(sub) + win.t0)
            col.append(sub.col + win.lo * psi.nlon_in)
            val.append(sub.val)
            # minimal: the first and the last row carry entries, and rows of the global psi_hat for these outputs stay inside
            sel = (lat_out >= win.t0) & (lat_out < win.t1)
            rows = psi.col[sel] // psi.nlon_in
            assert (win.lo, win.hi) == (rows.min(), rows.max() + 1)
            np.testing.assert_array_equal(D.psi_dense(sub), dense[:, win.t0 : win.t1, win.lo : win.hi])
        assert np.array_equal(np.concatenate(ker), psi.ker) and np.array_equal(np.concatenate(t), lat_out)
        assert np.array_equal(np.concatenate(col), psi.col) and np.array_equal(np.concatenate(val), psi.val)   # bit for bit, same order
        plans = [DD.halo_plan(wins, mbd.compute_split_shapes(psi.nlat_in, h), r) for r in range(h)]
        for r in range(h):
            assert sum(plans[r][1]) == wins[r].hi - wins[r].lo
            for p in range(h):
                a, b = plans[r][0][p]
                assert b - a == plans[p][1][r], (h, r, p)


def test_a_window_spans_two_ranks():
    """4 polar ranks at the CPU test sizes: some window takes rows from beyond its nearest neighbour (the gloo tests below run this case)"""
    psi = _psi(WINDOW_GEOMS[0])
    h = 4
    wins = DD.disco_windows(psi, mbd.compute_split_shapes(psi.nlat_out, h))
    off = np.concatenate([[0], np.cumsum(mbd.compute_split_shapes(psi.nlat_in, h))])
    owners = [sorted({int(np.searchsorted(off, i, side="right") - 1) for i in range(w.lo, w.hi)}) for w in wins]
    assert any(max(o) - r > 1 or r - min(o) > 1 for r, o in enumerate(owners)), owners


# ---------------------------------------------------------------------------------------------------------------- gloo
# (C_in, C_out, in_shape, out_shape, kernel_shape, groups, bias, grid_in, grid_out, norm, cutoff in input spacings)
DISCO_CASES = [(6, 4, (17, 32), (17, 32), (3, 3), 1, True, "equiangular", "equiangular", "mean", 6.0),
               (4, 6, (33, 64), (17, 32), (3, 3), 2, True, "equiangular", "legendre-gauss", "individual", 2.0),
               (3, 3, (19, 30), (19, 30), (2, 3), 3, False, "legendre-gauss", "legendre-gauss", "support", 2.5),
               (1, 2, (17, 32), (17, 32), (3, 3), 1, True, "equiangular", "equiangular", "mean", 3.0)]   # C_in = 1 < w: B*C rows are split
# (nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out): up with pole expansion, down, up between equiangular grids
RESAMPLE_CASES = [(12, 24, 25, 48, "legendre-gauss", "equiangular"), (25, 48, 12, 24, "equiangular", "legendre-gauss"),
                  (13, 24, 25, 48, "equiangular", "equiangular")]


def _worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
        w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
        ih, iw = rank // w, rank % w
        mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
        mbd.set_disco_local_ops(OracleDiscoLocalOps)
        mbd.set_resample_local_ops(OracleResampleLocalOps)
        res = {}

        def shard(t, hs, ws):
            return torch.split(torch.split(t, hs, dim=-2)[ih], ws, dim=-1)[iw].contiguous()

        def allsum(t):
            t = t.clone()
            dist.all_reduce(t)
            return t

        # halo exchange and its adjoint
        psi = _psi(WINDOW_GEOMS[0])
        lat_in, lat_out = mbd.compute_split_shapes(psi.nlat_in, h), mbd.compute_split_shapes(psi.nlat_out, h)
        wins = DD.disco_windows(psi, lat_out)
        send, recv = DD.halo_plan(wins, lat_in, ih)
        g = torch.Generator().manual_seed(5)
        xg = torch.randn(3, psi.nlat_in, 7, dtype=torch.float64, generator=g)
        xl = torch.split(xg, lat_in, dim=1)[ih].contiguous()
        hx = DD.halo_exchange(xl, send, recv, mbd.polar_group())
        res["halo"] = (hx - xg[:, wins[ih].lo : wins[ih].hi]).abs().max().item()
        y = torch.randn(hx.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(100 + rank))
        hty = DD.halo_adjoint(y, send, recv, xl.shape[1], mbd.polar_group())
        lhs, rhs = allsum(torch.tensor((hx * y).sum().item())), allsum(torch.tensor((xl * hty).sum().item()))
        res["halo_adjoint"] = abs(lhs - rhs).item() / (1e-300 + allsum(torch.tensor((hx.abs() * y.abs()).sum().item())).item())

        for n, (cin, cout, ish, osh, ks, G, bias, gi, go, norm, u) in enumerate(DISCO_CASES):
            kw = dict(basis_type="morlet", basis_norm_mode=norm, groups=G, grid_in=gi, grid_out=go, bias=bias, theta_cutoff=u * np.pi / (ish[0] - 1))
            torch.manual_seed(17)
            ref = DO.DiscreteContinuousConvS2(cin, cout, ish, osh, ks, **kw).double()
            mod = mbd.DistributedDiscreteContinuousConvS2(cin, cout, ish, osh, ks, **kw)
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

            if w > 1 and cin == 1:
                try:
                    mod(shard(x[:1], mod.lat_in_shapes, mod.lon_in_shapes).float())
                    res[f"disco{n}/few_rows"] = 1.0
                except ValueError:
                    res[f"disco{n}/few_rows"] = 0.0

        for n, (hi, wi, ho, wo, gi, go) in enumerate(RESAMPLE_CASES):
            ref = RO.ResampleS2(hi, wi, ho, wo, grid_in=gi, grid_out=go)
            mod = mbd.DistributedResampleS2(hi, wi, ho, wo, grid_in=gi, grid_out=go)
            assert mod.expand_poles == ref.expand_poles == (n == 0)
            x = torch.randn(3, 5, hi, wi)
            gy = torch.randn(3, 5, ho, wo)
            xs = x.clone().requires_grad_(True)
            ys = ref(xs)
            ys.backward(gy)
            xd = shard(x, mod.lat_in_shapes, mod.lon_in_shapes).requires_grad_(True)
            yd = mod(xd)
            yd.backward(shard(gy, mod.lat_out_shapes, mod.lon_out_shapes))
            res[f"resample{n}/y"] = (yd.detach() - shard(ys.detach(), mod.lat_out_shapes, mod.lon_out_shapes)).abs().max().item()
            res[f"resample{n}/dx"] = (xd.grad - shard(xs.grad, mod.lat_in_shapes, mod.lon_in_shapes)).abs().max().item()
            try:
                mod(shard(torch.randn(h * w - 1, hi, wi), mod.lat_in_shapes, mod.lon_in_shapes))
                res[f"resample{n}/few_planes"] = 1.0
            except ValueError:
                res[f"resample{n}/few_planes"] = 0.0
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", [(2, 1), (1, 2), (2, 2), (4, 2)])
def test_distributed_disco_and_resample_match_serial_oracle(h, w):
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
        assert len(res) == 2 + 4 * len(DISCO_CASES) - 1 + (w > 1) + 3 * len(RESAMPLE_CASES), sorted(res)
        for k, v in res.items():
            # the convolution runs its GEMMs in fp32, as the single-GPU module does
            bound = 2e-6 if k.startswith("disco") else (1e-12 if k.startswith("halo") else 1e-6)
            assert v <= bound, (rank, k, v)


def test_grid_of_one_rank_is_refused_and_shim_names():
    import importlib
    import sys

    import makani_b200.compat as compat

    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        compat.install_torch_harmonics_shim()
        thd = importlib.import_module("torch_harmonics.distributed")
        assert thd.DistributedDiscreteContinuousConvS2 is mbd.DistributedDiscreteContinuousConvS2
        assert thd.DistributedResampleS2 is mbd.DistributedResampleS2
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    mbd.init(None, None)
    try:
        with pytest.raises(NotImplementedError, match="distributed DISCO.*DiscreteContinuousConvS2"):
            mbd.DistributedDiscreteContinuousConvS2(4, 4, (17, 32), (17, 32), (3, 3), basis_type="morlet", theta_cutoff=0.3)
        with pytest.raises(NotImplementedError, match="distributed resampling.*ResampleS2"):
            mbd.DistributedResampleS2(24, 48, 49, 96, grid_in="legendre-gauss", grid_out="equiangular")
    finally:
        mbd.finalize()

"""gloo tests (CPU, world sizes 2 to 8) of DistributedRealVectorSHT / DistributedInverseRealVectorSHT: the all-to-all choreography on vector
fields and its autograd against the SERIAL fp64 vector oracle (oracle/makani_vector_oracle.py).  The local stages are the oracle's arithmetic
on this rank's shard (the order slice of its D / Q tables); the CUDA stages are covered by tests/test_gpu_distributed_vector.py."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import makani_b200.distributed as mbd
from oracle import makani_oracle as O
from oracle import makani_vector_oracle as V
from test_distributed_cpu import OracleLocalOps, _free_port


class OracleVectorLocalOps(OracleLocalOps):
    """the scalar stand-in's fft / ifft on component rows, plus the vector Legendre stages on orders [m_offset, m_offset + mmax_local)"""

    def __init__(self, t):
        super().__init__(t)
        theta, _ = O.precompute_latitudes(t.nlat, t.grid)
        D, Q = V.vector_legpoly(t.mmax, t.lmax, theta, csphase=t.csphase)
        sl = slice(t.m_offset, t.m_offset + t.mmax_local)
        self.D, self.Q = torch.from_numpy(D[sl]).to(torch.complex128), torch.from_numpy(Q[sl]).to(torch.complex128)
        l = torch.arange(t.lmax, dtype=torch.float64)
        self.f = torch.where(l > 0, 1.0 / (l * (l + 1.0)).clamp_min(1.0), torch.zeros_like(l)).to(torch.complex128)[:, None]

    def ifft(self, xc, dtype):
        z = xc.to(torch.complex128).clone()
        z[..., 0] = z[..., 0].real
        if self.t.mmax > self.t.nlon // 2 and self.t.nlon % 2 == 0:
            z[..., self.t.nlon // 2] = z[..., self.t.nlon // 2].real
        return torch.fft.irfft(z, n=self.t.nlon, dim=-1, norm="forward")

    def vlegendre(self, xc):
        c = lambda a, t: torch.einsum("...km,mlk->...lm", a, t)
        xt, xp = xc[:, :, 0].to(torch.complex128), xc[:, :, 1].to(torch.complex128)
        S = (c(xt, self.D) - 1j * c(xp, self.Q)) * self.f
        T = (-1j * c(xt, self.Q) - c(xp, self.D)) * self.f
        return torch.stack([S, T], dim=2)

    def ivlegendre(self, xc):
        e = lambda a, t: torch.einsum("...lm,mlk->...km", a, t)
        s, t = xc[:, :, 0].to(torch.complex128), xc[:, :, 1].to(torch.complex128)
        return torch.stack([e(s, self.D) + 1j * e(t, self.Q), 1j * e(s, self.Q) - e(t, self.D)], dim=2)


# (grid, nlat, nlon, lmax, mmax): odd nlat, so every latitude (and, at the defaults, degree) split is uneven
CASES = [("equiangular", 33, 64, None, None), ("legendre-gauss", 33, 64, None, None), ("equiangular", 33, 64, 19, 21),
         ("legendre-gauss", 33, 64, 19, 21)]
# 5-D with 5 vector channels (divisible by neither group size), and the (B, E, C, 2, H, W) shape of VortDivCRPSLoss
LEADS = [(2, 5), (2, 3, 3)]


def _worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
        w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
        ih, iw = rank // w, rank % w
        mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
        mbd.set_local_ops(OracleVectorLocalOps)
        torch.manual_seed(333)
        results = {}

        def shard(t, hs, ws):
            t = torch.split(t, hs, dim=-2)[ih]
            return torch.split(t, ws, dim=-1)[iw].contiguous()

        for grid, nlat, nlon, lmax, mmax in CASES:
            dv = mbd.DistributedRealVectorSHT(nlat, nlon, lmax=lmax, mmax=mmax, grid=grid)
            div = mbd.DistributedInverseRealVectorSHT(nlat=nlat, nlon=nlon, lmax=lmax, mmax=mmax, grid=grid)
            assert dv.lat_shapes == O.compute_split_shapes(nlat, h) and dv.m_shapes == O.compute_split_shapes(dv.mmax, w)
            ov = V.RealVectorSHT(nlat, nlon, lmax, mmax, grid, dtype=torch.float64)
            oiv = V.InverseRealVectorSHT(nlat, nlon, lmax, mmax, grid, dtype=torch.float64)
            L, M = dv.lmax, dv.mmax
            for lead in LEADS:
                tag = f"{grid}/{nlat}x{nlon}/L{L}M{M}/{len(lead) + 3}d"
                x = torch.randn(*lead, 2, nlat, nlon, dtype=torch.float64)
                gc = torch.randn(*lead, 2, L, M, dtype=torch.complex128)
                xl = shard(x, dv.lat_shapes, dv.lon_shapes).requires_grad_(True)
                cl = dv(xl)
                assert cl.shape == (*lead, 2, dv.lmax_local, dv.mmax_local), (tag, cl.shape)
                xs = x.clone().requires_grad_(True)
                cs = ov(xs)
                results[f"{tag}/vsht"] = (cl - shard(cs, dv.l_shapes, dv.m_shapes)).abs().max().item()
                cl.backward(shard(gc, dv.l_shapes, dv.m_shapes))
                cs.backward(gc)
                results[f"{tag}/vsht_grad"] = (xl.grad - shard(xs.grad, dv.lat_shapes, dv.lon_shapes)).abs().max().item()

                c = torch.randn(*lead, 2, L, M, dtype=torch.complex128)
                gy = torch.randn(*lead, 2, nlat, nlon, dtype=torch.float64)
                cl = shard(c, div.l_shapes, div.m_shapes).requires_grad_(True)
                yl = div(cl, dtype=torch.float64)
                assert yl.shape == (*lead, 2, div.nlat_local, div.nlon_local), (tag, yl.shape)
                cs = c.clone().requires_grad_(True)
                ys = oiv(cs)
                results[f"{tag}/ivsht"] = (yl - shard(ys, div.lat_shapes, div.lon_shapes)).abs().max().item()
                yl.backward(shard(gy, div.lat_shapes, div.lon_shapes))
                ys.backward(gy)
                results[f"{tag}/ivsht_grad"] = (cl.grad - shard(cs.grad, div.l_shapes, div.m_shapes)).abs().max().item()
        q.put((rank, results, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", [(2, 1), (1, 2), (2, 2), (4, 2)])
def test_distributed_vector_sht_matches_serial_oracle(h, w):
    world = h * w
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, h, w, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in out:
        assert err is None, f"rank {rank}:\n{err}"
        assert len(res) == 4 * len(CASES) * len(LEADS)
        for k, v in res.items():
            assert v < 1e-9, (rank, k, v)


def test_oracle_vector_local_ops_world1_equals_oracle():
    """world size 1: the stand-in's stages compose to the oracle's vector transforms (so the gloo test pins the choreography alone)"""
    torch.manual_seed(333)
    mbd.set_local_ops(OracleVectorLocalOps)
    try:
        nlat, nlon = 17, 32
        x = torch.randn(2, 3, 2, nlat, nlon, dtype=torch.float64)
        c = mbd.DistributedRealVectorSHT(nlat, nlon)(x)
        assert (c - V.RealVectorSHT(nlat, nlon, dtype=torch.float64)(x)).abs().max().item() < 1e-12
        y = mbd.DistributedInverseRealVectorSHT(nlat, nlon)(c, dtype=torch.float64)
        assert (y - V.InverseRealVectorSHT(nlat, nlon, dtype=torch.float64)(c)).abs().max().item() < 1e-12
    finally:
        mbd.set_local_ops(None)


def test_vector_modules_shapes_and_shim_surface():
    import makani_b200.compat as compat

    compat.install_torch_harmonics_shim()
    import torch_harmonics.distributed as thd

    assert thd.DistributedRealVectorSHT is mbd.DistributedRealVectorSHT
    assert thd.DistributedInverseRealVectorSHT is mbd.DistributedInverseRealVectorSHT
    # the keyword call of makani/utils/losses/base_loss.py (VortDivBaseLoss, GradientBaseLoss)
    v = thd.DistributedRealVectorSHT(721, 1440, lmax=None, mmax=None, grid="equiangular")
    iv = thd.DistributedInverseRealVectorSHT(nlat=v.nlat, nlon=v.nlon, lmax=None, mmax=None, grid="equiangular")
    assert (v.lmax, v.mmax, iv.lmax, iv.mmax) == (721, 721, 721, 721)
    assert v.l_shapes == [721] and iv.lat_shapes == [721] and iv.m_shapes == [721]
    with pytest.raises(ValueError):
        v(torch.zeros(1, 3, 721, 1440))   # no component axis of size 2
    with pytest.raises(ValueError):
        iv(torch.zeros(1, 2, 721, 720, dtype=torch.complex64))

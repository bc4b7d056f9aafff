"""CPU tests of DistributedNeighborhoodAttentionS2 (makani_b200/distributed/attention.py):

* the windows of the neighbourhood (a K = 1 DiscoPsi) over every polar split the gloo runs use: together they are exactly the global
  neighbourhood (same entries, same (i, j) order, input rows re-indexed), each window's [lo, hi) is minimal, and the halo's send / receive
  lists agree between every pair of ranks;
* on gloo (2 x 1, 1 x 2, 2 x 2, 4 x 2): the whole choreography with the per-rank stage on the fp64 oracle (tests/attention_oracle.py) against
  the SERIAL fp64 oracle module: the output, the gradients of query, key and value, and every parameter gradient summed over the ranks, on the
  same grid (both grid types), 2:1 longitude downsampling from equiangular to Legendre-Gauss, a cutoff whose pole rows span whole rings, key
  and value defaulting to query, E_k != E_v, and B = 1 with 2 heads (at w = 2 the split is by heads); the refusals of B * heads < w and of a
  wrong local shape;
* a grid of one rank is refused, and torch_harmonics.distributed names the class.
The CUDA stage is covered by tests/test_gpu_distributed_attention.py."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import attention_oracle as AO
import makani_b200.distributed as mbd
from makani_b200 import attention as A
from makani_b200.distributed import disco as DD
from makani_b200.quadrature import _grid_np
from test_distributed_cpu import _free_port


class OracleAttentionLocalOps:
    """the window attention and its gradients on the fp64 oracle, over this rank's window of the neighbourhood"""

    def __init__(self, layer):
        w = layer.window
        self.psi = w.psi
        self.omega = np.zeros(w.hi - w.lo)
        self.omega[w.psi.col // w.psi.nlon_in] = w.psi.val

    def _attend(self, q, k, v, heads, scale):
        p = self.psi
        return AO.attention(q, k, v, p.row_ptr, p.col, self.omega, p.nlon_in, p.nlon_out, heads, scale)

    def forward_attention(self, q, k, v, heads, scale):
        y, lse = self._attend(q.double(), k.double(), v.double(), heads, scale)
        return y.float(), lse.float()

    def backward_attention(self, q, k, v, y, lse, dy, heads, scale):
        with torch.enable_grad():   # called from inside a backward
            qd, kd, vd = (x.double().requires_grad_(True) for x in (q, k, v))
            yd, _ = self._attend(qd, kd, vd, heads, scale)
            return tuple(g.float() for g in torch.autograd.grad(yd, (qd, kd, vd), dy.double()))


def _cutoff(ish, units):
    return units * np.pi / (ish[0] - 1)


# (in_channels, in_shape, out_shape, grid_in, grid_out, heads, k_channels, out_channels, bias, cutoff in input spacings, separate key / value, B)
CASES = [
    (6, (17, 32), (17, 32), "equiangular", "equiangular", 2, None, None, True, 2.5, True, 2),              # same grid, equiangular
    (4, (16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 2, 8, 6, True, 2.0, True, 2),              # same grid, Legendre-Gauss, E_k 4, E_v 3
    (4, (33, 64), (17, 32), "equiangular", "legendre-gauss", 2, None, None, True, 3.0, True, 2),           # 2:1 downsampling, lat_in != lat_out splits
    (4, (17, 32), (17, 32), "equiangular", "equiangular", 1, None, 6, False, 5.0, False, 2),               # whole-ring pole rows, k / v = query
    (4, (16, 32), (16, 32), "legendre-gauss", "legendre-gauss", 2, None, None, True, 2.0, False, 1),       # B = 1, 2 heads: at w = 2 split by heads
]
GRIDS = [(2, 1), (1, 2), (2, 2), (4, 2)]


def _key(case):
    ish, osh, gi, go, units = case[1], case[2], case[3], case[4], case[9]
    return (tuple(ish), tuple(osh), gi, go, float(_cutoff(ish, units)))


@pytest.mark.parametrize("case", CASES, ids=[f"case{n}" for n in range(len(CASES))])
def test_windows_partition_the_neighbourhood(case):
    nb = A.get_neighbourhood(*_key(case))
    counts = np.diff(nb.row_ptr)
    t_of = np.repeat(np.arange(nb.nlat_out), counts)
    for h in sorted({h for h, _ in GRIDS} | {1, 3}):
        wins = DD.disco_windows(nb, mbd.compute_split_shapes(nb.nlat_out, h))
        t, col, val, ker = [], [], [], []
        for win in wins:
            sub = win.psi
            assert (sub.nlat_out, sub.nlat_in, sub.nlon_in, sub.nlon_out, sub.kernel_size) == (win.t1 - win.t0, win.hi - win.lo, nb.nlon_in,
                                                                                              nb.nlon_out, 1)
            t.append(np.repeat(np.arange(sub.nlat_out), np.diff(sub.row_ptr)) + win.t0)
            col.append(sub.col + win.lo * nb.nlon_in)
            val.append(sub.val)
            ker.append(sub.ker)
            rows = nb.col[(t_of >= win.t0) & (t_of < win.t1)] // nb.nlon_in
            assert (win.lo, win.hi) == (rows.min(), rows.max() + 1), (h, win.t0)          # minimal: both end rows carry entries
            assert sub.col.min() >= 0 and sub.col.max() < (win.hi - win.lo) * nb.nlon_in
        assert np.array_equal(np.concatenate(t), t_of)
        assert np.array_equal(np.concatenate(col), nb.col) and np.array_equal(np.concatenate(val), nb.val)   # bit for bit, same order
        assert not np.concatenate(ker).any()
        plans = [DD.halo_plan(wins, mbd.compute_split_shapes(nb.nlat_in, h), r) for r in range(h)]
        for r in range(h):
            assert sum(plans[r][1]) == wins[r].hi - wins[r].lo
            for p in range(h):
                a, b = plans[r][0][p]
                assert b - a == plans[p][1][r], (h, r, p)
    if case[9] == 5.0:   # the whole-ring case: rows of the neighbourhood near the poles are whole rings of input points
        i = nb.col // nb.nlon_in
        whole = [t for t in range(nb.nlat_out) if np.bincount(i[nb.row_ptr[t] : nb.row_ptr[t + 1]]).max() == nb.nlon_in]
        assert 0 in whole and nb.nlat_out - 1 in whole and len(whole) > 2, whole


def _worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
        w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
        ih, iw = rank // w, rank % w
        mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
        mbd.set_attention_local_ops(OracleAttentionLocalOps)
        res = {}

        def shard(t, hs, ws):
            return torch.split(torch.split(t, hs, dim=-2)[ih], ws, dim=-1)[iw].contiguous()

        def allsum(t):
            t = t.clone()
            dist.all_reduce(t)
            return t

        rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
        for n, case in enumerate(CASES):
            cin, ish, osh, gi, go, H, ck, cv, bias, units, separate, B = case
            kw = dict(grid_in=gi, grid_out=go, num_heads=H, bias=bias, theta_cutoff=_cutoff(ish, units), k_channels=ck, out_channels=cv)
            torch.manual_seed(17)
            mod = mbd.DistributedNeighborhoodAttentionS2(cin, ish, osh, **kw)
            torch.manual_seed(17)
            serial = A.NeighborhoodAttentionS2(cin, ish, osh, **kw)
            sd = serial.state_dict()
            res[f"attn{n}/same_parameters"] = float(mod.state_dict().keys() != sd.keys() or
                                                    any(not torch.equal(v, sd[k]) for k, v in mod.state_dict().items()))
            res[f"attn{n}/tags"] = float(any(p.is_shared_mp != ["spatial"] or p.sharded_dims_mp != [None] * p.dim() for p in mod.parameters()))
            if bias:
                with torch.no_grad():
                    g = torch.Generator().manual_seed(3)
                    for name in ("q_bias", "k_bias", "v_bias", "proj_bias"):
                        getattr(mod, name).copy_(torch.randn(getattr(mod, name).shape, generator=g))
            params = {k: p.detach().double().requires_grad_(True) for k, p in mod.named_parameters()}
            g = torch.Generator().manual_seed(100 + n)
            query = torch.randn(B, cin, *osh, dtype=torch.float64, generator=g)
            key = torch.randn(B, cin, *ish, dtype=torch.float64, generator=g) if separate else query
            value = torch.randn(B, cin, *ish, dtype=torch.float64, generator=g) if separate else query
            gy = torch.randn(B, mod.out_channels, *osh, dtype=torch.float64, generator=g)

            refs = [x.clone().requires_grad_(True) for x in ((query, key, value) if separate else (query,))]
            nb = A.get_neighbourhood(*mod._key)
            omega = 2.0 * np.pi * _grid_np(ish[0], gi)[1] / ish[1]
            ref = AO.module_forward(params, *(refs if separate else refs * 3), nb.row_ptr, nb.col, omega, H, mod.scale)
            ref.backward(gy)

            ins = [shard(query, mod.lat_out_shapes, mod.lon_out_shapes).float().requires_grad_(True)]
            if separate:
                ins += [shard(x, mod.lat_in_shapes, mod.lon_in_shapes).float().requires_grad_(True) for x in (key, value)]
            out = mod(*ins)
            assert out.shape == (B, mod.out_channels, mod.nlat_out_local, mod.nlon_out_local) and out.dtype == torch.float32
            out.backward(shard(gy, mod.lat_out_shapes, mod.lon_out_shapes).float())
            res[f"attn{n}/out"] = rel(out.detach(), shard(ref.detach(), mod.lat_out_shapes, mod.lon_out_shapes))
            for what, a, b in zip(("dquery", "dkey", "dvalue"), ins, refs):
                shapes = (mod.lat_out_shapes, mod.lon_out_shapes) if what == "dquery" else (mod.lat_in_shapes, mod.lon_in_shapes)
                res[f"attn{n}/{what}"] = rel(a.grad, shard(b.grad, *shapes))
            for name, p in mod.named_parameters():
                if name == "k_bias":
                    # exactly zero (the softmax is invariant to a key bias): both sides are rounding noise, so hold the summed gradient to the
                    # bound of the key weights' gradient, as the serial module's test does
                    res[f"attn{n}/d{name}"] = allsum(p.grad).abs().max().item() / params["k_weights"].grad.abs().max().item()
                else:
                    res[f"attn{n}/d{name}"] = rel(allsum(p.grad), params[name].grad)

            # refusals: a wrong local shape, and fewer (b, h) pairs than azimuth ranks
            try:
                mod(query.float())
                res[f"attn{n}/wrong_shape"] = 1.0
            except ValueError:
                res[f"attn{n}/wrong_shape"] = 0.0
            if w > 1 and H == 1:
                try:
                    mod(shard(query[:1], mod.lat_out_shapes, mod.lon_out_shapes).float())
                    res[f"attn{n}/few_pairs"] = 1.0
                except ValueError:
                    res[f"attn{n}/few_pairs"] = 0.0
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", GRIDS)
def test_distributed_attention_matches_serial_oracle(h, w):
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
        for n, case in enumerate(CASES):
            want = {"same_parameters", "tags", "out", "dquery", "wrong_shape", "dq_weights", "dk_weights", "dv_weights", "dproj_weights"}
            want |= {"dkey", "dvalue"} if case[10] else set()
            want |= {"dq_bias", "dk_bias", "dv_bias", "dproj_bias"} if case[8] else set()
            want |= {"few_pairs"} if w > 1 and case[5] == 1 else set()
            assert {k.split("/")[1] for k in res if k.startswith(f"attn{n}/")} == want, (n, sorted(res))
        for k, v in res.items():
            # the projections run in fp32, as the single-GPU module does; the attention in fp64 on the oracle
            assert v <= 1e-5, (rank, k, v)


def test_grid_of_one_rank_is_refused_and_shim_name():
    import importlib
    import sys

    import makani_b200.compat as compat

    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        compat.install_torch_harmonics_shim()
        thd = importlib.import_module("torch_harmonics.distributed")
        assert thd.DistributedNeighborhoodAttentionS2 is mbd.DistributedNeighborhoodAttentionS2
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    mbd.init(None, None)
    try:
        with pytest.raises(NotImplementedError, match="distributed neighbourhood attention.*NeighborhoodAttentionS2"):
            mbd.DistributedNeighborhoodAttentionS2(4, (17, 32), (17, 32), num_heads=2, theta_cutoff=0.3)
    finally:
        mbd.finalize()

"""CPU tests of DistributedAttentionS2 (makani_b200/distributed/attention.py):

* on gloo (2 x 1, 1 x 2, 2 x 2, 4 x 2 and an uneven 3 x 2): the whole choreography with the per-rank stage on the fp64 oracle
  (tests/attention_global_oracle.py) against the SERIAL fp64 oracle module: the output, the gradients of query, key and value, and every
  parameter gradient summed over the ranks, on the same grid (equiangular and Legendre-Gauss), in_shape != out_shape, odd nlat / nlon with
  uneven splits, key and value defaulting to query, E_k != E_v, and B = 1 with one head;
* the global-order gather (uneven shards padded for gloo's all_gather) reproduces the global tensor exactly;
* state-dict and seed parity with AttentionS2, the parameter tags, and the refusals: a wrong local shape, a dtype the kernels do not take,
  dropout in training, an empty shard and a grid of one rank;
* torch_harmonics.distributed names the class, and the three separable backward entry points are in the header, the signature table and
  the built library.
The CUDA stage is covered by tests/test_gpu_distributed_attention_global.py."""
import os
import re

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import attention_global_oracle as GO
import makani_b200.distributed as mbd
from makani_b200 import _lib
from makani_b200 import attention as A
from test_distributed_cpu import _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class OracleGlobalAttentionLocalOps:
    """the per-rank stage in fp64: the forward on the oracle, the backward passes from their formulas with the given lse and D"""

    def __init__(self, layer):
        pass

    def forward(self, q, k, v, bias, scale, precision):
        o, lse = GO.attention(q.double(), k.double(), v.double(), bias.double(), scale)
        return o.float(), lse.float()

    def rowdot(self, o, do):
        return (o.double() * do.double()).sum(-1).float()

    @staticmethod
    def _ds(q, k, v, bias, lse, D, do, scale):
        q, k, v, b, lse, D, do = (t.double() for t in (q, k, v, bias, lse, D, do))
        p = torch.exp(scale * q @ k.transpose(-1, -2) + b - lse[..., None])
        return p, p * (do @ v - D[..., None])

    def backward_q(self, q, k, v, bias, lse, D, do, scale, precision):
        _, ds = self._ds(q, k, v, bias, lse, D, do, scale)
        return (scale * ds @ k.double()).float()

    def backward_kv(self, q, k, v, bias, lse, D, do, scale, precision):
        p, ds = self._ds(q, k, v, bias, lse, D, do, scale)
        return (scale * ds.transpose(-1, -2) @ q.double()).float(), (do.double().transpose(-1, -2) @ p).float()


# (in_channels, in_shape, out_shape, grid_in, grid_out, heads, k_channels, out_channels, bias, separate key / value, B)
CASES = [
    (16, (9, 16), (9, 16), "equiangular", "equiangular", 2, None, None, True, True, 2),             # same grid, equiangular
    (16, (8, 16), (8, 16), "legendre-gauss", "legendre-gauss", 2, None, None, True, True, 2),       # same grid, Legendre-Gauss
    (16, (13, 24), (7, 12), "equiangular", "legendre-gauss", 2, None, None, True, True, 2),         # in_shape != out_shape
    (8, (11, 15), (11, 15), "legendre-gauss", "legendre-gauss", 2, 32, 16, False, False, 2),        # odd grid, k / v = query, E_k 16, E_v 8
    (8, (9, 16), (9, 16), "equiangular", "equiangular", 1, None, None, True, True, 1),              # B = 1, one head
]
GRIDS = [(2, 1), (1, 2), (2, 2), (4, 2), (3, 2)]


def _worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
        w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
        ih, iw = rank // w, rank % w
        mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
        mbd.set_global_attention_local_ops(OracleGlobalAttentionLocalOps)
        res = {}

        def shard(t, hs, ws):
            return torch.split(torch.split(t, hs, dim=-2)[ih], ws, dim=-1)[iw].contiguous()

        def allsum(t):
            t = t.clone()
            dist.all_reduce(t)
            return t

        rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
        for n, case in enumerate(CASES):
            cin, ish, osh, gi, go, H, ck, cv, bias, separate, B = case
            kw = dict(grid_in=gi, grid_out=go, bias=bias, k_channels=ck, out_channels=cv)
            torch.manual_seed(17)
            mod = mbd.DistributedAttentionS2(cin, H, ish, osh, **kw)
            torch.manual_seed(17)
            serial = A.AttentionS2(cin, H, ish, osh, **kw)
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
            ref = GO.module_forward(params, *(refs if separate else refs * 3), gi, H, mod.scale)
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

            # the global-order gathers reproduce the global tensors exactly, from uneven shards
            E = 3
            gk = torch.arange(B * H * ish[0] * ish[1] * E, dtype=torch.float32).view(B, H, *ish, E)
            gv = -torch.arange(B * H * E * ish[0] * ish[1], dtype=torch.float32).view(B, H, E, *ish)
            kr = shard(gk.movedim(4, 2), mod.lat_in_shapes, mod.lon_in_shapes).movedim(2, 4).reshape(B, H, -1, E)
            vr = shard(gv, mod.lat_in_shapes, mod.lon_in_shapes).reshape(B, H, E, -1)
            K, V = mod._gather_keys(kr, vr)
            res[f"attn{n}/gather_keys"] = float(not (torch.equal(K, gk.reshape(B, H, -1, E)) and torch.equal(V, gv.reshape(B, H, E, -1))))
            gq = torch.arange(B * H * osh[0] * osh[1], dtype=torch.float32).view(B, H, *osh)
            res[f"attn{n}/gather_out"] = float(not torch.equal(mod._gather_out(shard(gq, mod.lat_out_shapes, mod.lon_out_shapes).reshape(B, H, -1), 2),
                                                               gq.reshape(B, H, -1)))

            # refusals: a wrong local shape, a dtype the kernels do not take, dropout in training
            for what, fn, exc in (("wrong_shape", lambda: mod(query.float()), ValueError),
                                  ("wrong_dtype", lambda: mod(*(x.detach().double() for x in ins)), TypeError)):
                try:
                    fn()
                    res[f"attn{n}/{what}"] = 1.0
                except exc:
                    res[f"attn{n}/{what}"] = 0.0
        drop = mbd.DistributedAttentionS2(8, 1, (9, 16), (9, 16), drop_rate=0.1)
        x = shard(torch.zeros(1, 8, 9, 16), drop.lat_out_shapes, drop.lon_out_shapes)
        try:
            drop(x)
            res["drop_rate"] = 1.0
        except NotImplementedError:
            res["drop_rate"] = 0.0
        drop.eval()
        res["drop_rate_eval"] = float(drop(x).shape != (1, 8, drop.nlat_out_local, drop.nlon_out_local))
        try:
            mbd.DistributedAttentionS2(8, 1, (1, 1), (1, 1), grid_in="legendre-gauss", grid_out="legendre-gauss")
            res["empty_shard"] = 1.0
        except ValueError as e:
            res["empty_shard"] = float("too small" not in str(e))
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", GRIDS)
def test_distributed_global_attention_matches_serial_oracle(h, w):
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
            want = {"same_parameters", "tags", "out", "dquery", "wrong_shape", "wrong_dtype", "gather_keys", "gather_out", "dq_weights",
                    "dk_weights", "dv_weights", "dproj_weights"}
            want |= {"dkey", "dvalue"} if case[9] else set()
            want |= {"dq_bias", "dk_bias", "dv_bias", "dproj_bias"} if case[8] else set()
            assert {k.split("/")[1] for k in res if k.startswith(f"attn{n}/")} == want, (n, sorted(res))
        assert {"drop_rate", "drop_rate_eval", "empty_shard"} <= set(res)
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
        assert thd.DistributedAttentionS2 is mbd.DistributedAttentionS2
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)
    mbd.init(None, None)
    try:
        with pytest.raises(NotImplementedError, match="distributed global attention.*AttentionS2"):
            mbd.DistributedAttentionS2(8, 1, (9, 16), (9, 16))
    finally:
        mbd.finalize()


def test_separable_backward_symbols():
    names = ["b200sht_attention_global_rowdot", "b200sht_attention_global_backward_kv", "b200sht_attention_global_backward_q"]
    header = open(os.path.join(ROOT, "include", "b200sht.h")).read()
    for n in names:
        assert re.search(r"\b" + n + r"\(", header), n
        assert n in _lib._SIGNATURES
    assert "also serves b200sht_attention_global_backward_kv and _backward_q" in header
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200sht.so is not built")
    lib = _lib.load()
    for n in names:
        assert hasattr(lib, n)

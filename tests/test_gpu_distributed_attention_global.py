"""DistributedAttentionS2 on an H100:

* the separable backward of the C ABI on the full grid: rowdot, the kv pass and the q pass give dq, dk and dv bit for bit equal to
  b200sht_attention_global_backward, in TF32 and 3 x TF32;
* virtual ranks on one GPU (h x w in {2 x 1, 1 x 2, 2 x 2, 4 x 2}) at 181 x 360 equiangular, 91 x 180 Legendre-Gauss <- 181 x 360
  equiangular and a small odd grid with dropped keys at d = 8, d = 128 and (dqk, dv) = (96, 72): every rank's o, lse, D, dq (its
  queries against every key) and dk, dv (its keys against every query),computed by the module's per-rank stage, are torch.equal to the matching slices of the serial
  kernels' outputs on the same operands, in both precisions; two runs are bit-identical, and the per-rank calls launch the same
  attention_global_kernel instantiations as the serial call;
* the module itself on gloo process groups whose ranks share the GPU: every rank's output and input gradients, and the rank-summed
  parameter gradients, against the single-GPU AttentionS2 (relative L2 1e-5 with TF32 off, 2e-3 with TF32 on: the cuBLAS projections at a
  different N may round differently), and bf16 inputs."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import attention_global_oracle as GO  # noqa: E402
import makani_b200.distributed as mbd  # noqa: E402
from makani_b200 import _lib  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.distributed import attention as DA  # noqa: E402
from test_distributed_cpu import _free_port  # noqa: E402
from test_gpu_engine import launched_kernels  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
PRECS = [_lib.PREC_TF32, _lib.PREC_FP32X3]
PREC_IDS = ["tf32", "fp32x3"]


def _operands(B, H, nq, nk, dqk, dv, bias, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, H, nq, dqk, device=DEV, generator=g)
    k = torch.randn(B, H, nk, dqk, device=DEV, generator=g)
    v = torch.randn(B, H, dv, nk, device=DEV, generator=g)
    do = torch.randn(B, H, nq, dv, device=DEV, generator=g)
    return q, k, v, do, bias.to(DEV)


def _masked_bias(nk, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    b = torch.log(torch.rand(nk, device=DEV, generator=g) * 0.01 + 1e-4)
    b[: min(40, nk - 1)] = -torch.inf
    b[45::7] = -torch.inf
    return b


@pytest.mark.parametrize("prec", PRECS, ids=PREC_IDS)
@pytest.mark.parametrize("size", [(2, 2, 700, 1100, 64, 64), (1, 3, 130, 97, 8, 128), (1, 1, 1, 5, 40, 8),
                                  (2, 1, 150, 301, 88, 72)], ids=lambda s: "x".join(map(str, s)))
def test_split_backward_equals_the_full_backward(size, prec):
    B, H, nq, nk, dqk, dv = size
    q, k, v, do, bias = _operands(B, H, nq, nk, dqk, dv, _masked_bias(nk, 1), seed=nq + nk)
    o, lse = A.global_attention_forward(q, k, v, bias, 0.2, prec)
    dq, dk, dvt = A.global_attention_backward(q, k, v, bias, o, lse, do, 0.2, prec)
    D = A.global_attention_rowdot(o, do)
    dk2, dv2 = A.global_attention_backward_kv(q, k, v, bias, lse, D, do, 0.2, prec)
    dq2 = A.global_attention_backward_q(q, k, v, bias, lse, D, do, 0.2, prec)
    torch.cuda.synchronize()
    assert torch.allclose(D.double(), (o.double() * do.double()).sum(-1), rtol=1e-5, atol=1e-5)
    assert torch.equal(dq, dq2) and torch.equal(dk, dk2) and torch.equal(dvt, dv2)


def _blocks(nlat, nlon, h, w):
    """the point indices (row-major over the global grid) of every rank's (lat, lon) block, rank = ih * w + iw"""
    lat, lon = mbd.compute_split_shapes(nlat, h), mbd.compute_split_shapes(nlon, w)
    la, lo = np.cumsum([0] + lat), np.cumsum([0] + lon)
    out = []
    for ih in range(h):
        for iw in range(w):
            rows, cols = np.arange(la[ih], la[ih + 1]), np.arange(lo[iw], lo[iw + 1])
            out.append(torch.from_numpy((rows[:, None] * nlon + cols[None, :]).reshape(-1)).to(DEV))
    return out


def _per_rank(ops, q, k, v, do, bias, lse, D, qi, ki, prec):
    """the per-rank stage of DistributedAttentionS2 on rank blocks qi (output points) and ki (input points): o, lse, D, dq of its queries
    against every key; dk, dv of its keys against every query (the gathered Q, dO, lse, D)"""
    c = lambda t: t.contiguous()   # noqa: E731
    qr, dor = c(q[:, :, qi]), c(do[:, :, qi])
    o_r, lse_r = ops.forward(qr, k, v, bias, 0.2, prec)
    D_r = ops.rowdot(o_r, dor)
    dq_r = ops.backward_q(qr, k, v, bias, lse_r, D_r, dor, 0.2, prec)
    dk_r, dv_r = ops.backward_kv(q, c(k[:, :, ki]), c(v[..., ki]), c(bias[ki]), lse, D, do, 0.2, prec)
    return o_r, lse_r, D_r, dq_r, dk_r, dv_r


# (out grid, in grid, B, H, dqk, dv, bias): 181 x 360 equiangular, 91 x 180 Legendre-Gauss <- 181 x 360 equiangular, an odd grid with
# dropped keys at d = 8, d = 128 and dqk, dv = 96, 72 (three head-dim chunks)
GEOMS = [((181, 360), (181, 360), 1, 2, 32, 32, "equiangular"), ((91, 180), (181, 360), 1, 2, 64, 64, "equiangular"),
         ((13, 27), (15, 29), 2, 2, 8, 8, "masked"), ((13, 27), (15, 29), 1, 2, 128, 128, "masked"),
         ((13, 27), (15, 29), 2, 1, 96, 72, "masked")]
GRIDS = [(2, 1), (1, 2), (2, 2), (4, 2)]


@pytest.mark.parametrize("prec", PRECS, ids=PREC_IDS)
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: f"{g[0][0]}x{g[0][1]}<-{g[1][0]}x{g[1][1]}-d{g[4]}")
def test_virtual_ranks_equal_the_serial_kernels(geom, prec):
    osh, ish, B, H, dqk, dv, kind = geom
    nq, nk = osh[0] * osh[1], ish[0] * ish[1]
    bias = _masked_bias(nk, 2) if kind == "masked" else GO.key_bias(*ish, kind).float()
    q, k, v, do, bias = _operands(B, H, nq, nk, dqk, dv, bias, seed=nq)
    ops = DA.CudaGlobalAttentionLocalOps(None)
    o, lse = A.global_attention_forward(q, k, v, bias, 0.2, prec)
    dq, dk, dvt = A.global_attention_backward(q, k, v, bias, o, lse, do, 0.2, prec)
    D = A.global_attention_rowdot(o, do)

    def ranks(h, w):
        return [_per_rank(ops, q, k, v, do, bias, lse, D, qi, ki, prec) for qi, ki in zip(_blocks(*osh, h, w), _blocks(*ish, h, w))]

    for h, w in GRIDS:
        got = ranks(h, w)
        for r, (qi, ki) in enumerate(zip(_blocks(*osh, h, w), _blocks(*ish, h, w))):
            want = (o[:, :, qi], lse[:, :, qi], D[:, :, qi], dq[:, :, qi], dk[:, :, ki], dvt[..., ki])
            for name, a, b in zip(("o", "lse", "D", "dq", "dk", "dv"), got[r], want):
                assert torch.equal(a, b), (h, w, r, name, (a - b).abs().max().item())
    for a, b in zip(got, ranks(*GRIDS[-1])):   # a second run of the last grid
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    ag = lambda names: {n for n in names if "attention_global_kernel" in n}   # noqa: E731
    serial = ag(launched_kernels(lambda: A.global_attention_backward(q, k, v, bias, o, lse, do, 0.2, prec) +
                                 A.global_attention_forward(q, k, v, bias, 0.2, prec), lambda n: len(ag(n)) == 3))
    dist_ = ag(launched_kernels(lambda: ranks(2, 2), lambda n: len(ag(n)) == 3))
    assert serial == dist_ and len(serial) == 3, (serial, dist_)


# ---------------------------------------------------------------------------------------------------------- the module on gloo, one GPU
MODULE_CASES = [((17, 32), (17, 32), 32, 2, None, None, "equiangular"), ((12, 24), (7, 14), 24, 3, 48, 24, "legendre-gauss")]


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _module_worker(rank, world, port, h, w, q):
    try:
        torch.cuda.set_device(0)
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
        w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
        ih, iw = rank // w, rank % w
        mbd.init(h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
        res = {}

        def shard(t, hs, ws):
            return torch.split(torch.split(t, hs, dim=-2)[ih], ws, dim=-1)[iw].contiguous()

        def allsum(t):
            t = t.clone()
            dist.all_reduce(t)
            return t

        for n, (ish, osh, C, heads, ck, cv, gi) in enumerate(MODULE_CASES):
            same = ish == osh
            for tf32 in (False, True):
                torch.backends.cuda.matmul.allow_tf32 = tf32
                kw = dict(grid_in=gi, k_channels=ck, out_channels=cv)
                torch.manual_seed(5)
                mod = mbd.DistributedAttentionS2(C, heads, ish, osh, **kw).to(DEV)
                torch.manual_seed(5)
                ser = A.AttentionS2(C, heads, ish, osh, **kw).to(DEV)
                with torch.no_grad():
                    g = torch.Generator(device=DEV).manual_seed(6)
                    for (_, a), (_, b) in zip(mod.named_parameters(), ser.named_parameters()):
                        if a.dim() == 1:
                            a.normal_(0.0, 0.2, generator=g)
                            b.copy_(a)
                g = torch.Generator(device=DEV).manual_seed(7 + n)
                query = torch.randn(2, C, *osh, device=DEV, generator=g)
                kv = query if same else torch.randn(2, C, *ish, device=DEV, generator=g)
                gy = torch.randn(2, mod.out_channels, *osh, device=DEV, generator=g)
                xs = [query.clone().requires_grad_(True)] + ([] if same else [kv.clone().requires_grad_(True)])
                y = ser(xs[0], None if same else xs[1], None if same else xs[1])
                y.backward(gy)
                ins = [shard(query, mod.lat_out_shapes, mod.lon_out_shapes).requires_grad_(True)]
                if not same:
                    ins.append(shard(kv, mod.lat_in_shapes, mod.lon_in_shapes).requires_grad_(True))
                yr = mod(ins[0], None if same else ins[1], None if same else ins[1])
                yr.backward(shard(gy, mod.lat_out_shapes, mod.lon_out_shapes))
                tag = f"m{n}/{'tf32' if tf32 else 'fp32'}"
                res[f"{tag}/out"] = (_rel(yr.detach(), shard(y.detach(), mod.lat_out_shapes, mod.lon_out_shapes)), tf32)
                res[f"{tag}/dquery"] = (_rel(ins[0].grad, shard(xs[0].grad, mod.lat_out_shapes, mod.lon_out_shapes)), tf32)
                if not same:
                    res[f"{tag}/dkv"] = (_rel(ins[1].grad, shard(xs[1].grad, mod.lat_in_shapes, mod.lon_in_shapes)), tf32)
                for (name, a), (_, b) in zip(mod.named_parameters(), ser.named_parameters()):
                    if name == "k_bias":   # exactly zero on one GPU up to rounding: hold it to the scale of the key weights' gradient
                        res[f"{tag}/d{name}"] = ((allsum(a.grad).norm() / ser.k_weights.grad.norm()).item(), tf32)
                    else:
                        res[f"{tag}/d{name}"] = (_rel(allsum(a.grad), b.grad), tf32)
        # bf16 inputs are accepted; the output is fp32
        torch.backends.cuda.matmul.allow_tf32 = False
        ish, osh, C, heads, ck, cv, gi = MODULE_CASES[1]
        torch.manual_seed(8)
        mod = mbd.DistributedAttentionS2(C, heads, ish, osh, grid_in=gi, k_channels=ck, out_channels=cv).to(DEV)
        torch.manual_seed(8)
        ser = A.AttentionS2(C, heads, ish, osh, grid_in=gi, k_channels=ck, out_channels=cv).to(DEV)
        g = torch.Generator(device=DEV).manual_seed(9)
        query = torch.randn(1, C, *osh, device=DEV, generator=g).bfloat16()
        kv = torch.randn(1, C, *ish, device=DEV, generator=g).bfloat16()
        with torch.no_grad():
            y = ser(query, kv, kv)
            kvr = shard(kv, mod.lat_in_shapes, mod.lon_in_shapes)
            yr = mod(shard(query, mod.lat_out_shapes, mod.lon_out_shapes), kvr, kvr)
        res["bf16/out"] = (_rel(yr, shard(y, mod.lat_out_shapes, mod.lon_out_shapes)) + float(yr.dtype != torch.float32), False)
        q.put((rank, res, None))
        dist.destroy_process_group()
    except Exception:  # pragma: no cover
        import traceback

        q.put((rank, None, traceback.format_exc()))


@pytest.mark.parametrize("h,w", [(2, 1), (2, 2), (4, 2)])
def test_module_on_one_gpu_against_attention_s2(h, w):
    world = h * w
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_module_worker, args=(r, world, port, h, w, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    for rank, res, err in out:
        assert err is None, f"rank {rank}:\n{err}"
        assert len(res) == 2 * (2 + 8) + 2 * (3 + 8) + 1, sorted(res)   # per precision: out, dquery (, dkv) and 8 parameters; bf16
        for k_, (v_, tf32) in res.items():
            assert v_ <= (2e-3 if tf32 else 1e-5), (rank, k_, v_)

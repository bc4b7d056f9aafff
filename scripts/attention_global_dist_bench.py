#!/usr/bin/env python
"""Per-rank cost of the distributed global attention (DistributedAttentionS2) on one GPU, with virtual ranks: 181 x 360 equiangular ->
itself, C = 256, 8 heads (E = 32), B = 1, in TF32 and fp32 (3 x TF32), on h x w grids 1 x 1 (the serial kernels), 2 x 1, 2 x 2 and 4 x 2.

Every rank runs the module's per-rank stage (makani_b200.distributed.attention.CudaGlobalAttentionLocalOps) on its shard of the same
operands: the forward and the q pass of its queries against all keys, the kv pass of its keys against all queries.  For each rank it prints
one JSON line with the ms of the three calls (CUDA events, L2 flushed before every call, median of --steps) and the bytes its gathers
receive, computed from the shapes: the forward receives the other ranks' k and v; the backward receives k and v again, plus q and dO, and
lse and D.  Per grid it prints the critical path (the max over ranks of forward + q pass + kv pass) against the 1 x 1 time.  It reads the
device name and power limit in the same run.  The collectives themselves need several GPUs and are not measured here.

    python scripts/attention_global_dist_bench.py [--steps 5] [--warmup 1] [--out results.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from disco_bench import device_info, timed  # noqa: E402

import makani_b200.distributed as mbd  # noqa: E402
from makani_b200 import _lib  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.distributed import attention as DA  # noqa: E402

SHAPE, C, HEADS, B = (181, 360), 256, 8, 1
GRIDS = [(1, 1), (2, 1), (2, 2), (4, 2)]


def blocks(nlat, nlon, h, w, dev):
    """the point indices of every rank's (lat, lon) block, rank = ih * w + iw"""
    lat, lon = mbd.compute_split_shapes(nlat, h), mbd.compute_split_shapes(nlon, w)
    out, a = [], 0
    for ih in range(h):
        b = 0
        for iw in range(w):
            rows, cols = torch.arange(a, a + lat[ih]), torch.arange(b, b + lon[iw])
            out.append((rows[:, None] * nlon + cols[None, :]).reshape(-1).to(dev))
            b += lon[iw]
        a += lat[ih]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attention_global_dist_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    info = device_info()
    print(json.dumps(info), flush=True)
    E = C // HEADS
    n = SHAPE[0] * SHAPE[1]
    g = torch.Generator(device=dev).manual_seed(0)
    q, k = torch.randn(B, HEADS, n, E, device=dev, generator=g), torch.randn(B, HEADS, n, E, device=dev, generator=g)
    v, do = torch.randn(B, HEADS, E, n, device=dev, generator=g), torch.randn(B, HEADS, n, E, device=dev, generator=g)
    bias = A.AttentionS2(C, HEADS, SHAPE, SHAPE).key_bias.to(dev)
    ops = DA.CudaGlobalAttentionLocalOps(None)
    scale = E ** -0.5
    rows, summary = [], []
    for prec_name, prec in (("tf32", _lib.PREC_TF32), ("fp32", _lib.PREC_FP32X3)):
        o, lse = ops.forward(q, k, v, bias, scale, prec)
        D = ops.rowdot(o, do)
        serial = None
        for h, w in GRIDS:
            p = h * w
            per = []
            for r, (qi, ki) in enumerate(zip(blocks(*SHAPE, h, w, dev), blocks(*SHAPE, h, w, dev))):
                qr, dor = q[:, :, qi].contiguous(), do[:, :, qi].contiguous()
                kr, vr, br = k[:, :, ki].contiguous(), v[..., ki].contiguous(), bias[ki].contiguous()
                o_r, lse_r = ops.forward(qr, k, v, bias, scale, prec)
                D_r = ops.rowdot(o_r, dor)
                t_f = timed(lambda: ops.forward(qr, k, v, bias, scale, prec), args.steps, args.warmup, True)
                t_q = timed(lambda: ops.backward_q(qr, k, v, bias, lse_r, D_r, dor, scale, prec), args.steps, args.warmup, True)
                t_kv = timed(lambda: ops.backward_kv(q, kr, vr, br, lse, D, do, scale, prec), args.steps, args.warmup, True)
                nq_o, nk_o = n - qi.numel(), n - ki.numel()   # points held by the other ranks
                kv_bytes = B * HEADS * nk_o * 2 * E * 4
                row = {"prec": prec_name, "h": h, "w": w, "rank": r, "nq": qi.numel(), "nk": ki.numel(), "forward_ms": round(t_f, 3),
                       "q_pass_ms": round(t_q, 3), "kv_pass_ms": round(t_kv, 3), "total_ms": round(t_f + t_q + t_kv, 3),
                       "recv_fwd_bytes": kv_bytes, "recv_bwd_bytes": kv_bytes + B * HEADS * nq_o * (2 * E + 2) * 4}
                per.append(row)
                rows.append(row)
                print(json.dumps(row), flush=True)
                del o_r, lse_r, D_r
            crit = max(x["total_ms"] for x in per)
            serial = crit if p == 1 else serial
            s = {"prec": prec_name, "grid": f"{h}x{w}", "ranks": p, "critical_ms": crit, "min_rank_ms": min(x["total_ms"] for x in per),
                 "speedup_vs_1x1": round(serial / crit, 2), "ideal": p}
            summary.append(s)
            print(json.dumps(s), flush=True)
        del o, lse, D
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"device": info, "ranks": rows, "grids": summary}, f, indent=1)


if __name__ == "__main__":
    main()

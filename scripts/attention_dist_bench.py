#!/usr/bin/env python
"""Per-rank cost of the distributed neighbourhood attention (DistributedNeighborhoodAttentionS2) at FCN3's processor shape on one GPU:
360 x 720 Legendre-Gauss -> itself, theta_cutoff = 4 pi / 359, C = 256, 8 heads (E = 32), B = 1, fp32; w = 1, so every polar rank holds the
8 (b, h) pairs and runs its window plan at heads = 1, B = 8.

For h in {1 (the serial plan), 2, 4} and every polar rank it prints one JSON line with the window (output rows, input rows lo .. hi), the ms
of the forward kernel and of the query-side and key/value-side kernels of the backward (L2 flushed before every call, median), and the halo
of the rank computed from the shapes: the input rows it receives from other ranks and the bytes of k and v that brings in per forward (the
backward's halo adjoint sends the same bytes of dk and dv back; at w > 1 both shrink by the share of pairs).  Once it prints the device name,
power limit and clocks read in the same run.  The collectives (azimuth all-to-all, polar halo) need several GPUs and are not measured here.

    python scripts/attention_dist_bench.py [--steps 10] [--warmup 3]
"""
import argparse
import json
import math
import os
import sys
from types import SimpleNamespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from attention_bench import kernel_times  # noqa: E402
from disco_bench import device_info, timed  # noqa: E402

import makani_b200.distributed as mbd  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.distributed import attention as DA  # noqa: E402
from makani_b200.distributed import disco as DD  # noqa: E402

KEY = ((360, 720), (360, 720), "legendre-gauss", "legendre-gauss", 4 * math.pi / 359)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--channels", type=int, default=256)
    ap.add_argument("--heads", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attention_dist_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    nb = A.get_neighbourhood(*KEY)
    (hi, wi), (ho, wo) = KEY[0], KEY[1]
    R, E = args.heads, args.channels // args.heads             # B = 1: one (b, h) pair per head
    scale = 1.0 / math.sqrt(E)
    q, dy = torch.randn(R, ho * wo, E, device=dev), torch.randn(R, ho * wo, E, device=dev)
    k, v = torch.randn(R, hi * wi, E, device=dev), torch.randn(R, hi * wi, E, device=dev)
    for h in (1, 2, 4):
        wins = DD.disco_windows(nb, mbd.compute_split_shapes(ho, h))
        for r, win in enumerate(wins):
            plan = DA.CudaAttentionLocalOps(SimpleNamespace(_key=KEY, window=win))._plan(dev)
            o, i = slice(win.t0 * wo, win.t1 * wo), slice(win.lo * wi, win.hi * wi)
            qw, dyw, kw, vw = q[:, o].contiguous(), dy[:, o].contiguous(), k[:, i].contiguous(), v[:, i].contiguous()
            y, lse = plan.forward_attention(qw, kw, vw, 1, scale)
            fwd = timed(lambda: plan.forward_attention(qw, kw, vw, 1, scale), args.steps, args.warmup, True)
            bwd = kernel_times(lambda: plan.backward_attention(qw, kw, vw, y, lse, dyw, 1, scale), args.steps, args.warmup)
            _, recv = DD.halo_plan(wins, mbd.compute_split_shapes(hi, h), r)
            halo_rows = int(sum(recv) - recv[r])
            print(json.dumps({"h": h, "rank": r, "out_rows": [win.t0, win.t1], "in_rows": [win.lo, win.hi], "pairs": R, "E": E,
                              "support_points": int(win.psi.row_ptr[-1]), "forward_kernel_ms": round(fwd, 3),
                              "query_side_kernel_ms": round(bwd["query_side_kernel_ms"], 3), "kv_side_kernel_ms": round(bwd["kv_side_kernel_ms"], 3),
                              "halo_rows_in": halo_rows, "halo_bytes_fwd": halo_rows * wi * R * 2 * E * 4}), flush=True)
            del y, lse
    print(json.dumps(device_info()))


if __name__ == "__main__":
    main()

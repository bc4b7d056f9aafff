#!/usr/bin/env python
"""Timing of the per-rank stages of DistributedInstanceNorm2d (makani_b200.distributed, on the staged norm kernels of csrc/norm.cu with q = 1)
against makani's formula of the same layer in eager PyTorch ops, on one GPU, for the local shard of rank 0 of realistic h x w splits:
1 x 384 x 240 x 480 at 2 x 2 and 4 x 2 (the SFNO inner grid at scale 3) and 1 x 8 x 721 x 1440 at 4 x 2, fp32 and bf16, affine.  The all-gathers
between the stages are not timed (one GPU, world size 1: the gather is the identity), so the numbers are the rank's own work.  ms per forward and per
backward (CUDA events, the median of --steps calls after --warmup, L2 flushed before every call) and the bytes-based share of HBM bandwidth:
3 N s bytes forward (statistics read x, apply reads x and writes y) and 5 N s backward, N elements of s bytes, over the H100 SXM data sheet's
3.35 TB/s.  The two implementations alternate round by round, so drifts of clock and neighbours fall on both alike.  Prints the device name, power
limit and clocks, then one JSON line per (round, workload, dtype, impl).

    python scripts/instance_norm_dist_bench.py [--rounds 2] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import makani_b200.distributed as mbd  # noqa: E402
from makani_b200.distributed.primitives import compute_split_shapes  # noqa: E402
from norm_s2_bench import HBM_BYTES_PER_S, device_info, timed  # noqa: E402

# (B, C, H, W) of the global field, (h, w) of the grid
WORKLOADS = [((1, 384, 240, 480), (2, 2)), ((1, 384, 240, 480), (4, 2)), ((1, 8, 721, 1440), (4, 2))]


def eager(x, weight, bias, eps):
    """makani's DistributedInstanceNorm2d.forward on one rank in eager torch operators (makani compiles its normalize and Welford kernels with
    torch.compile): var_mean, the point count, the Welford combine of the gathered [1] entries, normalize and affine in fp32, cast back"""
    B, C = x.shape[:2]
    xf = x.to(torch.float32)
    var, mean = torch.var_mean(xf, dim=(-2, -1), unbiased=False, keepdim=False)
    count = torch.sum(torch.ones_like(xf, requires_grad=False), dim=(-2, -1), keepdim=False)
    vmc = torch.stack([var, mean, count], dim=0).unsqueeze(1).contiguous()      # what makani all-gathers over the spatial group
    var, mean = (vmc[0, 0] * vmc[2, 0]) / vmc[2, 0], vmc[1, 0]
    xf = (xf - mean.reshape(B, C, 1, 1)) / torch.sqrt(var.reshape(B, C, 1, 1) + eps)
    xf = weight.reshape(-1, 1, 1) * xf + bias.reshape(-1, 1, 1)
    return xf.to(x.dtype)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("instance_norm_dist_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    print(json.dumps(device_info()), flush=True)
    for r in range(a.rounds):
        for (B, C, H, W), (h, w) in WORKLOADS:
            Hl, Wl = compute_split_shapes(H, h)[0], compute_split_shapes(W, w)[0]
            m = mbd.DistributedInstanceNorm2d(C, eps=1e-6, affine=True).to(dev)
            with torch.no_grad():
                m.weight.add_(0.3 * torch.randn(C, device=dev, generator=gen))
                m.bias.add_(0.2 * torch.randn(C, device=dev, generator=gen))
            for dtype in (torch.float32, torch.bfloat16):
                x = torch.randn(B, C, Hl, Wl, device=dev, generator=gen).to(dtype).requires_grad_(True)
                dy = torch.randn(B, C, Hl, Wl, device=dev, generator=gen).to(dtype)
                n_bytes = x.numel() * x.element_size()
                impls = [("kernels", lambda: m(x)), ("makani_eager", lambda: eager(x, m.weight, m.bias, m.eps))]
                for name, fwd in impls:
                    with torch.no_grad():
                        tf = timed(fwd, a.steps, a.warmup, flush)
                    y = fwd()
                    tb = timed(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), a.steps, a.warmup, flush)
                    del y
                    print(json.dumps({"round": r, "global": [B, C, H, W], "grid": f"{h}x{w}", "local": [B, C, Hl, Wl],
                                      "dtype": str(dtype).split(".")[-1], "impl": name, "forward_ms": round(tf, 4), "backward_ms": round(tb, 4),
                                      "forward_hbm_share": round(3 * n_bytes / (tf * 1e-3) / HBM_BYTES_PER_S, 3),
                                      "backward_hbm_share": round(5 * n_bytes / (tb * 1e-3) / HBM_BYTES_PER_S, 3)}), flush=True)
                del x, dy
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

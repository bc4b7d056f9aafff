#!/usr/bin/env python
"""Timing of the quadrature-weighted instance norm (GeometricInstanceNormS2 on the kernels of csrc/norm.cu) against makani's eager formula of the
same layer, B = 1, C = 384, at 240 x 480 (the SFNO inner grid at scale 3, Legendre-Gauss) and 721 x 1440 (the last block, equiangular), fp32 and
bf16, GELU fused.  ms per forward and per backward (CUDA events, the median of --steps calls after --warmup, L2 flushed before every call) and the
bytes-based share of HBM bandwidth: 3 N s bytes forward (statistics read x, apply reads x and writes y) and 5 N s backward (sums read x, dy; apply
reads x, dy and writes dx), N elements of s bytes, over the H100 SXM data sheet's 3.35 TB/s.  The two implementations alternate round by round, so
drifts of clock and neighbours fall on both alike.  Prints the device name, power limit and clocks, then one JSON line per (round, workload, impl).

    python scripts/norm_s2_bench.py [--rounds 3] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from makani_b200.norm import GeometricInstanceNormS2  # noqa: E402
from makani_b200.quadrature import crop_quadrature_np  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
WORKLOADS = [((240, 480), "legendre-gauss"), ((721, 1440), "equiangular")]
B, C = 1, 384


def device_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


def eager(x, qw, weight, bias, eps):
    """makani's GeometricInstanceNormS2.forward in eager torch operators (its normalize kernel is torch.compile'd there), then the GELU"""
    Bx, Cx = x.shape[:2]
    xf = x.to(torch.float32)
    mean = torch.sum(xf * qw, dim=(-2, -1))
    var = torch.sum(torch.square(xf - mean.reshape(Bx, Cx, 1, 1)) * qw, dim=(-2, -1))
    xf = (xf - mean.reshape(Bx, Cx, 1, 1)) / torch.sqrt(var.reshape(Bx, Cx, 1, 1) + eps)
    xf = weight.reshape(-1, 1, 1) * xf + bias.reshape(-1, 1, 1)
    return F.gelu(xf.to(x.dtype))


def timed(fn, steps, warmup, flush):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(steps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("norm_s2_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    print(json.dumps(device_info()), flush=True)
    for r in range(a.rounds):
        for (H, W), grid in WORKLOADS:
            m = GeometricInstanceNormS2((H, W), (H, W), (0, 0), grid, C, eps=1e-6, affine=True).to(dev)
            qw = torch.from_numpy(crop_quadrature_np(grid, (H, W))).to(dev, torch.float32)
            qw = qw.view(1, 1, H, 1).expand(1, 1, H, W).contiguous()      # makani holds the weights as a full (1, 1, H, W) tensor
            for dtype in (torch.float32, torch.bfloat16):
                x = torch.randn(B, C, H, W, device=dev, generator=gen).to(dtype).requires_grad_(True)
                dy = torch.randn(B, C, H, W, device=dev, generator=gen).to(dtype)
                n_bytes = B * C * H * W * x.element_size()
                impls = [("kernels", lambda: m(x, gelu=True)), ("makani_eager", lambda: eager(x, qw, m.weight, m.bias, m.eps))]
                for name, fwd in impls:
                    with torch.no_grad():
                        tf = timed(fwd, a.steps, a.warmup, flush)
                    y = fwd()
                    tb = timed(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), a.steps, a.warmup, flush)
                    del y
                    print(json.dumps({"round": r, "shape": [B, C, H, W], "grid": grid, "dtype": str(dtype).split(".")[-1], "impl": name,
                                      "forward_ms": round(tf, 4), "backward_ms": round(tb, 4),
                                      "forward_hbm_share": round(3 * n_bytes / (tf * 1e-3) / HBM_BYTES_PER_S, 3),
                                      "backward_hbm_share": round(5 * n_bytes / (tb * 1e-3) / HBM_BYTES_PER_S, 3)}), flush=True)
                del x, dy
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

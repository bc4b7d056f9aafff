#!/usr/bin/env python
"""Timing of the channel layer norm (DistributedLayerNorm on the kernels of csrc/norm.cu) against makani's eager formula of the same layer
(transpose -> nn.LayerNorm -> transpose -> .contiguous(), then the GELU that follows it in the SFNO block), B = 1, C = 384, at 240 x 480 (the SFNO
inner grid) and 721 x 1440, fp32, and bf16 under autocast as the network runs it (bf16 x, fp32 y and dy: layer_norm is on autocast's fp32 list),
GELU fused.  ms per forward and per backward (CUDA events, the median of --steps calls after --warmup, L2 flushed before every call) and the
bytes-based share of HBM bandwidth: the forward must read x and write y, the backward read x and dy and write dx, N elements each in their dtypes,
over the H100 SXM data sheet's 3.35 TB/s.  The two implementations alternate round by round, so drifts of clock and neighbours fall on both alike.
Prints the device name, power limit and clocks, then one JSON line per (round, workload, impl).

    python scripts/layer_norm_bench.py [--rounds 3] [--steps 20] [--warmup 5]
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

from makani_b200.norm import DistributedLayerNorm  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
SHAPES = [(240, 480), (721, 1440)]
B, C = 1, 384


def device_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


def eager(m, x):
    """makani's DistributedLayerNorm.forward (makani/mpu/layer_norm.py:284-290), then the GELU"""
    return F.gelu(torch.transpose(m.norm(torch.transpose(x, 1, 3)), 1, 3).contiguous())


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
        raise SystemExit("layer_norm_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    print(json.dumps(device_info()), flush=True)
    m = DistributedLayerNorm(C, eps=1e-6).to(dev)
    with torch.no_grad():
        m.norm.weight.add_(0.1 * torch.randn(C, device=dev, generator=gen))
        m.norm.bias.add_(0.1 * torch.randn(C, device=dev, generator=gen))
    for r in range(a.rounds):
        for H, W in SHAPES:
            for dtype, autocast in ((torch.float32, False), (torch.bfloat16, True)):
                x = torch.randn(B, C, H, W, device=dev, generator=gen).to(dtype).requires_grad_(True)
                out_dtype = torch.float32
                dy = torch.randn(B, C, H, W, device=dev, generator=gen).to(out_dtype)
                n = B * C * H * W
                fwd_bytes = n * (x.element_size() + dy.element_size())
                bwd_bytes = n * (2 * x.element_size() + dy.element_size())
                impls = [("kernels", lambda: m(x, gelu=True)), ("makani_eager", lambda: eager(m, x))]
                for name, fn in impls:
                    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                        with torch.no_grad():
                            tf = timed(fn, a.steps, a.warmup, flush)
                        y = fn()
                    assert y.dtype == out_dtype
                    tb = timed(lambda: torch.autograd.grad(y, x, dy, retain_graph=True), a.steps, a.warmup, flush)
                    del y
                    print(json.dumps({"round": r, "shape": [B, C, H, W], "dtype": str(dtype).split(".")[-1] + ("-autocast" if autocast else ""),
                                      "impl": name, "forward_ms": round(tf, 4), "backward_ms": round(tb, 4),
                                      "forward_hbm_share": round(fwd_bytes / (tf * 1e-3) / HBM_BYTES_PER_S, 3),
                                      "backward_hbm_share": round(bwd_bytes / (tb * 1e-3) / HBM_BYTES_PER_S, 3)}), flush=True)
                del x, dy
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

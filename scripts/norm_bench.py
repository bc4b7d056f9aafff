#!/usr/bin/env python
"""Timing of the instance norm (+ GELU) kernels (csrc/norm.cu) at the SFNO block's shape, B = 1, C = 384, 240 x 480, fp32 and bf16: ms per
forward (statistics + apply) and per backward (reduce + apply), CUDA events, the median of --steps calls after --warmup, L2 flushed before
every call.  Several builds of the library can be compared in one run: their calls alternate round by round, so drifts of clock and
neighbours fall on all of them alike.  Prints one JSON line per (round, library, dtype) and once the device name, power limit and clocks.

    python scripts/norm_bench.py [--libs a.so,b.so] [--rounds 5] [--steps 50] [--warmup 10]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from makani_b200 import _lib  # noqa: E402

B, C, H, W = 1, 384, 240, 480


def device_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


def load(path):
    lib = ctypes.CDLL(path)
    for name in ("b200sht_pointwise_workspace_floats", "b200sht_instance_norm_forward", "b200sht_instance_norm_backward", "b200sht_last_error"):
        res, args = _lib._SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


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
    ap.add_argument("--libs", default=_lib.LIB_PATH)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    libs = [(p, load(p)) for p in a.libs.split(",")]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    gen = torch.Generator(device=dev).manual_seed(0)
    print(json.dumps(device_info()), flush=True)
    for r in range(a.rounds):
        for dtype in (torch.float32, torch.bfloat16):
            dt = _lib.BF16 if dtype == torch.bfloat16 else _lib.F32
            x = torch.randn(B, C, H, W, device=dev, generator=gen).to(dtype)
            dy = torch.randn(B, C, H, W, device=dev, generator=gen).to(dtype)
            y, dx = torch.empty_like(x), torch.empty_like(x)
            gamma, beta = torch.ones(C, device=dev), torch.zeros(C, device=dev)
            stats, sums = torch.empty(B * C, 2, device=dev), torch.empty(B * C, 2, device=dev)
            for path, lib in libs:
                ws = torch.empty(int(lib.b200sht_pointwise_workspace_floats(B, C, H * W)), device=dev)
                p = lambda t: ctypes.c_void_p(t.data_ptr())
                fwd = lambda: lib.b200sht_instance_norm_forward(p(x), p(y), p(gamma), p(beta), p(stats), p(ws), dt, B, C, H * W, 1e-6, 1, st)
                bwd = lambda: lib.b200sht_instance_norm_backward(p(x), p(dy), p(dx), p(gamma), p(beta), p(stats), p(sums), p(ws), dt, B, C, H * W, 1, st)
                assert fwd() == 0 and bwd() == 0, lib.b200sht_last_error()
                tf, tb = timed(fwd, a.steps, a.warmup, flush), timed(bwd, a.steps, a.warmup, flush)
                print(json.dumps({"round": r, "lib": os.path.basename(path), "dtype": str(dtype).split(".")[-1], "shape": [B, C, H, W],
                                  "forward_ms": round(tf, 4), "backward_ms": round(tb, 4)}), flush=True)


if __name__ == "__main__":
    main()

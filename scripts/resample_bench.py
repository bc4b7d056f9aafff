#!/usr/bin/env python
"""Benchmark of the bilinear resampling (ResampleS2) at FCN3's two decoder resamplings, B = 1, 360 x 720 Legendre-Gauss -> 721 x 1440 equiangular:
  atmo  585 planes (13 pressure levels x atmo_embed_dim 45)
  surf   56 planes (surf_embed_dim 56)
For each it prints one JSON line with
  * the forward and the adjoint kernel time (CUDA events, median, the L2 flushed before every call), and the bytes each must move (input read
    once + output written once) over that time against the 3.35 TB/s of the H100 SXM data sheet;
  * the oracle's torch composition (pole concat, index gathers, torch.lerp; the shape of torch-harmonics' own path) in fp32 on the same GPU,
    forward and forward + backward, as the baseline;
  * one full DiscreteContinuousDecoder step, resample + DISCO convolution (morlet (3, 3), "mean", 45 -> 5 channels in groups of 5 per level for
    atmo, 56 -> 7 in groups of 7 for surf, FCN3's 72 output channels), forward + backward;
and once the device name, power limit and clocks, read in the same run.

    python scripts/resample_bench.py [--steps 20] [--warmup 3] [--only atmo,surf] [--no-baseline] [--no-decoder]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import makani_b200 as mb  # noqa: E402
from oracle import makani_resample_oracle as O  # noqa: E402

PEAK_TBS = 3.35
IN, OUT, GRID_IN, GRID_OUT = (360, 720), (721, 1440), "legendre-gauss", "equiangular"
# (batch rows, input channels, output channels) of the decoder: the atmospheric decoder runs on B * 13 levels
SHAPES = {"atmo": (13, 45, 5), "surf": (1, 56, 7)}


def device_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


_FLUSH = None


def timed(step, steps, warmup, flush=True):
    global _FLUSH
    if _FLUSH is None:
        _FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # larger than the 50 MB L2
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        if flush:
            _FLUSH.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def bench(name, rows, cin, cout, steps, warmup, baseline, decoder):
    dev = torch.device("cuda", 0)
    planes = rows * cin
    res_mod = mb.ResampleS2(*IN, *OUT, grid_in=GRID_IN, grid_out=GRID_OUT).to(dev)
    plan = res_mod.plan(dev)
    x = torch.randn(planes, *IN, device=dev)
    dy = torch.randn(planes, *OUT, device=dev)
    res = {"shape": name, "planes": planes, "in": IN, "out": OUT, "plan_bytes": plan.query(5)}
    nbytes = planes * (IN[0] * IN[1] + OUT[0] * OUT[1]) * 4
    res["bytes_per_call"] = nbytes
    for s, f in (("forward", lambda: plan.forward(x)), ("adjoint", lambda: plan.adjoint(dy))):
        ms = timed(f, steps, warmup)
        tbs = nbytes / (ms * 1e-3) / 1e12
        res[f"{s}_ms"], res[f"{s}_TBps"], res[f"{s}_frac_of_3.35TBps"] = round(ms, 4), round(tbs, 3), round(tbs / PEAK_TBS, 3)
    if baseline:
        tab = O.tables(*IN, *OUT, GRID_IN, GRID_OUT)
        res["oracle_forward_ms"] = round(timed(lambda: O.resample(x, tab), max(3, steps // 4), 1), 3)
        xg = x.detach().requires_grad_(True)
        res["oracle_fwd_bwd_ms"] = round(timed(lambda: O.resample(xg, tab).backward(dy), max(3, steps // 4), 1), 3)
        del xg
        torch.cuda.empty_cache()
    if decoder:
        conv = mb.DiscreteContinuousConvS2(cin, cout, OUT, OUT, (3, 3), basis_type="morlet", basis_norm_mode="mean", grid_in=GRID_OUT,
                                           grid_out=GRID_OUT, groups=math.gcd(cin, cout), bias=False,
                                           theta_cutoff=(3 + 1) * 0.5 * math.pi / float(OUT[0] - 1)).to(dev)
        xd = torch.randn(rows, cin, *IN, device=dev, requires_grad=True)
        gy = torch.randn(rows, cout, *OUT, device=dev)

        def step():
            conv(res_mod(xd)).backward(gy)

        try:
            res["decoder_step_ms"] = round(timed(step, max(3, steps // 4), 1), 3)
            res["decoder_peak_GB"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
        except torch.cuda.OutOfMemoryError:
            res["decoder_step_ms"] = "not measured (out of memory)"
        del xd, gy, conv
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default=",".join(SHAPES))
    ap.add_argument("--no-baseline", action="store_true")
    ap.add_argument("--no-decoder", action="store_true")
    a = ap.parse_args()
    print(json.dumps(device_info()), flush=True)
    for name in a.only.split(","):
        print(json.dumps(bench(name, *SHAPES[name], a.steps, a.warmup, not a.no_baseline, not a.no_decoder)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

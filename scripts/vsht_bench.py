#!/usr/bin/env python
"""Benchmark of the vector SHT on the workload of makani's VortDivCRPSLoss: forward and backward of isht(vsht(x)) for x of shape
(1, E, 15, 2, 721, 1440) fp32 (the 15 u / v pairs of the 73-channel set), with the losses' defaults lmax = 721, mmax = 721.

For each precision (fp32, tf32) it prints, as one JSON line:
  * ms per step (forward + backward), CUDA events, the L2 flushed before every step;
  * per-kernel device time from torch.profiler (a separate, shorter run) and, for the kernels whose traffic is fixed by the shapes,
    the algorithmic bytes over that time;
  * the same computation as the oracle's einsums on the GPU (torch.fft + cuBLAS, fp32, TF32 allowed at tf32) as an informational baseline;
and once the device name, power limit and clocks (read in the same run) and the vector plan's table bytes.

    python scripts/vsht_bench.py [--ensemble 4] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import makani_b200 as mb  # noqa: E402
from oracle import makani_vector_oracle as V  # noqa: E402

NLAT, NLON, PAIRS = 721, 1440, 15


def device_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


def timed(step, steps, warmup):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # larger than the 50 MB L2
    for _ in range(warmup):
        step()
    times = []
    for _ in range(steps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return {"median_ms": times[len(times) // 2], "min_ms": times[0], "max_ms": times[-1]}


def kernel_times(step, n=3):
    from torch.profiler import ProfilerActivity, profile

    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            step()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t > 0:
            out[e.key[:90]] = round(t / 1000.0 / n, 4)   # ms per step
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ensemble", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-baseline", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vsht_bench.py measures on a CUDA device; none found")
    torch.manual_seed(333)
    E = a.ensemble
    x = torch.randn(1, E, PAIRS, 2, NLAT, NLON, device="cuda")
    gy = torch.randn_like(x)
    n = E * PAIRS   # vector fields
    info = device_info()
    plan = mb.get_plan(NLAT, NLON, NLAT, NLAT, "equiangular", True, "cuda", vector=True)
    kp, L, M = plan.kp, NLAT, NLAT
    info["table_bytes"] = plan.query(5)
    info["workload"] = f"isht(vsht(x)) forward + backward, x (1, {E}, {PAIRS}, 2, {NLAT}, {NLON}) fp32, lmax = mmax = {NLAT}"
    print(json.dumps(info), flush=True)
    # algorithmic bytes of the kernels whose traffic the shapes fix (fp32): the Legendre stages read the stacked table once and their
    # activation operand once and write their result once
    lat = 4 * ((M + 7) // 8 * 8) * 2 * (2 * n) * kp
    spec = 4 * 2 * L * M * 2 * ((2 * n + 3) // 4 * 4)
    legendre_bytes = info["table_bytes"] + lat + spec
    for precision in ("fp32", "tf32"):
        vsht = mb.RealVectorSHT(NLAT, NLON, precision=precision)
        ivsht = mb.InverseRealVectorSHT(NLAT, NLON, precision=precision)
        xr = x.clone().requires_grad_(True)

        def step():
            xr.grad = None
            y = ivsht(vsht(xr))
            y.backward(gy)

        res = {"impl": "makani_b200", "precision": precision, **timed(step, a.steps, a.warmup)}
        ks = kernel_times(step)
        res["kernels_ms_per_step"] = ks
        # each Legendre stage runs twice per step (analysis: forward + backward of the inverse; synthesis: inverse + backward of the forward)
        leg = {k: v for k, v in ks.items() if "umma_kernel" in k or "legendre" in k}
        res["legendre_GBps"] = {k: round(2 * legendre_bytes / (v * 1e-3) / 1e9, 1) for k, v in leg.items()}
        print(json.dumps(res), flush=True)
        if not a.no_baseline:
            torch.backends.cuda.matmul.allow_tf32 = precision == "tf32"
            ov = V.RealVectorSHT(NLAT, NLON, dtype=torch.float32).cuda()
            oiv = V.InverseRealVectorSHT(NLAT, NLON, dtype=torch.float32).cuda()
            xb = x[:, :1].clone().requires_grad_(True)   # one ensemble member: the einsum baseline's intermediates are large
            gb = gy[:, :1]

            def base():
                xb.grad = None
                oiv(ov(xb)).backward(gb)

            r = timed(base, max(3, a.steps // 4), 2)
            print(json.dumps({"impl": "oracle einsums (torch.fft + cuBLAS), informational", "precision": precision, "ensemble_members": 1,
                              **r, "median_ms_scaled_to_E": r["median_ms"] * E}), flush=True)
            torch.backends.cuda.matmul.allow_tf32 = False
            del ov, oiv
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

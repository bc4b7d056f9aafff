#!/usr/bin/env python
"""Benchmark of the DISCO convolution (DiscreteContinuousConvS2, morlet (3, 3), "mean") at FCN3's three shapes, B = 1:
  encoder    721 x 1440 equiangular -> 360 x 720 Legendre-Gauss, 72 -> 677 channels, cutoff (3 + 1) / 2 pi / 720
  processor  360 x 720 -> 360 x 720 Legendre-Gauss, 677 -> 677 channels, cutoff 2 (3 + 1) / 2 pi / 359 (the "local" blocks)
  decoder    721 x 1440 -> 721 x 1440 equiangular, 72 -> 72 channels, cutoff (3 + 1) / 2 pi / 720
For each shape it prints one JSON line with
  * ms per forward + backward step (CUDA events), with the L2 warm and with it flushed before every step;
  * ms per stage, the L2 flushed: the contraction x -> X, the adjoint dX -> dx, and the three cuBLAS GEMMs (y = W X, dX = W^T dy, dW = dy X^T),
    and for the two kernels the bytes they must move (x read + X written; dX read + dx written) over their time against the 3.35 TB/s of
    the H100 SXM data sheet;
  * the oracle's roll-and-matmul contraction with psi as a torch sparse COO matrix on the same GPU (fp32), the shape of torch-harmonics' own
    torch path, as the library baseline (forward contraction only);
and once the device name, power limit and clocks, read in the same run.

    python scripts/disco_bench.py [--steps 10] [--warmup 3] [--only encoder,processor,decoder] [--no-baseline]
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
from makani_b200 import disco as D  # noqa: E402
from oracle import makani_disco_oracle as O  # noqa: E402

PEAK_TBS = 3.35
SHAPES = {
    "encoder": dict(cin=72, cout=677, ish=(721, 1440), osh=(360, 720), gi="equiangular", go="legendre-gauss", cutoff=(3 + 1) * 0.5 * math.pi / 720),
    "processor": dict(cin=677, cout=677, ish=(360, 720), osh=(360, 720), gi="legendre-gauss", go="legendre-gauss",
                      cutoff=2 * (3 + 1) * 0.5 * math.pi / 359),
    "decoder": dict(cin=72, cout=72, ish=(721, 1440), osh=(721, 1440), gi="equiangular", go="equiangular", cutoff=(3 + 1) * 0.5 * math.pi / 720),
}


def device_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


_FLUSH = None


def timed(step, steps, warmup, flush):
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


def bench(name, cfg, steps, warmup, baseline):
    dev = torch.device("cuda", 0)
    conv = mb.DiscreteContinuousConvS2(cfg["cin"], cfg["cout"], cfg["ish"], cfg["osh"], (3, 3), basis_type="morlet", grid_in=cfg["gi"],
                                       grid_out=cfg["go"], bias=True, theta_cutoff=cfg["cutoff"]).to(dev)
    plan = conv.plan(dev)
    x = torch.randn(1, cfg["cin"], *cfg["ish"], device=dev, requires_grad=True)
    gy = torch.randn(1, cfg["cout"], *cfg["osh"], device=dev)

    def step():
        conv(x).backward(gy)

    res = {"shape": name, "cin": cfg["cin"], "cout": cfg["cout"], "in": cfg["ish"], "out": cfg["osh"], "K": plan.K,
           "support_points": plan.query(6), "plan_bytes": plan.query(7), "tf32": torch.backends.cuda.matmul.allow_tf32}
    res["step_ms_warm_l2"] = timed(step, steps, warmup, False)
    res["step_ms_flushed_l2"] = timed(step, steps, warmup, True)
    xd = x.detach()
    X = plan.forward(xd)
    W = conv.weight.detach().reshape(1, cfg["cout"], -1)
    HW = cfg["osh"][0] * cfg["osh"][1]
    Xg = X.view(1, 1, -1, HW)
    gyg = gy.view(1, 1, cfg["cout"], HW)
    stages = {
        "contraction": lambda: plan.forward(xd),
        "adjoint": lambda: plan.adjoint(X),
        "gemm_y": lambda: torch.matmul(W, Xg),
        "gemm_dX": lambda: torch.matmul(W.transpose(1, 2), gyg),
        "gemm_dW": lambda: torch.matmul(gyg, Xg.transpose(2, 3)),
    }
    for s, f in stages.items():
        res[f"{s}_ms"] = timed(f, steps, warmup, True)
    hi, wi = cfg["ish"]
    bytes_x, bytes_X = cfg["cin"] * hi * wi * 4, X.numel() * 4
    for s in ("contraction", "adjoint"):
        tbs = (bytes_x + bytes_X) / (res[f"{s}_ms"] * 1e-3) / 1e12
        res[f"{s}_TBps"] = round(tbs, 3)
        res[f"{s}_frac_of_3.35TBps"] = round(tbs / PEAK_TBS, 3)
    del X
    if baseline:
        psi = D.get_psi(*plan_key(cfg))
        idx = torch.stack([torch.from_numpy(psi.ker.astype("int64")) * psi.nlat_out + torch.from_numpy(D.psi_lat_out(psi).astype("int64")),
                           torch.from_numpy(psi.col.astype("int64"))])
        sp = torch.sparse_coo_tensor(idx, torch.from_numpy(psi.val).float(), (psi.kernel_size * psi.nlat_out, hi * wi)).coalesce().to(dev)
        res["oracle_sparse_contraction_ms"] = timed(lambda: O.contraction(xd, sp, psi.kernel_size, *cfg["osh"]), 1, 1, True)
    return res


def plan_key(cfg):
    return ((3, 3), "morlet", "mean", cfg["ish"], cfg["osh"], cfg["gi"], cfg["go"], cfg["cutoff"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default=",".join(SHAPES))
    ap.add_argument("--no-baseline", action="store_true")
    a = ap.parse_args()
    print(json.dumps(device_info()), flush=True)
    for name in a.only.split(","):
        print(json.dumps(bench(name, SHAPES[name], a.steps, a.warmup, not a.no_baseline)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

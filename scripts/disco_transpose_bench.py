#!/usr/bin/env python
"""Benchmark of the transposed DISCO convolution (DiscreteContinuousConvTransposeS2, morlet (3, 3), "mean", B = 1, fp32, TF32 off):
  upsample  360 x 720 Legendre-Gauss -> 721 x 1440 equiangular, 72 -> 72 channels (a learnable upsampling decoder at FCN3's resolution)
  same      360 x 720 -> 360 x 720 Legendre-Gauss, 256 -> 256 channels
with cutoff 4 * 0.5 * pi / (nlat_out - 1).  For each shape it prints one JSON line with
  * ms per forward + backward step (CUDA events, median), the L2 warm;
  * ms per stage with the L2 flushed: the gather y = psi_T * Y (the adjoint kernel of the plan), the contraction gY = psi_T^T * gy (the
    forward kernel), and the three cuBLAS GEMMs (Y = W x, dx = W^T gY, dW = gY x^T); for the two kernels the bytes they must move (Y read +
    y written; gy read + gY written) over their time, against the 3.35 TB/s of the H100 SXM data sheet;
  * the oracle's roll-and-matmul transposed contraction (tests/disco_transpose_oracle.py) with psi_T as a torch sparse COO matrix (fp32) on
    the same GPU, the shape of torch-harmonics' own torch path, as the library baseline (the gather only), and its largest difference from
    the library's gather relative to its largest value;
and once the device name, power limit and clocks, read in the same run.

    python scripts/disco_transpose_bench.py [--steps 10] [--warmup 3] [--only upsample,same] [--no-baseline]
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import makani_b200 as mb  # noqa: E402
from makani_b200 import disco as D  # noqa: E402
from scripts.disco_bench import PEAK_TBS, device_info, timed  # noqa: E402
import disco_transpose_oracle as TO  # noqa: E402

SHAPES = {
    "upsample": dict(cin=72, cout=72, ish=(360, 720), osh=(721, 1440), gi="legendre-gauss", go="equiangular"),
    "same": dict(cin=256, cout=256, ish=(360, 720), osh=(360, 720), gi="legendre-gauss", go="legendre-gauss"),
}


def bench(name, cfg, steps, warmup, baseline):
    dev = torch.device("cuda", 0)
    cutoff = 4 * 0.5 * math.pi / (cfg["osh"][0] - 1)
    conv = mb.DiscreteContinuousConvTransposeS2(cfg["cin"], cfg["cout"], cfg["ish"], cfg["osh"], (3, 3), basis_type="morlet",
                                                grid_in=cfg["gi"], grid_out=cfg["go"], bias=True, theta_cutoff=cutoff).to(dev)
    plan = conv.plan(dev)
    x = torch.randn(1, cfg["cin"], *cfg["ish"], device=dev, requires_grad=True)
    gy = torch.randn(1, cfg["cout"], *cfg["osh"], device=dev)

    def step():
        conv(x).backward(gy)

    res = {"shape": name, "cin": cfg["cin"], "cout": cfg["cout"], "in": cfg["ish"], "out": cfg["osh"], "K": plan.K, "cutoff": cutoff,
           "support_points": plan.query(6), "plan_bytes": plan.query(7), "tf32": torch.backends.cuda.matmul.allow_tf32}
    res["step_ms"] = timed(step, steps, warmup, False)
    HW = cfg["ish"][0] * cfg["ish"][1]
    Wt = D._transposed_mix(conv.weight.detach(), 1)                                      # (1, C_out K, C_in)
    xg = x.detach().view(1, 1, cfg["cin"], HW)
    Y = torch.matmul(Wt, xg).view(1, cfg["cout"], plan.K, *cfg["ish"])
    gY = plan.forward(gy)
    gYg = gY.view(1, 1, -1, HW)
    stages = {
        "gather": lambda: plan.adjoint(Y),
        "contraction": lambda: plan.forward(gy),
        "gemm_Y": lambda: torch.matmul(Wt, xg),
        "gemm_dx": lambda: torch.matmul(Wt.transpose(1, 2), gYg),
        "gemm_dW": lambda: torch.matmul(gYg, xg.transpose(2, 3)),
    }
    for s, f in stages.items():
        res[f"{s}_ms"] = timed(f, steps, warmup, True)
    bytes_y, bytes_Y = gy.numel() * 4, Y.numel() * 4
    for s in ("gather", "contraction"):
        tbs = (bytes_y + bytes_Y) / (res[f"{s}_ms"] * 1e-3) / 1e12
        res[f"{s}_TBps"] = round(tbs, 3)
        res[f"{s}_frac_of_3.35TBps"] = round(tbs / PEAK_TBS, 3)
    if baseline:
        psi = D.get_psi(*conv._key)
        lat = torch.from_numpy(D.psi_lat_out(psi).astype("int64"))
        idx = torch.stack([torch.from_numpy(psi.ker.astype("int64")) * psi.nlat_out + lat, torch.from_numpy(psi.col.astype("int64"))])
        sp = torch.sparse_coo_tensor(idx, torch.from_numpy(psi.val).float(), (psi.kernel_size * psi.nlat_out, psi.nlat_in * psi.nlon_in))
        sp = sp.coalesce().to(dev)
        ref = TO.transpose_contraction(Y, sp, *cfg["osh"])
        res["oracle_vs_library_max_rel"] = ((ref - plan.adjoint(Y)).abs().max() / ref.abs().max()).item()
        del ref
        res["oracle_sparse_gather_ms"] = timed(lambda: TO.transpose_contraction(Y, sp, *cfg["osh"]), 1, 1, True)
    del Y, gY
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default=",".join(SHAPES))
    ap.add_argument("--no-baseline", action="store_true")
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    print(json.dumps(device_info()), flush=True)
    for name in a.only.split(","):
        print(json.dumps(bench(name, SHAPES[name], a.steps, a.warmup, not a.no_baseline)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

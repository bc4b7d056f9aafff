#!/usr/bin/env python
"""Per-rank cost of the distributed DISCO convolution (DistributedDiscreteContinuousConvS2) at FCN3's processor shape on one GPU:
360 x 720 Legendre-Gauss -> itself, morlet (3, 3), "mean", cutoff 2 (3 + 1) / 2 pi / 359, B = 1, C = 677 rows (w = 1).

For h in {1 (the serial plan), 2, 4} and every polar rank it prints one JSON line with the window (output rows, input rows lo .. hi) and the ms
of the window contraction x -> X and of the window adjoint dX -> dx (CUDA events, L2 flushed, median), and once the device name, power
limit and clocks read in the same run.  The collectives (azimuth all-to-all, polar halo) need several GPUs and are not measured here.

    python scripts/disco_dist_bench.py [--steps 10] [--warmup 3] [--channels 677]
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

from disco_bench import device_info, timed  # noqa: E402

import makani_b200.distributed as mbd  # noqa: E402
from makani_b200 import disco as D  # noqa: E402
from makani_b200.distributed import disco as DD  # noqa: E402

KEY = ((3, 3), "morlet", "mean", (360, 720), (360, 720), "legendre-gauss", "legendre-gauss", 2 * (3 + 1) * 0.5 * math.pi / 359)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--channels", type=int, default=677)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("disco_dist_bench.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    psi = D.get_psi(*KEY)
    C, K, (hi, wi), (ho, wo) = args.channels, psi.kernel_size, KEY[3], KEY[4]
    x = torch.randn(C, hi, wi, device=dev)
    for h in (1, 2, 4):
        for r, win in enumerate(DD.disco_windows(psi, mbd.compute_split_shapes(ho, h))):
            ops = DD.CudaDiscoLocalOps(SimpleNamespace(_key=KEY, window=win))
            xw = x[:, win.lo : win.hi].contiguous()
            dX = torch.randn(C, K, win.t1 - win.t0, wo, device=dev)
            fwd = timed(lambda: ops.contract(xw), args.steps, args.warmup, True)
            adj = timed(lambda: ops.adjoint(dX), args.steps, args.warmup, True)
            print(json.dumps({"h": h, "rank": r, "out_rows": [win.t0, win.t1], "in_rows": [win.lo, win.hi], "C": C,
                              "contraction_ms": round(fwd, 3), "adjoint_ms": round(adj, 3)}), flush=True)
            del dX
    print(json.dumps(device_info()))


if __name__ == "__main__":
    main()

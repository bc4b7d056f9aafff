#!/usr/bin/env python
"""Benchmark of the neighbourhood attention on the sphere (NeighborhoodAttentionS2, B = 1, fp32, TF32 off):
  processor   360 x 720 Legendre-Gauss, C = 256, 8 heads, theta_cutoff = 4 pi / 359 (FCN3's processor grid)
  downsample  keys / values on 721 x 1440 equiangular, queries on 360 x 720 Legendre-Gauss, C = 64, 4 heads, theta_cutoff = 4 pi / 1440
For each shape it prints one JSON line with
  * ms per module forward and per forward + backward step (CUDA events, median), the L2 warm;
  * ms per kernel with the L2 flushed (the forward and the backward pair through the C ABI, the two backward kernels apart from the profiler) and the
    bytes each must move, computed from the shapes (every operand read once, every output written once), over its time against the 3.35 TB/s of
    the H100 SXM data sheet;
  * as the baseline, the fp32 gather formulation of the oracle (tests/attention_oracle.py: a gather over the neighbourhood and a segment
    softmax, one output row at a time so that the pole rows fit) on the same GPU, forward only;
and once the device name, power limit and clocks, read in the same run.

    python scripts/attention_bench.py [--steps 10] [--warmup 3] [--only processor,downsample] [--no-baseline]
"""
import argparse
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import makani_b200 as mb  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.quadrature import _grid_np  # noqa: E402
from scripts.disco_bench import PEAK_TBS, device_info, timed  # noqa: E402
import attention_oracle as AO  # noqa: E402

SHAPES = {
    "processor": dict(c=256, heads=8, ish=(360, 720), osh=(360, 720), gi="legendre-gauss", go="legendre-gauss", cutoff=4 * math.pi / 359),
    "downsample": dict(c=64, heads=4, ish=(721, 1440), osh=(360, 720), gi="equiangular", go="legendre-gauss", cutoff=4 * math.pi / 1440),
}


def kernel_times(fn, steps, warmup):
    """median device time of each attention kernel `fn` launches, from the profiler, the L2 flushed before every call"""
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        fn()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            flush.zero_()
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        for key, tag in (("attn_query_kernel", "query_side_kernel"), ("attn_kv_kernel", "kv_side_kernel")):
            if key in e.name:
                us = getattr(e, "device_time_total", None)
                per.setdefault(tag, []).append(us if us is not None else e.cuda_time_total)
    return {f"{k}_ms": sorted(v)[len(v) // 2] / 1e3 for k, v in per.items()}


def bench(name, cfg, steps, warmup, baseline):
    dev = torch.device("cuda", 0)
    C, H, ish, osh = cfg["c"], cfg["heads"], cfg["ish"], cfg["osh"]
    att = mb.NeighborhoodAttentionS2(C, ish, osh, cfg["gi"], cfg["go"], num_heads=H, theta_cutoff=cfg["cutoff"]).to(dev)
    plan = att.plan(dev)
    query = torch.randn(1, C, *osh, device=dev, requires_grad=True)
    kv = torch.randn(1, C, *ish, device=dev, requires_grad=True)
    gy = torch.randn(1, C, *osh, device=dev)
    res = {"shape": name, "C": C, "heads": H, "in": ish, "out": osh, "cutoff": cfg["cutoff"], "support_points": plan.query(6),
           "tf32": torch.backends.cuda.matmul.allow_tf32}

    def fwd():
        with torch.no_grad():
            att(query, kv, kv)

    res["forward_ms"] = timed(fwd, steps, warmup, False)
    res["step_ms"] = timed(lambda: att(query, kv, kv).backward(gy), steps, warmup, False)

    HWi, HWo = ish[0] * ish[1], osh[0] * osh[1]
    q = torch.randn(1, HWo, C, device=dev)
    k, v = torch.randn(1, HWi, C, device=dev), torch.randn(1, HWi, C, device=dev)
    dy = torch.randn(1, HWo, C, device=dev)
    y, lse = plan.forward_attention(q, k, v, H, att.scale)
    dq, dk, dv, D = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v), torch.empty_like(lse)
    E = C // H

    def backward_kernels():   # the query side, then the key/value side, which reads the D the first writes
        mb._lib.call("b200sht_attention_backward", plan.handle, *[mb.sht._ptr(x) for x in (q, k, v, y, lse, dy, dq, dk, dv, D)], 1, H, E, E,
                     att.scale, mb.sht._stream(dev))

    res["forward_kernel_ms"] = timed(lambda: plan.forward_attention(q, k, v, H, att.scale), steps, warmup, True)
    res["backward_kernels_ms"] = timed(backward_kernels, steps, warmup, True)
    res.update(kernel_times(backward_kernels, steps, warmup))          # the two backward kernels apart
    f = 4  # bytes per fp32 element
    bytes_ = {"forward_kernel": f * (HWo * C + 2 * HWi * C + HWo * C + H * HWo),                  # q, k, v -> y, lse
              "query_side_kernel": f * (4 * HWo * C + 2 * H * HWo + 2 * HWi * C),                 # q, y, dy, k, v, lse -> dq, D
              "kv_side_kernel": f * (4 * HWi * C + 2 * HWo * C + 2 * H * HWo)}                    # k, v, q, dy, lse, D -> dk, dv
    for s, b in bytes_.items():
        if f"{s}_ms" not in res:
            continue
        res[f"{s}_bytes"] = b
        tbs = b / (res[f"{s}_ms"] * 1e-3) / 1e12
        res[f"{s}_TBps"] = round(tbs, 3)
        res[f"{s}_frac_of_3.35TBps"] = round(tbs / PEAK_TBS, 3)
    if baseline:
        nb = A.get_neighbourhood(*att._key)
        om = 2.0 * np.pi * _grid_np(ish[0], cfg["gi"])[1] / ish[1]
        ref, _ = AO.attention(q, k, v, nb.row_ptr, nb.col, om, ish[1], osh[1], H, att.scale)
        res["oracle_vs_library_max_rel"] = ((ref - y).abs().max() / ref.abs().max()).item()
        del ref
        res["oracle_gather_forward_ms"] = timed(lambda: AO.attention(q, k, v, nb.row_ptr, nb.col, om, ish[1], osh[1], H, att.scale), 1, 1, True)
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

"""Global attention on the sphere: the wgmma kernels of csrc/attention_global.cu against torch's scaled_dot_product_attention with the same
float attn_mask (log quadrature weight per key), forward + backward of the attention core, on the same card in the same process, the two
timed alternately.  Prints one table row per (shape, precision) and the card's name and power limit.

    python scripts/attention_global_bench.py [--reps 5] [--out results.json]

Precision "tf32": torch.backends.cuda.matmul.allow_tf32 = True (this module: single TF32 wgmma); "fp32": False (3 x TF32 in the same
kernels).  SDPA picks its own backend for fp32 operands with a float mask; which one ran is not recorded.  FLOP/s count the algorithmic
4 nq nk d (forward) + 10 nq nk d (backward) per head over the measured time, against the data-sheet dense TF32 peak of 495 TFLOP/s."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from makani_b200 import _lib  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200.quadrature import _grid_np  # noqa: E402

# (output grid, input grid, channels, heads): the attention of a spherical transformer block at ERA5-like resolutions
SHAPES = [((91, 180), (91, 180), 64, 4), ((181, 360), (181, 360), 128, 4), ((181, 360), (181, 360), 256, 8), ((361, 720), (181, 360), 256, 8)]
TF32_PEAK = 495e12


def _card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return torch.cuda.get_device_name()


def _time(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attention_global_bench: needs a CUDA device")
    card = _card()
    print(f"card: {card}")
    rows = []
    tf32_before = torch.backends.cuda.matmul.allow_tf32
    for out_shape, in_shape, C, H in SHAPES:
        nq, nk, d = out_shape[0] * out_shape[1], in_shape[0] * in_shape[1], C // H
        g = torch.Generator(device="cuda").manual_seed(0)
        q = torch.randn(1, H, nq, d, device="cuda", generator=g)
        k = torch.randn(1, H, nk, d, device="cuda", generator=g)
        v = torch.randn(1, H, d, nk, device="cuda", generator=g)
        do = torch.randn(1, H, nq, d, device="cuda", generator=g)
        w = torch.from_numpy(2 * torch.pi * _grid_np(in_shape[0], "equiangular")[1] / in_shape[1]).repeat_interleave(in_shape[1])
        bias = torch.log(w).float().cuda()
        mask = bias.view(1, 1, 1, nk).expand(1, H, nq, nk)
        vt = v.transpose(2, 3).contiguous()
        for tf32 in (True, False):
            torch.backends.cuda.matmul.allow_tf32 = tf32
            prec = _lib.PREC_TF32 if tf32 else _lib.PREC_FP32X3
            scale = d ** -0.5

            def ours():
                o, lse = A.global_attention_forward(q, k, v, bias, scale, prec)
                A.global_attention_backward(q, k, v, bias, o, lse, do, scale, prec)

            qs, ks, vs = (t.detach().clone().requires_grad_(True) for t in (q, k, vt))

            def sdpa():
                o = F.scaled_dot_product_attention(qs, ks, vs, attn_mask=mask, scale=scale)
                torch.autograd.grad(o, (qs, ks, vs), do)

            ok_sdpa = True
            try:
                sdpa()
            except RuntimeError as e:   # e.g. out of memory for the materialised mask path
                ok_sdpa = False
                print(f"sdpa failed at {out_shape} <- {in_shape}: {str(e).splitlines()[0]}")
                torch.cuda.empty_cache()
            ours()
            torch.cuda.synchronize()
            t_ours, t_sdpa = [], []
            for _ in range(a.rounds):
                t_ours.append(_time(ours, a.reps))
                if ok_sdpa:
                    t_sdpa.append(_time(sdpa, a.reps))
            flops = 14.0 * nq * nk * d * H
            row = {"out": out_shape, "in": in_shape, "C": C, "heads": H, "prec": "tf32" if tf32 else "fp32",
                   "ours_ms": [round(t, 3) for t in t_ours], "sdpa_ms": [round(t, 3) for t in t_sdpa],
                   "ours_tflops": round(flops / min(t_ours) / 1e9, 1), "ours_of_tf32_peak": round(flops / min(t_ours) / 1e-3 / TF32_PEAK, 3),
                   "sdpa_tflops": round(flops / min(t_sdpa) / 1e9, 1) if t_sdpa else None}
            rows.append(row)
            print(json.dumps(row), flush=True)
    torch.backends.cuda.matmul.allow_tf32 = tf32_before
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"card": card, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()

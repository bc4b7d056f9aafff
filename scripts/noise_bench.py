#!/usr/bin/env python
"""FourCastNet 3's input noise at the shipped shape (DiffusionNoiseS2, 721 x 1440, lmax 721, 8 channels, config/fourcastnet3.yaml's kT, lambd 1):
makani_b200.noise against makani's formulation of the same steps in torch ops around the same InverseRealSHT.

    update()                   library: normal_ -> b200sht_noise_update (AR step)
                               makani:  normal_ -> sigma * xi -> phi * state + eta -> copy_
    update(replace_state=True) library: normal_ -> b200sht_noise_update (stationary redraw)
                               makani:  normal_ -> sigma * xi -> / sqrt(1 - phi^2) on step 0 -> copy_
    forward()                  library: b200sht_noise_spectrum -> InverseRealSHT.forward_packed
                               makani:  torch.complex -> InverseRealSHT (pack -> forward_packed)

Both paths draw from same-seeded generators, so their outputs are compared bit for bit after the timing.  CUDA events around `--iters` calls after
`--warmup` calls; the median of `--repeats` windows, the paths alternating.  Prints the device name and power limit, and one JSON line.

    python scripts/noise_bench.py [--batch 1 8] [--precision fp32|tf32]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from makani_b200 import noise as mn  # noqa: E402

SHIPPED_KT = [3.0806e-5, 1.2322e-4, 4.9289e-4, 1.9716e-3, 7.8862e-3, 3.1545e-2, 1.2618e-1, 5.0472e-1]


def device_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


class MakaniPath:
    """makani/models/noise.py's DiffusionNoiseS2.update / forward of T = 1 in torch ops, on the module's buffers, transform and a generator of its own"""

    def __init__(self, n, seed):
        self.n = n
        self.state = n.state.clone()
        self.rng = torch.Generator(device=n.state.device)
        self.rng.manual_seed(seed)

    def update(self, replace_state=False):
        n = self.n
        if replace_state:
            eta = torch.empty_like(self.state)
        else:
            eta = torch.empty((self.state.shape[0], 1, n.num_channels, n.lmax_local, n.mmax_local, 2), device=self.state.device)
        eta.normal_(mean=0.0, std=1.0, generator=self.rng)
        eta = n.sigma_l * eta
        if not replace_state:
            new = n.phi * self.state + eta
        else:
            new = eta
            new[:, 0, ...] = new[:, 0, ...] / torch.sqrt(1.0 - n.phi**2)
        self.state.copy_(new)

    def forward(self):
        n = self.n
        c = torch.complex(self.state[..., 0], self.state[..., 1])
        B = c.shape[0]
        c = c.reshape(B, n.num_time_steps * n.num_channels, n.lmax_local, n.mmax_local)
        with torch.autocast("cuda", enabled=False):
            eta = n.isht(c)
        return eta.reshape(B, n.num_time_steps, n.num_channels, n.nlat_local, n.nlon_local)


def time_ms(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / iters


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--precision", default="fp32", choices=["fp32", "tf32"])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("noise_bench.py needs a CUDA device")
    info = device_info()
    print(f"device: {info['device']} | nvidia-smi name, power.limit, clocks.max.sm: {info['nvidia_smi']}")
    results = []
    for B in args.batch:
        n = mn.DiffusionNoiseS2((721, 1440), B, 8, kT=SHIPPED_KT, lambd=1.0, seed=333).cuda()
        n.isht.precision = args.precision
        ref = MakaniPath(n, 333)
        cases = {
            "update": (lambda: n.update(), lambda: ref.update()),
            "update(replace_state=True)": (lambda: n.update(replace_state=True), lambda: ref.update(replace_state=True)),
            "forward": (lambda: n(), lambda: ref.forward()),
        }
        n.update(replace_state=True)
        ref.update(replace_state=True)
        for name, (lib_fn, ref_fn) in cases.items():
            for _ in range(args.warmup):
                lib_fn()
                ref_fn()
            t_lib, t_ref = [], []
            for _ in range(args.repeats):
                t_lib.append(time_ms(lib_fn, args.iters))
                t_ref.append(time_ms(ref_fn, args.iters))
            # one more call of each from equal generator positions (both paths have drawn equally often), then compare
            same_state = torch.equal(n.state, ref.state)
            if name == "forward":
                same_out = torch.equal(n(), ref.forward())
            else:
                lib_fn()
                ref_fn()
                same_out = torch.equal(n.state, ref.state)
            row = dict(batch=B, op=name, precision=args.precision, library_ms=sorted(t_lib)[len(t_lib) // 2],
                       makani_ms=sorted(t_ref)[len(t_ref) // 2], bit_identical=bool(same_state and same_out))
            row["speedup"] = row["makani_ms"] / row["library_ms"]
            print(f"B={B:<2d} {name:<28s} library {row['library_ms']:8.3f} ms   makani formulation {row['makani_ms']:8.3f} ms   "
                  f"x{row['speedup']:.2f}   outputs bit-identical: {row['bit_identical']}")
            results.append(row)
        del n, ref
        torch.cuda.empty_cache()
    print(json.dumps({"noise_bench": results, **info}))
    if not all(r["bit_identical"] for r in results):
        raise SystemExit("library and makani formulation disagree")


if __name__ == "__main__":
    main()

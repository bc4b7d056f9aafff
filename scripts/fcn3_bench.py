#!/usr/bin/env python
"""Training step of FourCastNet 3 (makani_b200.fcn3.AtmoSphericNeuralOperatorNet on the CUDA kernels) at the shipped shape on one GPU: BASELINE
configs[4], fcn3_sc2_edim45_layers10 (config/fourcastnet3.yaml).

  721 x 1440 equiangular data grid -> 360 x 720 Legendre-Gauss model grid (scale factor 2), morlet (3, 3) "mean", 10 blocks with
  sfno_block_frequency 5 (blocks 0 and 5 global dhconv, the other 8 local DISCO), serial MLPs of ratio 2, gelu, layer scale, no norm, no bias,
  no big skip, water clamp on.
  72 channels (13 pressure levels x u, v, z, t, q + 7 surface variables) and 12 auxiliary channels, as makani's preprocessor appends them for
  this config (utils/features.py get_auxiliary_channels): zenith angle 1 (add_zenith), the concatenated diffusion noise 8 (input_noise
  n_channels 8, mode "concatenate"), orography 1 (add_orography) and the land-sea mask 2 (add_landmask, "floor" preprocessing: land and sea
  fractions).  84 input channels; processor width 13 x 45 + 56 + 36 = 677 channels.

Per multistep count it prints one JSON line: ms per forward + backward step (CUDA events over --steps steps after --warmup, median and min),
samples/s at batch 1 per GPU, peak memory; bf16 autocast, loss = mean squared error summed over the rollout steps, the prediction with the
auxiliary channels appended being the next step's input.  A configuration that does not fit in memory reports "out of memory" and the script
goes on.  For one step it also prints the per-stage split from CUDA events, forward and backward: encoders (atmosphere, surface, auxiliary),
local blocks, global blocks, decoders (backward boundaries are recorded from gradient hooks on the stage boundaries).  Device name, power limit
and clocks are read in the same run.

    python scripts/fcn3_bench.py [--steps 10] [--warmup 3] [--multistep 1,2] [--checkpointing 0] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from makani_b200.fcn3 import AtmoSphericNeuralOperatorNet  # noqa: E402

LEVELS = (50, 100, 150, 200, 250, 300, 400, 500, 600, 700, 850, 925, 1000)
CHANNELS = ["u10m", "v10m", "u100m", "v100m", "t2m", "msl", "tcwv"] + [f"{v}{p}" for v in "uvztq" for p in LEVELS]
AUX = ["xzen"] + [f"xnoise{i}" for i in range(8)] + ["xoro", "xlsml", "xlsms"]
CONFIG = dict(model_grid_type="equiangular", sht_grid_type="legendre-gauss", inp_shape=(721, 1440), out_shape=(721, 1440), scale_factor=2,
              kernel_shape=[3, 3], filter_basis_type="morlet", filter_basis_norm_mode="mean", channel_names=CHANNELS, aux_channel_names=AUX,
              atmo_embed_dim=45, surf_embed_dim=56, aux_embed_dim=36, encoder_mlp=False, num_layers=10, num_groups=1, sfno_block_frequency=5,
              normalization_layer="none", hard_thresholding_fraction=1.0, use_mlp=True, mlp_mode="serial", mlp_ratio=2, activation_function="gelu",
              pos_embed=False, big_skip=False, bias=False, clamp_water=True)


def device_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"unavailable: {e}"
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out}


def rollout_loss(net, x, targets):
    n_out = len(CHANNELS)
    loss, inp = 0.0, x
    with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
        for t in targets:
            y = net(inp)
            loss = loss + (y.float() - t).square().mean()
            inp = torch.cat([y.float(), x[:, n_out:]], dim=1)
    return loss


def time_steps(net, x, targets, steps, warmup):
    def step():
        net.zero_grad(set_to_none=True)
        rollout_loss(net, x, targets).backward()

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return times, torch.cuda.max_memory_allocated() / 2**30


def stage_split(net, x, target, reps):
    """forward and backward ms per stage of one step, through the network's public stages (encode_auxiliary_channels, encode, blocks, decode,
    clamp_water_channels) in forward's order; backward boundaries from gradient hooks"""
    names = ["encoders"] + [f"block{i}" for i in range(len(net.blocks))] + ["decoders"]
    fwd = {n: [] for n in names}
    bwd = {n: [] for n in names}
    for _ in range(reps):
        net.zero_grad(set_to_none=True)
        ev = {}

        def mark(key):
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            ev[key] = e

        def hook(key):
            def h(grad):
                mark(key)
            return h

        with torch.autocast(device_type="cuda", dtype=torch.bfloat16):
            mark("f_start")
            x_aux = net.encode_auxiliary_channels(x)
            h = net.pos_drop(net.encode(x))
            mark("f_encoders")
            h.register_hook(hook("b_encoders"))      # the encoders' backward starts when the first block has returned this gradient
            for i, blk in enumerate(net.blocks):
                h = blk(torch.cat([h, x_aux], dim=-3))
                mark(f"f_block{i}")
                h.register_hook(hook(f"b_block{i}"))
            y = net.clamp_water_channels(net.decode(h))
            mark("f_decoders")
            loss = (y.float() - target).square().mean()
        mark("b_start")
        loss.backward()
        mark("b_end")
        torch.cuda.synchronize()
        prev = "f_start"
        for n in names:
            fwd[n].append(ev[prev].elapsed_time(ev[f"f_{n}"]))
            prev = f"f_{n}"
        # backward runs decoders -> block9 ... block0 -> encoders; b_<stage> marks the gradient reaching the stage's output
        order = ["decoders"] + [f"block{i}" for i in reversed(range(len(net.blocks)))] + ["encoders"]
        ends = {"decoders": f"b_block{len(net.blocks) - 1}", "encoders": "b_end"}
        for i in range(len(net.blocks)):
            ends[f"block{i}"] = f"b_block{i - 1}" if i > 0 else "b_encoders"
        start = "b_start"
        for n in order:
            bwd[n].append(ev[start].elapsed_time(ev[ends[n]]))
            start = ends[n]
    med = {n: (statistics.median(fwd[n]), statistics.median(bwd[n])) for n in names}
    glob = [f"block{i}" for i, b in enumerate(net.blocks) if hasattr(b, "global_conv")]
    loc = [f"block{i}" for i, b in enumerate(net.blocks) if hasattr(b, "local_conv")]
    out = {}
    for label, group in (("encoders", ["encoders"]), ("local_blocks", loc), ("global_blocks", glob), ("decoders", ["decoders"])):
        f, b = sum(med[n][0] for n in group), sum(med[n][1] for n in group)
        out[label] = {"n": len(group), "fwd_ms": round(f, 2), "bwd_ms": round(b, 2), "total_ms": round(f + b, 2)}
    out["sum_ms"] = round(sum(v["total_ms"] for v in out.values()), 2)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--multistep", default="1,2")
    ap.add_argument("--checkpointing", default="0", help="comma-separated checkpointing levels to time (0: none, 3: every block)")
    ap.add_argument("--split-reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fcn3_bench.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = True
    info = device_info()
    lines = [{"device_info": info}]
    print(json.dumps(lines[0]), flush=True)
    torch.manual_seed(0)
    x = torch.randn(1, len(CHANNELS) + len(AUX), *CONFIG["inp_shape"], device="cuda")
    for level in [int(v) for v in args.checkpointing.split(",")]:
        net = AtmoSphericNeuralOperatorNet(**CONFIG, checkpointing_level=level).cuda()
        nparams = sum(p.numel() for p in net.parameters())
        for ms in [int(v) for v in args.multistep.split(",")]:
            targets = torch.randn(ms, 1, len(CHANNELS), *CONFIG["out_shape"], device="cuda")
            rec = {"workload": "fcn3_sc2_edim45_layers10", "multistep": ms, "checkpointing_level": level, "batch_per_gpu": 1, "autocast": "bf16",
                   "params": nparams, "device": info["device"]}
            try:
                times, peak = time_steps(net, x, targets, args.steps, args.warmup)
                med = statistics.median(times)
                rec.update(ms_per_step=round(med, 2), ms_min=round(min(times), 2), samples_per_s=round(1000.0 / med, 3), peak_mem_gib=round(peak, 2),
                           steps=args.steps, warmup=args.warmup)
            except torch.OutOfMemoryError as e:
                rec.update(error="out of memory", detail=str(e).split("\n")[0][:200])
            del targets
            net.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        if level == 0:
            try:
                split = stage_split(net, x, torch.randn(1, len(CHANNELS), *CONFIG["out_shape"], device="cuda"), args.split_reps)
                rec = {"stage_split_ms": split, "multistep": 1, "reps": args.split_reps}
            except torch.OutOfMemoryError as e:
                rec = {"stage_split_ms": None, "error": "out of memory", "detail": str(e).split("\n")[0][:200]}
            print(json.dumps(rec), flush=True)
            lines.append(rec)
        del net
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()

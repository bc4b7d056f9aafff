#!/usr/bin/env python
"""Training step of FourCastNet 3 under h x w spatial model parallelism (makani_b200.fcn3 on the grid of makani_b200.distributed), NCCL, one GPU
per rank, at the shipped shape of scripts/fcn3_bench.py: BASELINE configs[4], fcn3_sc2_edim45_layers10, 721 x 1440, batch 1, bf16 autocast,
TF32 on.

Launch with torchrun, one process per GPU:

    torchrun --nproc-per-node 8 scripts/fcn3_dist_bench.py [--grids 2x1,2x2,2x4] [--multistep 1,2] [--checkpointing 0,2] [--steps 5] [--warmup 2]

A grid of h x w ranks runs on the first h * w ranks (rank = ih * w + iw); the other ranks wait.  A grid that needs more GPUs than there are ranks
is reported as not measured: ranks never share a GPU here.  Each step is forward + backward of the rollout loss of scripts/fcn3_bench.py on this
rank's shard, then reduce_shared_gradients.  Per grid, multistep count and checkpointing level rank 0 prints one JSON line: each rank's median
and minimum step time (CUDA events), the maximum over ranks of the medians, and each rank's max_memory_allocated; a rank that runs out of memory
reports it.  Device name and power limit are read in the same run.  Started without torchrun it reports every grid as not measured.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import makani_b200.distributed as mbd  # noqa: E402
from fcn3_bench import AUX, CHANNELS, CONFIG, device_info, rollout_loss  # noqa: E402
from makani_b200.fcn3 import AtmoSphericNeuralOperatorNet  # noqa: E402


def make_grid(h, w):
    """the polar and azimuth groups of the first h * w ranks; every rank creates every group in the same order"""
    rank = dist.get_rank()
    mine = (None, None)
    h_groups = [dist.new_group([ih * w + iw for ih in range(h)]) for iw in range(w)]
    w_groups = [dist.new_group([ih * w + iw for iw in range(w)]) for ih in range(h)]
    if rank < h * w:
        ih, iw = rank // w, rank % w
        mine = (h_groups[iw] if h > 1 else None, w_groups[ih] if w > 1 else None)
    return mine


def run(h, w, level, multistep, steps, warmup):
    """this rank's step times and peak memory on an h x w grid (rank < h * w)"""
    rank = dist.get_rank()
    ih, iw = rank // w, rank % w
    lat = mbd.compute_split_shapes(CONFIG["inp_shape"][0], h)[ih]
    lon = mbd.compute_split_shapes(CONFIG["inp_shape"][1], w)[iw]
    torch.manual_seed(rank)
    net = AtmoSphericNeuralOperatorNet(**CONFIG, checkpointing_level=level).cuda()
    mbd.sync_shared_params(net)
    x = torch.randn(1, len(CHANNELS) + len(AUX), lat, lon, device="cuda")
    targets = torch.randn(multistep, 1, len(CHANNELS), lat, lon, device="cuda")

    def step():
        net.zero_grad(set_to_none=True)
        rollout_loss(net, x, targets).backward()
        mbd.reduce_shared_gradients(net)

    try:
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
        return {"ms_median": round(statistics.median(times), 2), "ms_min": round(min(times), 2),
                "max_memory_allocated_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2)}
    except torch.OutOfMemoryError as e:
        return {"error": "out of memory", "detail": str(e).split("\n")[0][:200]}
    finally:
        del net, x, targets
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--grids", default="2x1,2x2,2x4")
    ap.add_argument("--multistep", default="1,2")
    ap.add_argument("--checkpointing", default="0,2")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    grids = [tuple(int(v) for v in g.split("x")) for g in args.grids.split(",")]
    if "RANK" not in os.environ:
        for h, w in grids:
            print(json.dumps({"grid": f"{h}x{w}", "measured": False, "reason": "not started under torchrun"}), flush=True)
        return
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, world = dist.get_rank(), dist.get_world_size()
    if int(os.environ.get("LOCAL_WORLD_SIZE", world)) > torch.cuda.device_count():
        sys.exit(f"{os.environ['LOCAL_WORLD_SIZE']} ranks per node but {torch.cuda.device_count()} GPUs: ranks must not share a GPU")
    torch.backends.cuda.matmul.allow_tf32 = True
    infos = [None] * world
    dist.all_gather_object(infos, device_info())
    if rank == 0:
        print(json.dumps({"device_info": infos, "ranks": world}), flush=True)
    for h, w in grids:
        if h * w > world:
            if rank == 0:
                print(json.dumps({"grid": f"{h}x{w}", "measured": False, "reason": f"needs {h * w} GPUs, {world} ranks"}), flush=True)
            continue
        polar, azimuth = make_grid(h, w)
        for level in [int(v) for v in args.checkpointing.split(",")]:
            for ms in [int(v) for v in args.multistep.split(",")]:
                res = None
                if rank < h * w:
                    mbd.init(polar, azimuth)
                    res = run(h, w, level, ms, args.steps, args.warmup)
                    mbd.finalize()
                per_rank = [None] * world
                dist.all_gather_object(per_rank, res)
                if rank == 0:
                    per_rank = per_rank[: h * w]
                    ok = all("ms_median" in r for r in per_rank)
                    print(json.dumps({"workload": "fcn3_sc2_edim45_layers10", "grid": f"{h}x{w}", "multistep": ms, "checkpointing_level": level,
                                      "batch": 1, "autocast": "bf16", "measured": True, "steps": args.steps, "warmup": args.warmup,
                                      "ms_median_max_over_ranks": max(r["ms_median"] for r in per_rank) if ok else None,
                                      "per_rank": per_rank}), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

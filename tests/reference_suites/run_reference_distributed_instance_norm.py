#!/usr/bin/env python
"""Run makani's own distributed instance-norm test, `TestDistributedLayers.test_distributed_instance_norm_2d` (tests/distributed/
tests_distributed_layers.py of a makani checkout: 256 x 512 with B = 32, C = 8 and 181 x 360 with B = 1, C = 10, affine and not, tolerance 1e-4),
unmodified on CPU / gloo at h x w = 2x1, 1x2, 2x2 and 4x2, after makani_b200.compat.patch_makani_instance_norm().

The test builds torch's nn.InstanceNorm2d as the serial layer and makani's DistributedInstanceNorm2d -- which the patch has pointed at
makani_b200.distributed's -- wraps the distributed one in makani's gradient-reduction hooks when it is affine (DDP over the spatial group, fed by
the `is_shared_mp` tags), runs forward and backward serially on the full input and distributed on the shards, and compares the gathered output,
the gathered input gradient and, when affine, the reduced weight and bias gradients of every rank against the serial run.

What is real: makani's test body, its split / gather helpers, its gradient-reduction hooks (makani/mpu/mappings.py), torch.distributed over gloo,
torch's serial InstanceNorm2d, and the distributed class's choreography: the exchange of the global point count, the all-gathers of the per-rank
statistics and sums and the autograd Function.  What stands in:
  * the distributed class's per-rank stages: the fp64 oracle's with every latitude weight 1 (oracle/makani_norm_oracle.py OracleStages,
    `set_norm_local_ops`); the CUDA stages are pinned against fp64 and against virtual ranks by tests/test_gpu_distributed_instance_norm.py;
  * the environment of run_reference_distributed.py: its h x w stand-in for `makani.utils.comm`, the oracle posed as `torch_harmonics`, DDP
    without device_ids on CPU, all_gather of shards of different sizes on gloo, and a per-call CPU random stream (the test draws its full-size
    input after building the sharded module).

    python tests/reference_suites/run_reference_distributed_instance_norm.py [H W]     (default: all grids)
    python tests/reference_suites/run_reference_distributed_instance_norm.py --report  (all grids; rewrites report_distributed_instance_norm.txt)
"""
import importlib
import os
import socket
import sys
import time
import types
import unittest

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

GRIDS = [(2, 1), (1, 2), (2, 2), (4, 2)]


def install(h, w):
    """the environment of the test on this rank; returns (test module, count of distributed norms built)"""
    import run_reference_distributed as RD
    import run_reference_tests as R

    R.install_environment()
    comm = RD.make_comm(h, w)
    sys.modules["makani.utils.comm"] = comm
    sys.modules["makani.utils"].comm = comm

    import makani.mpu.layer_norm  # noqa: F401  (imported before the patch, as a network module would have)

    import makani_b200.compat as compat
    import makani_b200.distributed as mbd
    from oracle.makani_norm_oracle import OracleStages

    compat.patch_makani_instance_norm()
    built = {"dist": 0}

    def stages(layer):
        built["dist"] += 1
        return OracleStages()

    mbd.set_norm_local_ops(stages)

    import makani.mpu.mappings as mappings
    from torch.nn.parallel import DistributedDataParallel as RealDDP

    def ddp_cpu_ok(module, device_ids=None, output_device=None, **kw):
        if device_ids and torch.device(device_ids[0]).type == "cpu":
            device_ids, output_device = None, None
        return RealDDP(module, device_ids=device_ids, output_device=output_device, **kw)

    mappings.DistributedDataParallel = ddp_cpu_ok
    real_all_gather = dist.all_gather

    def all_gather_uneven_ok(tensor_list, tensor, group=None, async_op=False):
        if all(t.shape == tensor.shape for t in tensor_list):
            return real_all_gather(tensor_list, tensor, group=group, async_op=async_op)
        grank = dist.get_rank(group=group)
        for i, t in enumerate(tensor_list):
            buf = tensor.contiguous() if i == grank else t
            dist.broadcast(buf, src=dist.get_global_rank(group, i) if group is not None else i, group=group)
            if i == grank and t.data_ptr() != tensor.data_ptr():
                t.copy_(tensor)
        return None

    dist.all_gather = all_gather_uneven_ok
    rng = {"seed": 0, "calls": 0}
    real_seed, real_randn, real_randn_like = torch.manual_seed, torch.randn, torch.randn_like

    def manual_seed(seed):
        rng["seed"], rng["calls"] = int(seed), 0
        return real_seed(seed)

    def stream():
        rng["calls"] += 1
        return torch.Generator().manual_seed(1000003 * rng["seed"] + rng["calls"])

    def randn(*size, **kw):
        if kw.get("generator") is None and torch.device(kw.get("device") or "cpu").type == "cpu":
            kw["generator"] = stream()
        return real_randn(*size, **kw)

    def randn_like(t, **kw):
        if t.device.type == "cpu":
            return real_randn(t.shape, dtype=kw.get("dtype", t.dtype), generator=stream())
        return real_randn_like(t, **kw)

    torch.manual_seed, torch.randn, torch.randn_like = manual_seed, randn, randn_like
    ns = types.ModuleType("tests.distributed")
    ns.__path__ = [f"{REF}/tests/distributed"]
    sys.modules["tests.distributed"] = ns
    M = importlib.import_module("tests.distributed.tests_distributed_layers")
    assert M.DistributedInstanceNorm2d is mbd.DistributedInstanceNorm2d
    return M, built


def worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GRID_H=str(h), GRID_W=str(w), RANK=str(rank), WORLD_SIZE=str(world))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        M, built = install(h, w)
        checked = []
        real_compare = M.compare_tensors

        def compare_recorded(msg, *a, **k):
            ok = real_compare(msg, *a, **k)
            checked.append((msg, bool(ok)))
            return ok

        M.compare_tensors = compare_recorded
        Case = M.TestDistributedLayers
        names = [n for n in unittest.defaultTestLoader.getTestCaseNames(Case) if n.startswith("test_distributed_instance_norm_2d")]
        Case.setUpClass()
        r = unittest.TextTestRunner(verbosity=0, stream=open(os.devnull, "w")).run(unittest.TestSuite(Case(n) for n in names))
        msgs = [t.id().split(".")[-1] + ": " + tb.strip().splitlines()[-1][:600] for t, tb in r.failures + r.errors]
        q.put((rank, r.testsRun, len(r.failures) + len(r.errors), checked, msgs, built["dist"]))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        import traceback

        q.put((rank, 0, 1, [], [traceback.format_exc()[-1500:]], 0))


def run(h, w):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    world = h * w
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, world, port, h, w, q)) for r in range(world)]
    for p in procs:
        p.start()
    out = [q.get(timeout=1500) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    return sorted(out, key=lambda o: o[0])


def main():
    if not os.path.isdir(f"{REF}/tests/distributed"):
        print("reference tree not mounted: nothing to run")
        return 0
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    grids = [(int(args[0]), int(args[1]))] if len(args) == 2 else GRIDS
    lines = ["makani's TestDistributedLayers.test_distributed_instance_norm_2d (4 cases), unmodified, CPU / gloo, after",
             "makani_b200.compat.patch_makani_instance_norm(); per grid the tests run and the comparisons of rank 0 (output, input gradients,",
             "weight and bias gradients of every rank in the affine cases), the failures of every rank, and the distributed norms built on rank 0."]
    bad = 0
    for h, w in grids:
        t0 = time.time()
        res = run(h, w)
        failed = sum(o[2] for o in res) + sum(1 for o in res if o[1] == 0)
        kinds = {"output": 0, "input gradients": 0, "weight gradient": 0, "bias gradient": 0}
        for msg, _ in res[0][3]:
            for k in kinds:
                if msg.startswith(k):
                    kinds[k] += 1
        n_bad_cmp = sum(1 for o in res for _, ok in o[3] if not ok)
        ok = (failed == 0 and n_bad_cmp == 0 and res[0][1] == 4 and kinds["output"] == kinds["input gradients"] == 4
              and kinds["weight gradient"] == kinds["bias gradient"] == 2 * h * w and res[0][5] == 4)
        bad += not ok
        lines.append(f"grid {h}x{w} ({h * w} ranks, {time.time() - t0:.0f} s): {'OK' if ok else 'FAILED'}")
        lines.append(f"    tests run on rank 0: {res[0][1]}; compared on rank 0: output {kinds['output']}, input gradients {kinds['input gradients']}, "
                     f"weight gradients {kinds['weight gradient']}, bias gradients {kinds['bias gradient']}; failing comparisons on all ranks: {n_bad_cmp}")
        lines.append(f"    built on rank 0: {res[0][5]} DistributedInstanceNorm2d (per-rank stages on the oracle)")
        for o in res:
            for m in o[4][:3]:
                lines.append(f"    rank {o[0]}: {m}")
        print("\n".join(lines[-3:]), flush=True)
    lines.append(f"TOTAL: {len(grids)} grids, {bad} failing")
    print(lines[-1])
    if "--report" in sys.argv:
        with open(os.path.join(HERE, "report_distributed_instance_norm.txt"), "w") as f:
            f.write("python tests/reference_suites/run_reference_distributed_instance_norm.py --report\n" + "\n".join(lines) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""Run makani's own distributed model test, `TestDistributedModel.test_distributed_model_fwd_bwd("FCN3", 1e-4)`
(tests/distributed/tests_distributed_model.py of a makani checkout), unmodified on CPU / gloo at h x w = 2x1, 1x2, 2x2 and 4x2.

The test builds FCN3 serially, runs forward and backward on the full input, saves a flexible checkpoint, then initialises the h x w grid,
builds the same network again -- now with torch_harmonics.distributed.DistributedDiscreteContinuousConvS2 / DistributedResampleS2 /
DistributedRealSHT, which are makani_b200.distributed's -- restores the checkpoint into it, runs forward and backward on the shards and
compares the gathered output, the loss, the gathered input gradient and every gathered weight gradient against the serial run at 1e-4.

What is real: makani's test body, its split / gather helpers, model registry, FCN3, checkpoint save / restore and gathered state dicts, its
gradient-reduction hooks (makani/mpu/mappings.py), torch.distributed over gloo, and the choreography and autograd of makani_b200.distributed
(transposes, the DISCO halo and window plans, the resampling transposes).  What stands in:
  * the per-rank stages: the oracle's arithmetic (DISCO window contraction / adjoint and resampling from tests/test_distributed_disco_cpu.py,
    the SHT's FFT / Legendre stages in fp32 as in run_reference_distributed.py); the CUDA stages are pinned against the single-GPU kernels by
    tests/test_gpu_distributed_disco.py;
  * the serial network's torch_harmonics.DiscreteContinuousConvS2 / ResampleS2 / RealSHT / InverseRealSHT: the oracles;
  * `mpi4py`: a facade over torch.distributed (COMM_WORLD.Dup, Get_rank, Get_size, bcast, Barrier, Free);
  * `makani.utils.comm`: run_reference_distributed.py's h x w stand-in (the real one needs physicsnemo's DistributedManager);
  * physicsnemo, `parameterized`: the stubs of build_reference_sfno.py / run_reference_tests.py;
  * empty modules for the packages makani imports but this test never calls: wandb, h5py, zarr, ruamel.yaml, moviepy, more_itertools;
  * gloo stand-ins for two calls NCCL accepts and gloo does not, as in run_reference_distributed.py: DDP without device_ids on CPU, and
    all_gather of shards of different sizes;
  * the model registry's "FCN3" entry point, taken from makani's pyproject.toml (makani is not pip-installed here);
  * `filter_basis_type="morlet"` injected into the test's default parameters: FCN3's constructor defaults to "harmonic", which this package
    does not build.

    python tests/reference_suites/run_reference_distributed_fcn3.py [H W]     (default: all grids)
    python tests/reference_suites/run_reference_distributed_fcn3.py --report  (all grids; rewrites report_distributed_fcn3.txt)
"""
import importlib
import importlib.abc
import importlib.machinery
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

GRIDS = [(2, 1), (1, 2), (2, 2), (4, 2)]
BUILT = {}      # distributed DISCO convolutions / resamplings constructed on this rank
EMPTY = ("wandb", "h5py", "zarr", "ruamel", "moviepy", "more_itertools")


class _Anything:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return None


class _EmptyPackages(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    """empty modules (any attribute is a do-nothing class) for packages makani imports but the test never calls"""

    def find_spec(self, name, path, target=None):
        if name.split(".")[0] in EMPTY:
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []

        def getattr_(a):
            if a.startswith("__"):
                raise AttributeError(a)
            return _Anything
        m.__getattr__ = getattr_
        return m

    def exec_module(self, m):
        pass


def mpi4py_facade():
    """mpi4py.MPI.COMM_WORLD over the default torch.distributed group"""
    class Comm:
        def Dup(self):
            return Comm()

        def Get_rank(self):
            return dist.get_rank()

        def Get_size(self):
            return dist.get_world_size()

        def bcast(self, obj, root=0):
            box = [obj]
            dist.broadcast_object_list(box, src=root)
            return box[0]

        def Barrier(self):
            dist.barrier()

        def Free(self):
            pass

    mpi = types.ModuleType("mpi4py.MPI")
    mpi.COMM_WORLD = Comm()
    pkg = types.ModuleType("mpi4py")
    pkg.MPI = mpi
    sys.modules.update({"mpi4py": pkg, "mpi4py.MPI": mpi})


def install(h, w):
    """the environment of the test on this rank; returns the test module"""
    import build_reference_sfno as S
    import run_reference_distributed as RD
    import run_reference_tests as R

    R.install_environment()
    S.stub_physicsnemo()
    # makani's real package __init__ files and YParams this time (the model registry and the driver need them): drop the namespace stand-ins
    for k in [k for k in sys.modules if k in ("makani", "tests") or k.startswith(("makani.", "tests."))]:
        del sys.modules[k]
    sys.meta_path.insert(0, _EmptyPackages())
    mpi4py_facade()
    comm = RD.make_comm(h, w)
    comm.cleanup = lambda: None
    sys.modules["makani.utils.comm"] = comm          # before `import makani`, whose package __init__ imports it
    sys.path.insert(0, REF)
    import makani.utils

    makani.utils.comm = comm

    import math

    import numpy as np

    import makani_b200.disco as mbdisco
    import makani_b200.distributed as mbd
    from oracle import makani_disco_oracle as DO
    from oracle import makani_oracle as O
    from oracle import makani_resample_oracle as RO
    from test_distributed_disco_cpu import OracleDiscoLocalOps, OracleResampleLocalOps

    th = sys.modules["torch_harmonics"]
    th.DiscreteContinuousConvS2, th.ResampleS2 = DO.DiscreteContinuousConvS2, RO.ResampleS2
    th.filter_basis = mbdisco
    sys.modules["torch_harmonics.filter_basis"] = mbdisco

    class OracleShtOps:
        """the SHT's four per-rank stages with torch-harmonics' dtype behaviour (fp32 tables, fp32 in -> complex64 out)"""

        def __init__(self, t):
            self.t = t
            theta, wq = O.precompute_latitudes(t.nlat, t.grid)
            P = O.legpoly(t.mmax, t.lmax, np.cos(theta), csphase=t.csphase)
            self.P = torch.from_numpy(P[t.m_offset:t.m_offset + t.mmax_local]).float()
            self.w_local = torch.from_numpy(wq[t.lat_offset:t.lat_offset + t.nlat_local]).float()

        def fft(self, x):
            X = 2.0 * math.pi * torch.fft.rfft(x.float(), dim=-1, norm="forward")[..., :self.t.mmax]
            return X * self.w_local[:, None]

        def legendre(self, xc):
            return torch.einsum("...km,mlk->...lm", xc, self.P.to(xc.dtype))

        def ilegendre(self, xc):
            return torch.einsum("...lm,mlk->...km", xc, self.P.to(xc.dtype))

        def ifft(self, xc, dtype):
            re, im = xc.real, xc.imag.clone()
            im[..., 0] = 0.0
            return torch.fft.irfft(torch.complex(re, im), n=self.t.nlon, dim=-1, norm="forward")

    mbd.set_local_ops(OracleShtOps)
    BUILT.update(disco=0, resample=0)

    def counted(kind, cls):
        def make(layer):
            BUILT[kind] += 1
            return cls(layer)
        return make

    mbd.set_disco_local_ops(counted("disco", OracleDiscoLocalOps))
    mbd.set_resample_local_ops(counted("resample", OracleResampleLocalOps))

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

    ns = types.ModuleType("tests.distributed")
    ns.__path__ = [f"{REF}/tests/distributed"]
    sys.modules["tests.distributed"] = ns
    M = importlib.import_module("tests.distributed.tests_distributed_model")
    real_defaults = M.get_default_parameters

    def defaults_with_morlet():
        params = real_defaults()
        params.filter_basis_type = "morlet"
        return params

    M.get_default_parameters = defaults_with_morlet
    # makani is not pip-installed here: register FCN3's entry point of makani's pyproject.toml as the installed package would
    from importlib.metadata import EntryPoint

    import makani.models.model_registry as registry

    registry._model_registry.setdefault("FCN3", EntryPoint(name="FCN3", value="makani.models.networks.fourcastnet3:AtmoSphericNeuralOperatorNet",
                                                           group="makani.models"))
    return M


def worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), GRID_H=str(h), GRID_W=str(w), RANK=str(rank), WORLD_SIZE=str(world))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        M = install(h, w)
        checked = []
        real_compare = M.compare_tensors

        def compare_recorded(msg, *a, **k):
            ok = real_compare(msg, *a, **k)
            checked.append((msg, bool(ok)))
            return ok

        M.compare_tensors = compare_recorded
        Case = M.TestDistributedModel
        names = [n for n in unittest.defaultTestLoader.getTestCaseNames(Case) if n.startswith("test_distributed_model_fwd_bwd")]
        Case.setUpClass()
        r = unittest.TextTestRunner(verbosity=0, stream=open(os.devnull, "w")).run(unittest.TestSuite(Case(n) for n in names))
        msgs = [t.id().split(".")[-1] + ": " + tb.strip().splitlines()[-1][:600] for t, tb in r.failures + r.errors]
        q.put((rank, r.testsRun, len(r.failures) + len(r.errors), checked, msgs, dict(BUILT)))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        import traceback

        q.put((rank, 0, 1, [], [traceback.format_exc()[-1500:]], {}))


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
    out = [q.get(timeout=3000) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    return sorted(out, key=lambda o: o[0])


def main():
    if not os.path.isdir(f"{REF}/tests/distributed"):
        print("reference tree not mounted: nothing to run")
        return 0
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    grids = [(int(args[0]), int(args[1]))] if len(args) == 2 else GRIDS
    lines = ["makani's TestDistributedModel.test_distributed_model_fwd_bwd(\"FCN3\", 1e-4), unmodified, CPU / gloo; per grid the comparisons",
             "of rank 0 (output, loss, input gradients, one per weight gradient) and the failures of every rank."]
    bad = 0
    for h, w in grids:
        t0 = time.time()
        res = run(h, w)
        failed = sum(o[2] for o in res) + sum(1 for o in res if o[1] == 0)
        checked = res[0][3]
        kinds = {"output": 0, "loss": 0, "input gradients": 0, "weight gradient": 0}
        for msg, _ in checked:
            for k in kinds:
                if msg.startswith(k):
                    kinds[k] += 1
        n_bad_cmp = sum(1 for o in res for _, ok in o[3] if not ok)
        built = res[0][5]
        ok = (failed == 0 and n_bad_cmp == 0 and kinds["output"] == kinds["loss"] == kinds["input gradients"] == 1 and kinds["weight gradient"] > 0
              and built.get("disco", 0) > 0 and built.get("resample", 0) > 0)
        bad += not ok
        lines.append(f"grid {h}x{w} ({h * w} ranks, {time.time() - t0:.0f} s): {'OK' if ok else 'FAILED'}")
        lines.append(f"    compared on rank 0: output {kinds['output']}, loss {kinds['loss']}, input gradients {kinds['input gradients']}, "
                     f"weight gradients {kinds['weight gradient']}; failing comparisons on all ranks: {n_bad_cmp}")
        lines.append(f"    built on rank 0: {built.get('disco', 0)} DistributedDiscreteContinuousConvS2, {built.get('resample', 0)} DistributedResampleS2")
        for o in res:
            for m in o[4][:3]:
                lines.append(f"    rank {o[0]}: {m}")
        print("\n".join(lines[-3:]), flush=True)
    lines.append(f"TOTAL: {len(grids)} grids, {bad} failing")
    print(lines[-1])
    if "--report" in sys.argv:
        with open(os.path.join(HERE, "report_distributed_fcn3.txt"), "w") as f:
            f.write("python tests/reference_suites/run_reference_distributed_fcn3.py --report\n" + "\n".join(lines) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())

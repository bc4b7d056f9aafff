#!/usr/bin/env python
"""makani's own VortDivCRPSLoss and GradientCRPSLoss (makani/utils/losses/crps_loss.py) under h x w spatial model parallelism on CPU / gloo:
each loss is built twice, with spatial_distributed=True on this rank's shard of the inputs -- so that it constructs
torch_harmonics.distributed.DistributedRealVectorSHT / DistributedInverseRealVectorSHT (and DistributedRealSHT), which are
makani_b200.distributed's -- and with spatial_distributed=False on the full tensors.  Loss values and the input gradients (of forecasts and
observations) must agree.

What is real: the reference's loss classes, GridQuadrature and distributed reductions, torch.distributed over gloo, and the all-to-all
choreography + autograd of makani_b200.distributed.  What stands in: the per-rank FFT / Legendre stages are the fp64 oracle's arithmetic
(tests/test_distributed_vector_cpu.py, with torch-harmonics' dtypes at the boundary: fp32 in, complex64 / fp32 out); the serial losses use
the oracle's vector transforms as torch_harmonics; makani.utils.comm is run_reference_distributed.py's h x w stand-in.  Needs a checkout of
makani, as the other runners.

    python tests/reference_suites/run_reference_distributed_vector.py [H W]     (default: grids 2x1, 1x2, 2x2)
    python tests/reference_suites/run_reference_distributed_vector.py --report  (all three grids; rewrites report_distributed_vector.txt)
"""
import os
import socket
import sys
import time

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

GRIDS = [(2, 1), (1, 2), (2, 2)]
CHANNELS = ["u500", "v500", "u850", "v850", "t500"]
# (loss, grid, nlat, nlon, crps_type): odd nlat, so the latitude split is uneven
CASES = [(loss, grid, 33, 64, crps) for loss in ("VortDivCRPSLoss", "GradientCRPSLoss") for grid in ("equiangular", "legendre-gauss")
         for crps in ("skillspread", "cdf")]
RTOL = 1e-4


def worker(rank, world, port, h, w, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        dist.init_process_group("gloo", rank=rank, world_size=world)
        import run_reference_distributed as RD
        import run_reference_tests as R

        R.install_environment()
        comm = RD.make_comm(h, w)
        sys.modules["makani.utils.comm"] = comm
        sys.modules["makani.utils"].comm = comm
        comm.init()
        from oracle import makani_vector_oracle as V

        th = sys.modules["torch_harmonics"]
        th.RealVectorSHT, th.InverseRealVectorSHT = V.RealVectorSHT, V.InverseRealVectorSHT
        import makani_b200.distributed as mbd
        from test_distributed_vector_cpu import OracleVectorLocalOps

        class Fp32BoundaryOps(OracleVectorLocalOps):
            """fp64 arithmetic, torch-harmonics' dtypes at the stage boundaries"""

            def fft(self, x):
                return super().fft(x).to(torch.complex64 if x.dtype != torch.float64 else torch.complex128)

            def ifft(self, xc, dtype):
                return super().ifft(xc, dtype).to(dtype)

            def legendre(self, xc):
                return super().legendre(xc.to(torch.complex128)).to(xc.dtype)

            def ilegendre(self, xc):
                return super().ilegendre(xc).to(xc.dtype)

            def vlegendre(self, xc):
                return super().vlegendre(xc).to(xc.dtype)

            def ivlegendre(self, xc):
                return super().ivlegendre(xc).to(xc.dtype)

        mbd.set_local_ops(Fp32BoundaryOps)
        import importlib

        losses = importlib.import_module("makani.utils.losses.crps_loss")
        ih, iw = comm.get_rank("h"), comm.get_rank("w")

        def shard(t):
            t = torch.split(t, mbd.compute_split_shapes(t.shape[-2], h), dim=-2)[ih]
            return torch.split(t, mbd.compute_split_shapes(t.shape[-1], w), dim=-1)[iw].contiguous()

        def rel(a, b):
            return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()

        results = []
        for name, grid, nlat, nlon, crps in CASES:
            gen = torch.Generator().manual_seed(333)
            B, E, C = 2, 3, len(CHANNELS)
            fc = torch.randn(B, E, C, nlat, nlon, generator=gen) * 2.0 + 1.0
            ob = torch.randn(B, C, nlat, nlon, generator=gen) * 2.0 + 1.0
            kw = dict(img_shape=(nlat, nlon), crop_shape=None, crop_offset=(0, 0), channel_names=CHANNELS, grid_type=grid, crps_type=crps,
                      ensemble_distributed=False)
            cls = getattr(losses, name)
            mbd.finalize()
            dist_fn = cls(spatial_distributed=True, **kw)
            serial_fn = cls(spatial_distributed=False, **kw)
            assert type(dist_fn.isht if name == "VortDivCRPSLoss" else dist_fn.ivsht).__name__.startswith("Distributed")
            fs, os_ = fc.clone().requires_grad_(True), ob.clone().requires_grad_(True)
            ls = serial_fn(fs, os_)
            g = torch.randn(ls.shape, generator=gen)
            ls.backward(g)
            fd, od = shard(fc).requires_grad_(True), shard(ob).requires_grad_(True)
            ld = dist_fn(fd, od)
            ld.backward(g)
            errs = {"loss": rel(ld.detach(), ls.detach()), "d_forecasts": rel(fd.grad, shard(fs.grad)), "d_observations": rel(od.grad, shard(os_.grad))}
            results.append((f"{name} {grid} {nlat}x{nlon} {crps}", errs))
        q.put((rank, results, None))
        dist.barrier()
        dist.destroy_process_group()
    except Exception:  # noqa: BLE001
        import traceback

        q.put((rank, None, traceback.format_exc()[-2000:]))


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
    return sorted(out, key=lambda r: r[0])


def main():
    import run_reference_tests as R

    if not os.path.isdir(R.REF):
        print("reference tree not mounted: nothing to run")
        return 0
    args = [a for a in sys.argv[1:] if a != "--report"]
    grids = [(int(args[0]), int(args[1]))] if len(args) == 2 else GRIDS
    lines, total, bad = [], 0, 0
    for h, w in grids:
        t0 = time.time()
        res = run(h, w)
        ok = True
        worst = {}
        for rank, results, err in res:
            if err is not None:
                ok = False
                lines.append(f"grid {h}x{w} rank {rank}: ERROR\n{err}")
                continue
            for case, errs in results:
                total += 1
                for k, v in errs.items():
                    worst[(case, k)] = max(worst.get((case, k), 0.0), v)
                if max(errs.values()) > RTOL:
                    bad += 1
                    ok = False
        lines.append(f"grid {h}x{w} ({h * w} ranks, {time.time() - t0:.0f} s): {'OK' if ok else 'FAILED'}")
        cases = sorted({c for c, _ in worst})
        for case in cases:
            lines.append(f"    {case}: " + "  ".join(f"{k} {worst[(case, k)]:.1e}" for k in ("loss", "d_forecasts", "d_observations")))
    lines.append(f"TOTAL: {total} rank-cases (loss value, d forecasts, d observations within max-relative {RTOL:g} of the serial loss), "
                 f"{bad} failing")
    print("\n".join(lines))
    if "--report" in sys.argv:
        with open(os.path.join(HERE, "report_distributed_vector.txt"), "w") as f:
            f.write("python tests/reference_suites/run_reference_distributed_vector.py --report   (CPU / gloo)\n"
                    "makani's VortDivCRPSLoss and GradientCRPSLoss, spatial_distributed=True on shards against spatial_distributed=False on the\n"
                    "full tensors; per case the largest |difference| / max|serial| over the ranks.\n" + "\n".join(lines) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""Build makani's own, unmodified DISCO layers -- `DiscreteContinuousEncoder` and `NeuralOperatorBlock(conv_type="local")` of
makani/models/networks/fourcastnet3.py and snonet.py -- with the settings FCN3 ships (basis "morlet", kernel (3, 3), norm "mean";
config/fourcastnet3.yaml) on a scaled-down version of its 721 x 1440 equiangular -> 360 x 720 Legendre-Gauss geometry.

Each layer is built twice in one process, with the same seed:
  (a) on the oracle's DiscreteContinuousConvS2 (oracle/makani_disco_oracle.py) posed as torch_harmonics.DiscreteContinuousConvS2 -> a CPU
      forward and backward run, and their outputs must be finite and of the right shape;
  (b) on makani_b200's DiscreteContinuousConvS2 (what compat.install_torch_harmonics_shim installs) -> construction only (its kernels need a GPU).
Parameter names, shapes, dtypes, values and the model-parallel tags (`is_shared_mp`, `sharded_dims_mp`) must be identical, and neither state dict
may hold psi.  The environment is run_reference_tests.py's (the oracle posed as torch_harmonics, the reference's modules imported unmodified
from where they lie) plus build_reference_sfno.py's physicsnemo stub.

    python tests/reference_suites/run_reference_disco.py            # one line per layer, exit code 1 on any failure
    python tests/reference_suites/run_reference_disco.py --report   # also rewrites tests/reference_suites/report_disco.txt

Only runs where a checkout of makani is mounted; tests/test_reference_disco_suites.py checks the committed report.
"""
import importlib
import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_reference_sfno as S  # noqa: E402
import run_reference_tests as base  # noqa: E402

# 721 x 1440 -> 360 x 720 scaled by 1/15 (in 49 x 96 equiangular, model 24 x 48 Legendre-Gauss); FCN3's settings
IN_SHAPE, MODEL_SHAPE, CIN, EMBED = (49, 96), (24, 48), 6, 10
SETTINGS = dict(kernel_shape=(3, 3), basis_type="morlet", basis_norm_mode="mean")


def describe(net):
    return {name: (tuple(p.shape), str(p.dtype), getattr(p, "is_shared_mp", None), getattr(p, "sharded_dims_mp", None))
            for name, p in net.named_parameters()}


def layers(M, O):
    """(label, constructor) of the DISCO layers of network module M"""
    fwd = O.RealSHT(*MODEL_SHAPE, grid="legendre-gauss")
    fwd.grid = "legendre-gauss"
    inv = O.InverseRealSHT(*MODEL_SHAPE, grid="legendre-gauss")
    inv.grid = "legendre-gauss"
    out = [("DiscreteContinuousEncoder", lambda: M.DiscreteContinuousEncoder(
        inp_shape=IN_SHAPE, out_shape=MODEL_SHAPE, grid_in="equiangular", grid_out="legendre-gauss", inp_chans=CIN, out_chans=EMBED,
        groups=math.gcd(CIN, EMBED), bias=False, use_mlp=True, **SETTINGS), (1, CIN, *IN_SHAPE))]
    out.append(("NeuralOperatorBlock(local)", lambda: M.NeuralOperatorBlock(fwd, inv, EMBED, EMBED, conv_type="local", use_mlp=True, **SETTINGS),
                (1, EMBED, *MODEL_SHAPE)))
    return out


def run():
    """-> list of (network module, layer, [problems], note)"""
    base.install_environment()
    S.stub_physicsnemo()
    from oracle import makani_disco_oracle as DO
    from oracle import makani_oracle as O

    import makani_b200.disco as mbdisco

    th = sys.modules["torch_harmonics"]
    th.filter_basis = mbdisco     # get_filter_basis (host-only)
    sys.modules["torch_harmonics.filter_basis"] = mbdisco
    sys.modules["torch_harmonics.distributed"].DistributedDiscreteContinuousConvS2 = mbdisco.DistributedDiscreteContinuousConvS2
    results = []
    for modname in ("makani.models.networks.fourcastnet3", "makani.models.networks.snonet"):
        try:
            M = importlib.import_module(modname)
        except Exception as e:  # noqa: BLE001
            results.append((modname, "import", [f"{type(e).__name__}: {e}"[:200]], ""))
            continue
        for label, make, xshape in layers(M, O):
            problems = []
            try:
                th.DiscreteContinuousConvS2 = DO.DiscreteContinuousConvS2
                torch.manual_seed(17)
                a = make()
                th.DiscreteContinuousConvS2 = mbdisco.DiscreteContinuousConvS2
                torch.manual_seed(17)
                b = make()
                da, db = describe(a), describe(b)
                if da != db:
                    problems.append(f"parameters differ: oracle {da} product {db}")
                for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
                    if not torch.equal(pa.detach().double(), pb.detach().double()):
                        problems.append(f"initial value of {n} differs")
                for net, who in ((a, "oracle"), (b, "product")):
                    if any("psi" in k for k in net.state_dict()):
                        problems.append(f"{who} state dict holds psi")
                convs = [m for m in b.modules() if isinstance(m, mbdisco.DiscreteContinuousConvS2)]
                if len(convs) != 1:
                    problems.append(f"{len(convs)} product DISCO convolutions built, expected 1")
                a = a.double()
                x = torch.randn(*xshape, dtype=torch.float64, requires_grad=True)
                y = a(x)
                y = y[0] if isinstance(y, tuple) else y
                y.square().sum().backward()
                grads = [p.grad for p in a.parameters() if p.requires_grad]
                if not torch.isfinite(y).all() or not torch.isfinite(x.grad).all() or any(g is None or not torch.isfinite(g).all() for g in grads):
                    problems.append("non-finite forward / backward")
                note = f"{len(da)} parameters, conv weight {tuple(convs[0].weight.shape) if convs else None}, y {tuple(y.shape)}"
            except Exception as e:  # noqa: BLE001
                problems.append(f"{type(e).__name__}: {e}"[:200])
                note = ""
            results.append((modname, label, problems, note))
    return results


def main():
    if not os.path.isdir(base.REF):
        print("reference tree not mounted: nothing to run")
        return 0
    results = run()
    lines = []
    for modname, label, problems, note in results:
        lines.append(f"{modname}.{label}: {'ok' if not problems else 'FAILED'}  {note}")
        lines += ["    " + p for p in problems]
    bad = sum(1 for r in results if r[2])
    lines.append(f"TOTAL: {len(results)} layers built on the oracle and on makani_b200 as torch_harmonics.DiscreteContinuousConvS2, {bad} failing")
    print("\n".join(lines))
    if "--report" in sys.argv:
        with open(os.path.join(HERE, "report_disco.txt"), "w") as f:
            f.write("python tests/reference_suites/run_reference_disco.py --report\n" + "\n".join(lines) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())

#!/usr/bin/env python
"""Build makani's own, unmodified FourCastNet 3 pieces that resample on the sphere -- FCN3's and SNO's `DiscreteContinuousDecoder` with
upsample_sht False (th.ResampleS2) and True (th.RealSHT / InverseRealSHT), and the whole `AtmoSphericNeuralOperatorNet` with the architecture
settings of config/fourcastnet3.yaml (scale factor 2, morlet (3, 3) "mean", no encoder MLP, serial MLPs of ratio 2, gelu, no norm, no big skip,
no bias, upsample_sht left at its default False) -- scaled to 49 x 96 with two pressure levels of four variables, four surface and three
auxiliary channels, 4 blocks and sfno_block_frequency 2, so that both block types occur.

Each object is built twice in one process, with the same seed, in the environment of run_reference_disco.py:
  (a) on the oracles (oracle/makani_resample_oracle.py, oracle/makani_disco_oracle.py) posed as torch_harmonics.ResampleS2 /
      DiscreteContinuousConvS2 -> a CPU forward and backward run, whose outputs must be finite and of the right shape;
  (b) on makani_b200's ResampleS2 and DiscreteContinuousConvS2 -> construction only (their kernels need a GPU).
Parameter names, shapes, dtypes, values and model-parallel tags must be identical, and no state dict may hold resample tables or psi.

    python tests/reference_suites/run_reference_fcn3.py            # one line per object, exit code 1 on any failure
    python tests/reference_suites/run_reference_fcn3.py --report   # also rewrites tests/reference_suites/report_fcn3.txt

Only runs where a checkout of makani is mounted; tests/test_reference_fcn3_suites.py checks the committed report.
"""
import importlib
import math
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_reference_sfno as S  # noqa: E402
import run_reference_disco as disco  # noqa: E402
import run_reference_tests as base  # noqa: E402

MODEL_SHAPE, DATA_SHAPE, EMBED, COUT = disco.MODEL_SHAPE, disco.IN_SHAPE, 10, 6
SETTINGS = disco.SETTINGS
CHANNELS = ["u10m", "v10m", "t2m", "msl", "u500", "v500", "z500", "t500", "u850", "v850", "z850", "t850"]
AUX = ["xoro", "xlsml", "xzen"]
NET = dict(model_grid_type="equiangular", sht_grid_type="legendre-gauss", inp_shape=DATA_SHAPE, out_shape=DATA_SHAPE, kernel_shape=[3, 3],
           filter_basis_type="morlet", filter_basis_norm_mode="mean", scale_factor=2, encoder_mlp=False, channel_names=CHANNELS,
           aux_channel_names=AUX, atmo_embed_dim=6, surf_embed_dim=7, aux_embed_dim=5, num_layers=4, num_groups=1, use_mlp=True, mlp_mode="serial",
           mlp_ratio=2, activation_function="gelu", normalization_layer="none", hard_thresholding_fraction=1.0, sfno_block_frequency=2,
           pos_embed=False, big_skip=False, bias=False)
TABLES = ("lat_idx", "lat_w", "lon_left", "lon_right", "lon_w", "lat_weights", "lon_idx_left", "lon_idx_right", "lon_weights", "psi")


def objects(M, modname):
    """(label, constructor, input shape) of the objects of network module M"""
    out = []
    for up in (False, True):
        out.append((f"DiscreteContinuousDecoder(upsample_sht={up})", lambda up=up: M.DiscreteContinuousDecoder(
            inp_shape=MODEL_SHAPE, out_shape=DATA_SHAPE, grid_in="legendre-gauss", grid_out="equiangular", inp_chans=EMBED, out_chans=COUT,
            groups=math.gcd(EMBED, COUT), bias=False, use_mlp=False, upsample_sht=up, **SETTINGS), (1, EMBED, *MODEL_SHAPE)))
    if modname.endswith("fourcastnet3"):
        out.append(("AtmoSphericNeuralOperatorNet", lambda: M.AtmoSphericNeuralOperatorNet(**NET), (1, len(CHANNELS) + len(AUX), *DATA_SHAPE)))
    return out


def run():
    """-> list of (network module, object, [problems], note)"""
    base.install_environment()
    S.stub_physicsnemo()
    from oracle import makani_disco_oracle as DO
    from oracle import makani_resample_oracle as RO

    import makani_b200.disco as mbdisco
    import makani_b200.resample as mbres

    th = sys.modules["torch_harmonics"]
    th.filter_basis = mbdisco     # get_filter_basis (host-only)
    sys.modules["torch_harmonics.filter_basis"] = mbdisco
    thd = sys.modules["torch_harmonics.distributed"]
    thd.DistributedDiscreteContinuousConvS2 = mbdisco.DistributedDiscreteContinuousConvS2
    thd.DistributedResampleS2 = mbres.DistributedResampleS2
    results = []
    for modname in ("makani.models.networks.fourcastnet3", "makani.models.networks.snonet"):
        try:
            M = importlib.import_module(modname)
        except Exception as e:  # noqa: BLE001
            results.append((modname, "import", [f"{type(e).__name__}: {e}"[:200]], ""))
            continue
        for label, make, xshape in objects(M, modname):
            problems = []
            try:
                th.DiscreteContinuousConvS2, th.ResampleS2 = DO.DiscreteContinuousConvS2, RO.ResampleS2
                torch.manual_seed(17)
                a = make()
                th.DiscreteContinuousConvS2, th.ResampleS2 = mbdisco.DiscreteContinuousConvS2, mbres.ResampleS2
                torch.manual_seed(17)
                b = make()
                da, db = disco.describe(a), disco.describe(b)
                if da != db:
                    problems.append(f"parameters differ: oracle {da} product {db}")
                for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
                    if pa.dtype != pb.dtype or not torch.equal(pa.detach(), pb.detach()):
                        problems.append(f"initial value of {n} differs")
                for net, who in ((a, "oracle"), (b, "product")):
                    held = [k for k in net.state_dict() if k.rsplit(".", 1)[-1] in TABLES]
                    if held:
                        problems.append(f"{who} state dict holds {held[:4]}")
                n_res = sum(isinstance(m, mbres.ResampleS2) for m in b.modules())
                n_conv = sum(isinstance(m, mbdisco.DiscreteContinuousConvS2) for m in b.modules())
                if n_res != sum(isinstance(m, RO.ResampleS2) for m in a.modules()) or n_conv != sum(isinstance(m, DO.DiscreteContinuousConvS2)
                                                                                                   for m in a.modules()):
                    problems.append("the product built a different number of resamplings / DISCO convolutions")
                if "upsample_sht=False" in label and n_res != 1:
                    problems.append(f"{n_res} product resamplings built, expected 1")
                a = a.double()
                x = torch.randn(*xshape, dtype=torch.float64, requires_grad=True)
                y = a(x)
                y = y[0] if isinstance(y, tuple) else y
                y.square().sum().backward()
                grads = [p.grad for p in a.parameters() if p.requires_grad]
                if not torch.isfinite(y).all() or not torch.isfinite(x.grad).all() or any(g is None or not torch.isfinite(g).all() for g in grads):
                    problems.append("non-finite forward / backward")
                note = f"{len(da)} parameters, {n_res} ResampleS2, {n_conv} DiscreteContinuousConvS2, y {tuple(y.shape)}"
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
    lines.append(f"TOTAL: {len(results)} objects built on the oracles and on makani_b200 as torch_harmonics.ResampleS2 / DiscreteContinuousConvS2, "
                 f"{bad} failing")
    print("\n".join(lines))
    if "--report" in sys.argv:
        with open(os.path.join(HERE, "report_fcn3.txt"), "w") as f:
            f.write("python tests/reference_suites/run_reference_fcn3.py --report\n" + "\n".join(lines) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())

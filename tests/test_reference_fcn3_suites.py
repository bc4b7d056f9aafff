"""The record of makani's own FCN3 / SNO decoders (upsample_sht False and True) and the whole FCN3 network built unmodified on the oracles and on
makani_b200 as `torch_harmonics.ResampleS2` / `DiscreteContinuousConvS2` (tests/reference_suites/run_reference_fcn3.py, which needs a checkout
of makani): the committed report must be green."""
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def test_committed_fcn3_report_is_green():
    rep = open(os.path.join(HERE, "reference_suites", "report_fcn3.txt")).read()
    lines = rep.splitlines()
    total = [ln for ln in lines if ln.startswith("TOTAL:")]
    assert total and total[0].rstrip().endswith(" 0 failing"), total
    rows = [("fourcastnet3", "AtmoSphericNeuralOperatorNet")]
    rows += [(net, f"DiscreteContinuousDecoder(upsample_sht={up})") for net in ("fourcastnet3", "snonet") for up in (False, True)]
    for net, obj in rows:
        row = [ln for ln in lines if ln.startswith(f"makani.models.networks.{net}.{obj}:")]
        assert row and ": ok " in row[0], (net, obj, row)
    net_row = [ln for ln in lines if ".AtmoSphericNeuralOperatorNet:" in ln][0]
    assert " 2 ResampleS2" in net_row, net_row          # the atmospheric and the surface decoder

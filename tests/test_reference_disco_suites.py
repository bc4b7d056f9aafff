"""The record of makani's own FCN3 / SNO DISCO layers (DiscreteContinuousEncoder, NeuralOperatorBlock(conv_type="local")) built unmodified on the
oracle and on makani_b200 as `torch_harmonics.DiscreteContinuousConvS2` (tests/reference_suites/run_reference_disco.py, which needs a checkout of
makani): the committed report must be green."""
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def test_committed_disco_report_is_green():
    rep = open(os.path.join(HERE, "reference_suites", "report_disco.txt")).read()
    lines = rep.splitlines()
    total = [ln for ln in lines if ln.startswith("TOTAL:")]
    assert total and total[0].rstrip().endswith(" 0 failing"), total
    for net in ("fourcastnet3", "snonet"):
        for layer in ("DiscreteContinuousEncoder", "NeuralOperatorBlock(local)"):
            row = [ln for ln in lines if ln.startswith(f"makani.models.networks.{net}.{layer}:")]
            assert row and ": ok " in row[0], (net, layer, row)

"""The record of makani's own GradientCRPSLoss / VortDivCRPSLoss test classes run unmodified against the oracle's vector transforms posing
as `torch_harmonics` (tests/reference_suites/run_reference_vector_tests.py, which needs a checkout of makani): the committed report must be
green."""
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def test_committed_vector_report_is_green():
    rep = open(os.path.join(HERE, "reference_suites", "report_vector.txt")).read()
    lines = rep.splitlines()
    total = [ln for ln in lines if ln.startswith("TOTAL:")]
    assert total and total[0].rstrip().endswith(" 0 failing"), total
    for cls in ("TestGradientCRPSLoss", "TestVortDivCRPSLoss"):
        row = [ln for ln in lines if ln.startswith(f"tests.test_losses.{cls}:")]
        assert row and " ran 0 " not in row[0] and "failures 0  errors 0" in row[0], row

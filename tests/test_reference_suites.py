"""The record of the original makani test classes at the SHT boundary, run unmodified against the oracle posing as `torch_harmonics`
(tests/reference_suites/run_reference_tests.py, which needs a checkout of makani): the committed report must be green."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "reference_suites"))


def test_committed_report_is_green():
    rep = open(os.path.join(HERE, "reference_suites", "report.txt")).read()
    total = [ln for ln in rep.splitlines() if ln.startswith("TOTAL:")]
    assert total and total[0].rstrip().endswith(" 0 failing"), total

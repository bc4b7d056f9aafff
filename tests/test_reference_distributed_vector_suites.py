"""The record of makani's VortDivCRPSLoss and GradientCRPSLoss under h x w spatial model parallelism (on DistributedRealVectorSHT /
DistributedInverseRealVectorSHT) against the same losses on the full tensors, from tests/reference_suites/run_reference_distributed_vector.py
(which needs a checkout of makani): the committed report must be green on every grid."""
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def test_committed_report_is_green():
    rep = open(os.path.join(HERE, "reference_suites", "report_distributed_vector.txt")).read()
    lines = rep.splitlines()
    total = [ln for ln in lines if ln.startswith("TOTAL:")]
    assert total and total[0].rstrip().endswith(" 0 failing"), total
    grids = [ln for ln in lines if ln.startswith("grid ")]
    assert [g.split()[1] for g in grids] == ["2x1", "1x2", "2x2"], grids
    assert all(g.rstrip().endswith(": OK") for g in grids), grids

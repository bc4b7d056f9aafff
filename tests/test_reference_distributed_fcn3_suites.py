"""The record of makani's own TestDistributedModel.test_distributed_model_fwd_bwd("FCN3", 1e-4) run unmodified on CPU / gloo with
DistributedDiscreteContinuousConvS2 / DistributedResampleS2 / DistributedRealSHT from makani_b200.distributed
(tests/reference_suites/run_reference_distributed_fcn3.py, which needs a checkout of makani): the committed report must be green on every grid,
compare the output, the loss, the input gradient and the weight gradients, and have built both distributed classes."""
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def test_committed_distributed_fcn3_report_is_green():
    rep = open(os.path.join(HERE, "reference_suites", "report_distributed_fcn3.txt")).read()
    lines = rep.splitlines()
    total = [ln for ln in lines if ln.startswith("TOTAL:")]
    assert total and total[0].rstrip().endswith(" 0 failing"), total
    grids = [ln for ln in lines if ln.startswith("grid ")]
    assert [g.split()[1] for g in grids][:3] == ["2x1", "1x2", "2x2"], grids
    assert all(g.rstrip().endswith(": OK") for g in grids), grids
    compared = [ln for ln in lines if ln.strip().startswith("compared on rank 0:")]
    assert len(compared) == len(grids)
    for ln in compared:
        assert "output 1, loss 1, input gradients 1, weight gradients " in ln and ln.rstrip().endswith("failing comparisons on all ranks: 0"), ln
        assert int(ln.split("weight gradients ")[1].split(";")[0]) > 0, ln
    built = [ln for ln in lines if ln.strip().startswith("built on rank 0:")]
    assert len(built) == len(grids)
    for ln in built:
        n_conv, n_res = int(ln.split(":")[1].split()[0]), int(ln.split(",")[1].split()[0])
        assert n_conv > 0 and n_res > 0, ln

"""The record of makani's own TestDistributedLayers.test_distributed_instance_norm_2d run unmodified on CPU / gloo after
makani_b200.compat.patch_makani_instance_norm() (tests/reference_suites/run_reference_distributed_instance_norm.py, which needs a checkout of
makani): the committed report must be green on every grid, have run all four cases, compared the output and the input gradient of each and every
rank's weight and bias gradients of the two affine cases, and have built the distributed class through the patch."""
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def test_committed_distributed_instance_norm_report_is_green():
    rep = open(os.path.join(HERE, "reference_suites", "report_distributed_instance_norm.txt")).read()
    lines = rep.splitlines()
    total = [ln for ln in lines if ln.startswith("TOTAL:")]
    assert total and total[0].rstrip() == "TOTAL: 4 grids, 0 failing", total
    grids = [ln for ln in lines if ln.startswith("grid ")]
    assert [g.split()[1] for g in grids] == ["2x1", "1x2", "2x2", "4x2"], grids
    assert all(g.rstrip().endswith(": OK") for g in grids), grids
    compared = [ln for ln in lines if ln.strip().startswith("tests run on rank 0:")]
    assert len(compared) == len(grids)
    for g, ln in zip(grids, compared):
        h, w = (int(v) for v in g.split()[1].split("x"))
        assert ln.strip().startswith("tests run on rank 0: 4;"), ln
        assert f"output 4, input gradients 4, weight gradients {2 * h * w}, bias gradients {2 * h * w}" in ln, ln
        assert ln.rstrip().endswith("failing comparisons on all ranks: 0"), ln
    built = [ln for ln in lines if ln.strip().startswith("built on rank 0:")]
    assert len(built) == len(grids) and all(ln.split(":")[1].split()[:2] == ["4", "DistributedInstanceNorm2d"] for ln in built), built

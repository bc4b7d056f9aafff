#!/usr/bin/env python
"""Run the reference's own test classes of the losses built on torch_harmonics.RealVectorSHT / InverseRealVectorSHT (GradientCRPSLoss,
VortDivCRPSLoss and the E = 1 path of both) against the oracle's vector transforms.

Same environment as run_reference_tests.py (its install_environment(): the oracle posed as `torch_harmonics`, the reference's modules
imported unmodified from where they lie), plus the oracle's RealVectorSHT / InverseRealVectorSHT on the posed package.

    python tests/reference_suites/run_reference_vector_tests.py            # one line per class, exit code 1 on any failure
    python tests/reference_suites/run_reference_vector_tests.py --report   # also rewrites tests/reference_suites/report_vector.txt

Only runs where a checkout of makani is mounted; tests/test_reference_vector_suites.py checks the committed report.
"""
import importlib
import os
import sys
import unittest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import run_reference_tests as base  # noqa: E402

SUITES = {"tests.test_losses": ["TestGradientCRPSLoss", "TestVortDivCRPSLoss"]}
# Left out of the count, but run and reported: three of its 46 cases (the "_4" loss configuration) build a loss on
# torch_harmonics.DiscreteContinuousConvS2, a convolution neither the oracle nor makani_b200 provides; the cases that go through the
# vector transforms pass.
LEFT_OUT = {"tests.test_losses": ["TestEnsembleLossE1FastPath"]}


def run(suites=SUITES):
    """-> list of (module, class, ran, failures, errors, [messages])"""
    if "torch_harmonics" not in sys.modules:
        base.install_environment()
        from oracle import makani_vector_oracle as V

        th = sys.modules["torch_harmonics"]
        th.RealVectorSHT, th.InverseRealVectorSHT = V.RealVectorSHT, V.InverseRealVectorSHT
    results = []
    for modname, classes in suites.items():
        M = importlib.import_module(modname)
        for name in classes:
            if not hasattr(M, name):
                results.append((modname, name, 0, 0, 1, [f"{name}: not defined in this checkout of the reference"]))
                continue
            suite = unittest.defaultTestLoader.loadTestsFromTestCase(getattr(M, name))
            r = unittest.TextTestRunner(verbosity=0, stream=open(os.devnull, "w")).run(suite)
            msgs = [t.id().split(".")[-1] + ": " + tb.strip().splitlines()[-1][:160] for t, tb in r.failures + r.errors]
            results.append((modname, name, r.testsRun, len(r.failures), len(r.errors), msgs))
    return results


def main():
    if not os.path.isdir(base.REF):
        print("reference tree not mounted: nothing to run")
        return 0
    results = run()
    lines = []
    for modname, name, ran, nf, ne, msgs in results:
        lines.append(f"{modname}.{name}: ran {ran}  failures {nf}  errors {ne}")
        lines += ["    " + m for m in msgs]
    total = sum(r[2] for r in results)
    bad = sum(r[3] + r[4] for r in results)
    lines.append(f"TOTAL: {total} reference tests against the oracle's vector transforms as torch_harmonics, {bad} failing")
    lines.append("Left out of the total (three cases need torch_harmonics.DiscreteContinuousConvS2, which is not provided):")
    for modname, name, ran, nf, ne, msgs in run(LEFT_OUT):
        lines.append(f"    {modname}.{name}: ran {ran}  failures {nf}  errors {ne}")
        lines += ["        " + m for m in msgs]
    print("\n".join(lines))
    if "--report" in sys.argv:
        with open(os.path.join(HERE, "report_vector.txt"), "w") as f:
            f.write("python tests/reference_suites/run_reference_vector_tests.py --report\n" + "\n".join(lines) + "\n")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())

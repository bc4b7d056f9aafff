"""Every instantiation of the tensor-core engine is held to the exact-operand bound by a case of tests/test_gpu_engine.py.

csrc/umma.cu builds one `umma_kernel<Traits, NB, split>` per tile width NB of its width lists (`using ...Widths = Widths<...>`) and per
`...Widths::launch_nb<Traits, split>` that launches from that list.  Each width has its own straight-line MMA code (on wgmma its own
instruction and register list), so a wrong fragment order or accumulator offset at one width shows at that width only.  The Legendre
and mix case tables name the instantiations each case launches, and the GPU tests assert through the profiler that exactly those ran;
here, without a GPU, their union must be every instantiation the source builds.  Adding a width, or a tiling change that moves the
last case off a width, fails this test until a case runs the new instantiation."""
import os
import re

from test_gpu_engine import FORWARD_GRIDS, LEG_CASES, MIX_CASES, TF32, VEC_CASES, X3, leg_engine_kernels, mix_engine_kernels

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UMMA_CU = os.path.join(ROOT, "makani_b200", "csrc", "umma.cu")


def built_instantiations():
    """{(Traits, NB, split)} that csrc/umma.cu instantiates, from its width lists and the launches that draw on them"""
    with open(UMMA_CU) as f:
        src = f.read()
    widths = {name: [int(w) for w in body.split(",")] for name, body in re.findall(r"using (\w+)Widths = Widths<([\d,\s]+)>;", src)}
    launches = set(re.findall(r"(\w+)Widths::launch_nb<(\w+), (true|false)>", src))
    assert set(widths) == {"Legendre", "Split", "Mix"}, widths
    assert {t for _, t, _ in launches} == {"AnaTraits", "SynTraits", "MixFwdTraits", "MixDgradTraits", "MixWgradTraits"}, launches
    return {(traits, nb, split == "true") for lst, traits, split in launches for nb in widths[lst]}


def leg_columns():
    return {k for c in LEG_CASES for prec in (TF32, X3) for s in leg_engine_kernels(c[-1], prec) for k in s}


def mix_columns():
    return {k for c in MIX_CASES for s in mix_engine_kernels(c[-1]) for k in s}


def test_every_built_instantiation_runs_under_the_bound():
    built = built_instantiations()
    covered = leg_columns() | mix_columns()
    assert not built - covered, f"built but run by no exact-operand case: {sorted(built - covered)}"
    assert not covered - built, f"named by a case but not built: {sorted(covered - built)}"


def test_the_other_engine_tables_name_built_instantiations():
    """the SHT forward and vector Legendre cases assert their instantiations too: they must name kernels the engine builds"""
    named = {("AnaTraits", c[-1], False) for c in FORWARD_GRIDS}
    named |= {k for c in VEC_CASES for s in leg_engine_kernels(c[-1], TF32) for k in s}
    assert named <= built_instantiations(), sorted(named - built_instantiations())

"""Every instantiation of the longitude FFT kernels is run by a case of tests/test_gpu_fft.py.

csrc/fft.cu builds, for T in {float, bf16}: `fft_analysis_ct_kernel<T, plan>` and `fft_synthesis_ct_kernel<T, plan, TRUNC>` (TRUNC true and
false) for every CT_PLANS entry and for the 8-row-tile plan of the B200SHT_FFT_VARIANT=1 switch, and `fft_analysis_rt_kernel<T, P>` /
`fft_synthesis_rt_kernel<T, P>` for every pair count of `launch_rt`'s LAUNCH(P).  Each has its own unrolled stages, tile walk and
split, so an error in one shows there only.  The rows of tests/test_gpu_fft.py name the instantiations they launch and the GPU test asserts
through the profiler that exactly those ran; here, without a GPU, their union must be every instantiation the source builds.  Adding a plan,
or moving the last row off one, fails this test until a row runs it."""
import re

from test_fft_layout import ct_plans
from test_gpu_fft import FFT_CU, ROWS, dispatch_route, nstages, row_kernels, rt_pairs, variant_plan

TYPES = ("float", "__nv_bfloat16")


def _src():
    with open(FFT_CU) as f:
        return f.read()


def launch_pairs():
    """the pair counts of launch_rt's LAUNCH(P) chain"""
    src = _src()
    body = src[src.index("static int launch_rt"):]
    body = body[: body.index("#undef LAUNCH")]
    return sorted({int(p) for p in re.findall(r"LAUNCH\((\d+)\)", body)})


def built():
    """{(direction, family, T, template arguments after T)} that csrc/fft.cu instantiates"""
    plans = [tuple(p) for p in ct_plans()] + [variant_plan()[1]]
    out = set()
    for T in TYPES:
        for p in plans:
            out |= {("analysis", "ct", T, p), ("synthesis", "ct", T, p + (1,)), ("synthesis", "ct", T, p + (0,))}
        for P in launch_pairs():
            out |= {("analysis", "rt", T, (P,)), ("synthesis", "rt", T, (P,))}
    return out


def covered(rows=ROWS):
    """what the rows launch: each row as it stands, and the compile-time rows of the variant length once more in the child process of
    test_fft_variant_plan_in_a_child_process"""
    vn, _ = variant_plan()
    out = set()
    for r in rows:
        out |= row_kernels(r)
        if r[2] == vn and r[8] in ("T", "F"):
            out |= row_kernels(r, variant=True)
    return out


def test_the_source_lists_are_read():
    assert len(ct_plans()) == 15
    assert variant_plan() == (1440, (8, 2, 96, 8, 9, 10, 2))
    assert launch_pairs() == [1, 2, 4]
    assert len(built()) == 108
    # rt_pairs restates rt_pick_pairs: the shared-memory formula and its limits
    src = _src()
    assert "sizeof(float2) * ((size_t)N + 2 * (size_t)pairs * (N + 1))" in src
    limits = re.findall(r"if \(rt_smem_bytes\(N, (\d)\) <= (\d+) \* 1024\) return (\d);", src)
    assert limits == [("4", "110", "4"), ("2", "220", "2"), ("1", "220", "1")], limits
    assert [rt_pairs(n) for n in (1001, 2002, 4096, 8192, 9386, 9387)] == [4, 2, 2, 1, 1, 0]


def test_every_fft_instantiation_runs_under_the_bound():
    b, c = built(), covered()
    assert not b - c, f"built but run by no case: {sorted(b - c)}"
    assert not c - b, f"named by a case but not built: {sorted(c - b)}"


def test_the_rows_name_what_the_dispatch_picks():
    for r in ROWS:
        assert dispatch_route(r[2], r[3], r[7]) == r[8], r[0]


def test_run_time_rows_use_every_radix():
    """the run-time plans of the rows' lengths use every radix of B200_RADIX_SWITCH (the case 16 is its default)"""
    src = _src()
    macro = src[src.index("#define B200_RADIX_SWITCH"):]
    macro = macro[: macro.index("\n\n")]
    radices = {int(r) for r in re.findall(r"case (\d+):", macro)} | {16}
    used = set()
    for r in ROWS:
        if r[8] not in ("T", "F"):
            used |= set(nstages(r[2])[1])
    assert radices == {2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15, 16}
    assert not radices - used, f"radices no run-time row uses: {sorted(radices - used)}"


"""Every instantiation of the neighbourhood-attention kernels and of the DISCO forward kernel is run by a case of the GPU suite.

csrc/attention.cu builds `attn_query_kernel<EM, VEC, false>` (forward), `attn_query_kernel<EM, VEC, true>` (query side of the backward) and
`attn_kv_kernel<EM, VEC>` (key/value side) for every `B200_ATTN_CASE(EM)` of its dispatch switch and VEC in {true, false}; csrc/disco.cu
builds `disco_forward_kernel<KP, NP>` for every `launch_forward<KP>` of its width switch, NP = 4 up to KP = 16, else 2.  Each instantiation
has its own unrolled register rows, so an error at one width or on one load path shows there only.  The case tables of
tests/test_gpu_attention.py and tests/test_gpu_disco.py name the instantiations each case launches, and the GPU tests assert through the
profiler that exactly those ran; here, without a GPU, their union must be every instantiation the source builds.  Adding a width, or moving
the last case off one, fails this test until a case runs it."""
import os
import re

from test_gpu_attention import CASES as ATTN_CASES
from test_gpu_attention import attn_kernels, em_vec
from test_gpu_disco import CASES as DISCO_CASES
from test_gpu_disco import FWD_KERNELS, GEOMS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "makani_b200", "csrc")


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def built_attention():
    """{(kernel, EM, VEC, QUERY or None)} that csrc/attention.cu instantiates"""
    src = _read("attention.cu")
    macro = re.search(r"#define B200_ATTN_CASE\(EM\)(.*?)\n\s*switch", src, re.S)[1]
    kinds = set(re.findall(r"launch_query<EM, VEC, (true|false)>|launch_(kv)<EM, VEC>", macro))
    assert kinds == {("false", ""), ("true", ""), ("", "kv")}, kinds
    ems = [int(e) for e in re.findall(r"^\s*(?:default:\s*)?B200_ATTN_CASE\((\d+)\)", src, re.M)]
    assert ems and re.search(r"dispatch_em<true>", src) and re.search(r"dispatch_em<false>", src)
    return {x for em in ems for vec in (True, False) for x in attn_kernels(em, vec)}


def built_disco_forward():
    """{(KP, NP)} that csrc/disco.cu instantiates"""
    src = _read("disco.cu")
    np_rule = re.search(r"constexpr int NP = KP <= (\d+) \? (\d+) : (\d+);", src)
    lim, lo, hi = (int(g) for g in np_rule.groups())
    return {(kp, lo if kp <= lim else hi) for kp in map(int, re.findall(r"launch_forward<(\d+)>\(a, st\)", src))}


def attention_columns():
    return {x for c in ATTN_CASES for x in attn_kernels(*c[-1])}


def disco_columns():
    return {x for _, ks in DISCO_CASES for x in FWD_KERNELS[ks]}


def test_the_source_lists_are_read():
    assert len(built_attention()) == 30
    assert built_disco_forward() == {(4, 4), (8, 4), (12, 4), (16, 4), (20, 2), (24, 2), (28, 2), (32, 2)}


def test_every_attention_instantiation_runs_under_the_bound():
    built, covered = built_attention(), attention_columns()
    assert not built - covered, f"built but run by no kernel case: {sorted(built - covered, key=str)}"
    assert not covered - built, f"named by a case but not built: {sorted(covered - built, key=str)}"


def test_every_disco_forward_width_runs_under_the_bound():
    built, covered = built_disco_forward(), disco_columns()
    assert not built - covered, f"built but run by no kernel case: {sorted(built - covered)}"
    assert not covered - built, f"named by a case but not built: {sorted(covered - built)}"


def test_the_rows_name_what_the_dispatch_picks():
    """each attention row's (EM, VEC) is what head_em / vec_ok pick for its head dims and storage offset, and each DISCO row's widths are
    those of its K in launches of at most 32"""
    for c in ATTN_CASES:
        name, ek, ev, off = c[0], c[8], c[9], c[11]
        assert em_vec(ek, ev, off) == c[-1], name
    src = _read("disco.cu")
    kc = int(re.search(r"constexpr int kDiscoMaxKC = (\d+);", src)[1])
    built = dict(built_disco_forward())
    for name, ks in DISCO_CASES:
        assert name in GEOMS
        K = ks[0] * ks[1]
        kps = {-(-min(kc, K - k0) // 4) * 4 for k0 in range(0, K, kc)}
        assert FWD_KERNELS[ks] == {(kp, built[kp]) for kp in kps}, ks

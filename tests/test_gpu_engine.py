"""The tensor-core engine (csrc/umma.cu) through the C ABI against fp64 references of its exact operands (tests/engine_ref.py).

TF32 mode: inputs are TF32 values, the weight is packed at TF32 (unpacking it must give tf32_rna(w) bit for bit) and the reference uses
the table rounded as the plan rounds it, so every product is exact and the only error allowed is the fp32 accumulation (+ one TF32
rounding where the epilogue rounds): |got - ref| <= r |ref| + (1 + r) c K 2^-24 sum |a||b|, far tighter than a relative-L2 check.
fp32x3 mode: fp32 operands, the fp32 table, plus a derived term for the omitted lo.lo product.

Inputs the kernels must not read hold NaN (unstored spec entries, latitude padding of the analysis input).  Outputs start as a NaN with
a fixed payload: stored entries must be finite and in the bound, the padding and the l < m entries exact zeros, everything else
untouched.  Every mix case asserts that it runs on the tensor cores.  Each case id names the tile boundary it exercises.  Every check
prints its worst bound ratio and the smallest c it would pass with (run with -s).

Every engine case also names the `umma_kernel<Traits, NB, split>` instantiations it launches (the last column of its table) and asserts,
through the profiler, that exactly those ran: together the tables run every tile width csrc/umma.cu builds under the bound, which
tests/test_engine_coverage_cpu.py checks without a GPU against the width lists in the source."""
import re

import pytest
import torch

import engine_ref as E
import makani_b200 as mb
from makani_b200 import _lib
from makani_b200.quadrature import _grid_np
from makani_b200.sht import Plan, _ptr, _stream

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = 0x7FC05EED   # quiet NaN with a payload no kernel writes
TF32, X3, FP32 = _lib.PREC_TF32, _lib.PREC_FP32X3, _lib.PREC_FP32


def sentinel(n):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)


def untouched(t):
    return bool((t.contiguous().view(torch.int32) == SENTINEL).all())


def check(case, what, got, ref, mag, K, r=0.0, extra=0.0, floor=0.0, c=E.C_ACC):
    ratio = E.bound_ratio(got, ref, mag, K, r=r, c=c, extra=extra, floor=floor)
    need = E.needed_c(got, ref, mag, K, r=r, extra=extra, floor=floor)
    print(f"[engine] {case} {what}: worst ratio {ratio:.3e}, needs c >= {need:.3e} (c = {c})")
    if ratio > 1.0:
        g, f = (torch.view_as_real(got), torch.view_as_real(ref)) if torch.is_complex(got) else (got, ref)
        err = (g.double() - f).abs().flatten()
        err[~torch.isfinite(err)] = float("inf")
        i = int(err.argmax())
        m = mag.double().flatten()[i // 2 if torch.is_complex(got) else i]
        raise AssertionError(f"{case} {what}: |got - ref| exceeds the bound by {ratio:.3g}x; worst at flat index {i}: got {g.flatten()[i].item()!r}, "
                             f"ref {f.flatten()[i].item()!r}, sum |a||b| {m.item()!r}")


def call(name, *args):
    _lib.call(name, *args)
    torch.cuda.synchronize()


def launched_kernels(fn, done=bool):
    """names of the library's CUDA kernels (namespace b200sht) that `fn` launches.  After many profiler sessions in one process the
    profiler often loses the first kernel of a session (on an H100 late in the GPU suite: the lone kernel of a one-kernel call, or the
    first of three, while 3 x TF32 calls, which launch a residual kernel first, kept every umma_kernel; rarely more than one), so each
    session starts with a few throwaway kernels of PyTorch's, and `fn` runs again until `done(names)` holds.  The calls profiled here are
    idempotent."""
    for _ in range(6):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(4):
                torch.zeros(1, device=DEV)
            fn()
            torch.cuda.synchronize()
        names = sorted({e.name for e in prof.events() if "b200sht::" in e.name})
        if done(names):
            break
    return names


# the profiler reports void b200sht::umma_kernel<b200sht::AnaTraits, 12, false>(...); cu++filt prints (int)12, (bool)0
UMMA_KERNEL = re.compile(r"umma_kernel<(?:b200sht::)?(\w+), (?:\(int\))?(\d+), (?:\(bool\))?(0|1|false|true)>")


def _engine_kernels(names):
    return {(m[1], int(m[2]), m[3] in ("1", "true")) for m in map(UMMA_KERNEL.search, names) if m}


def assert_engine_ran(tag, what, fn, want):
    """runs `fn` (idempotent) under the profiler: the umma_kernel instantiations (Traits, NB, split) it launches must be exactly `want`"""
    names = launched_kernels(fn, lambda n: _engine_kernels(n) == want)
    assert _engine_kernels(names) == want, f"{tag} {what}: expected umma_kernel {sorted(want)}, launched {names}"


# ------------------------------------------------------------------------------------------------------ Legendre
# id, grid, nlat, nlon, lmax, mmax, B, C, m_offset (None: ordinary plan), tile widths NB (analysis, synthesis at TF32; analysis,
# synthesis at 3 x TF32): see leg_engine_kernels
LEG_CASES = [
    ("one-kblock-one-ltile", "legendre-gauss", 32, 64, 32, 17, 1, 4, None, (4, 4, 8, 8)),
    ("ktail1-lstart32-cppad", "equiangular", 33, 64, 33, 33, 2, 5, None, (4, 4, 8, 8)),
    ("ltiles128+1-kp136-PBc3", "legendre-gauss", 129, 256, 129, 129, 2, 73, None, (32, 32, 16, 16)),
    ("B32-two-pbtiles-JP512", "equiangular", 91, 180, 91, 91, 32, 8, None, (32, 32, 16, 16)),
    ("nct2-JP400", "legendre-gauss", 64, 128, 64, 65, 1, 200, None, (32, 32, 16, 16)),
    ("JP152-ragged-coltile-C73", "legendre-gauss", 64, 128, 64, 65, 1, 73, None, (20, 20, 16, 16)),
    ("L65-lstart32-ltile-tail", "equiangular", 65, 128, 65, 65, 3, 6, None, (8, 8, 8, 8)),
    ("headline-23kblocks-tail17", "equiangular", 721, 1440, 240, 241, 1, 3, None, (4, 4, 8, 8)),
    ("m0=23", "equiangular", 65, 128, 40, 45 - 23, 2, 5, 23, (4, 4, 8, 8)),
    ("m0=32", "equiangular", 65, 128, 40, 45 - 32, 2, 5, 32, (4, 4, 8, 8)),
    ("cols96-C48", "legendre-gauss", 96, 192, 96, 97, 1, 48, None, (12, 12, 16, 16)),
    ("cols128-C64", "equiangular", 91, 180, 91, 91, 1, 64, None, (16, 16, 16, 16)),
    ("cols128-C64-m0=40", "equiangular", 91, 180, 91, 91 - 40, 1, 64, 40, (16, 16, 16, 16)),
    ("cols184-C90-cp92", "legendre-gauss", 64, 128, 64, 65, 1, 90, None, (24, 24, 16, 16)),
    ("cols192-B3-C30-PBc6", "equiangular", 33, 64, 33, 33, 3, 30, None, (24, 24, 16, 16)),
    # 2048 analysis tiles (2 column tiles x 32 image pairs x 32 orders) of one K-block for 131 CTAs: each wraps the 4-stage ring
    ("ring-wrap-1kblock-2048tiles", "legendre-gauss", 32, 64, 32, 32, 32, 200, None, (32, 32, 16, 16)),
    ("ring-wrap-2kblocks-2048tiles", "equiangular", 64, 128, 32, 32, 32, 200, None, (32, 32, 16, 16)),
]


def leg_engine_kernels(widths, prec):
    """the umma_kernel instantiations (analysis, synthesis) of a Legendre case at `prec` (`widths`: the last column of LEG_CASES or
    VEC_CASES); FP32 runs on the CUDA cores"""
    if prec == FP32:
        return set(), set()
    split = prec == X3
    a, s = widths[2:] if split else widths[:2]
    return {("AnaTraits", a, split)}, {("SynTraits", s, split)}


def _plan(grid, nlat, nlon, L, M, m0, vector=False):
    if m0 is None:
        return mb.get_plan(nlat, nlon, L, M, grid, True, DEV, vector=vector), 0
    cost, w = _grid_np(nlat, grid)
    return Plan.create_ex(nlat, nlon, L, M, m0, _lib.PLAN_VECTOR if vector else 0, cost, w, True, DEV), m0


def check_spec(case, what, sv, ref, mag, K, C, m0=0, dense=False, r=0.0, extra=0.0, zeros=True, floor=0.0, c=E.C_ACC, zero_mask=None):
    """packed spec output [L][M][2][B][cp]: unstored entries untouched, stored ones in the bound (the padding channels and, with
    `zeros`, the l < m entries exact zeros; `zero_mask` [L][M] replaces the scalar convention's l < m entries)"""
    L, M = sv.shape[:2]
    st = E.stored_mask(L, M, m0, dense, device=DEV)
    assert untouched(sv[~st]), f"{case} {what}: an unstored entry was written"
    assert (sv[st][..., C:] == 0).all(), f"{case} {what}: channel padding must hold exact zeros"
    if zeros:
        zm = E.zero_mask(L, M, m0, dense, device=DEV) if zero_mask is None else zero_mask
        assert (sv[zm] == 0).all(), f"{case} {what}: l < m entries must be exact zeros"
    check(case, what, sv[st], ref[st], mag[st], K, r=r, extra=extra, floor=floor, c=c)


@pytest.mark.parametrize("prec", [TF32, X3, FP32], ids=["tf32", "fp32x3", "fp32"])
@pytest.mark.parametrize("case,grid,nlat,nlon,L,M,B,C,m0,widths", LEG_CASES, ids=[c[0] for c in LEG_CASES])
def test_legendre_engine(case, grid, nlat, nlon, L, M, B, C, m0, widths, prec):
    """TF32 and 3 x TF32 on the tensor-core engine; FP32 on the CUDA-core kernels (64 x 64 output tiles, 16-deep k / l slabs), held to
    the same bound with the fp32 table and operands as they are"""
    plan, m0 = _plan(grid, nlat, nlon, L, M, m0)
    if prec != FP32:
        assert plan.umma_ok, "tensor-core path unavailable"
    kp, cp = plan.kp, (C + 3) // 4 * 4
    split = prec == X3
    tf32 = prec == TF32
    st = _stream(DEV)
    gen = torch.Generator(device=DEV).manual_seed(1234)
    T = E.tf32_rna(plan.table()) if tf32 else plan.table()
    rnd = (lambda *s: E.rand_tf32(*s, device=DEV, generator=gen)) if tf32 else (lambda *s: torch.randn(*s, device=DEV, generator=gen))
    tag = f"{case} {'fp32x3' if split else 'tf32' if tf32 else 'fp32'}"
    extra = E.SPLIT_TERM if split else 0.0
    kmul = 3 if split else 1   # hi.hi + hi.lo + lo.hi into one accumulator
    c = E.C_ACC if prec != FP32 else E.C_FMA
    want_ana, want_syn = leg_engine_kernels(widths, prec)

    # analysis: latspec [M8][2][B][C][kp] with NaN in the latitude padding and the padding orders
    lat = torch.full((plan.latspec_elems(B, C),), float("nan"), device=DEV)
    X = lat[: M * 2 * B * C * kp].view(M, 2, B, C, kp)
    X[..., :nlat] = rnd(M, 2, B, C, nlat)
    spec = sentinel(plan.spec_elems(B, C))
    assert_engine_ran(tag, "analysis", lambda: call("b200sht_legendre_analysis", plan.handle, _ptr(lat), _ptr(spec), B, C, prec, st), want_ana)
    ref, mag = E.legendre_analysis_ref(T, X, nlat, cp, m0)
    check_spec(tag, "analysis", spec.view(L, M, 2, B, cp), ref, mag, kmul * nlat, C, m0, r=E.R_TF32 if tf32 else 0.0, extra=extra,
               floor=E.underflow_floor(kmul * nlat, X[..., :nlat]), c=c)

    # synthesis: spec with NaN in the unstored region, zeros where l < m and in the channel padding
    S = rnd(L, M, 2, B, cp)
    S[..., C:] = 0
    S[E.zero_mask(L, M, m0, device=DEV)] = 0
    S[~E.stored_mask(L, M, m0, device=DEV)] = float("nan")
    ref, mag, K = E.legendre_synthesis_ref(T, S, C, m0)
    n = M * 2 * B * C * kp
    Z = sentinel(plan.latspec_elems(B, C))
    assert_engine_ran(tag, "synthesis", lambda: call("b200sht_legendre_synthesis", plan.handle, _ptr(S), _ptr(Z), B, C, prec, st), want_syn)
    assert untouched(Z[n:]), f"{tag}: the padding orders of the standard layout must not be written"
    Zv = Z[:n].view(M, 2, B, C, kp)
    assert (Zv[..., nlat:] == 0).all(), f"{tag}: latitude padding rows must be exact zeros"
    floor = E.underflow_floor(kmul * L, S)
    check(tag, "synthesis", Zv, ref, mag, kmul * K, extra=extra, floor=floor, c=c)
    if tf32 and plan.dft_ok:
        Zt = sentinel(plan.latspec_elems(B, C))
        assert_engine_ran(tag, "synthesis-tiled", lambda: call("b200sht_legendre_synthesis_tiled", plan.handle, _ptr(S), _ptr(Zt), B, C, st), want_syn)
        R = B * C
        tK = E.to_tiled(K.expand(M, 2, B, C, kp).reshape(M, 2, R, kp))
        # padding orders [M, 8 M2) have K = 0: exact zeros
        check(tag, "synthesis-tiled", Zt, E.to_tiled(ref.view(M, 2, R, kp)), E.to_tiled(mag.view(M, 2, R, kp)), tK, floor=floor)
        assert (Zt.view(R, kp // 8, 2, -1, 8, 8).permute(3, 4, 2, 0, 1, 5).reshape(-1, 2, R, kp)[M:] == 0).all()


# id, grid, nlat, nlon, lmax, mmax, B, C (vector fields: 2C component rows), m_offset (None: ordinary plan), tile widths NB (analysis,
# synthesis at TF32)
VEC_CASES = [
    ("DQ-split-in-ltile-L91-C3", "equiangular", 91, 192, 91, 91, 2, 3, None, (4, 4)),
    ("rows64-cols128-C32", "legendre-gauss", 64, 128, 64, 65, 1, 32, None, (16, 16)),
    ("order-shard-m0=51-C12", "equiangular", 91, 192, 91, 91 - 51, 1, 12, 51, (8, 8)),
]


@pytest.mark.parametrize("prec", [TF32, FP32], ids=["tf32", "fp32"])
@pytest.mark.parametrize("case,grid,nlat,nlon,L,M,B,C,m0,widths", VEC_CASES, ids=[c[0] for c in VEC_CASES])
def test_vector_legendre_engine(case, grid, nlat, nlon, L, M, B, C, m0, widths, prec):
    """b200sht_vector_legendre_analysis / _synthesis: the engine (TF32) and the CUDA-core kernels (FP32) on a vector plan's stacked table,
    rows D_l then Q_l of each order ([M][2L][kp]), with the 2C component rows as channels.  The stacked spec [2L][M][2][B][cp] is stored
    from row lstart(m0 + m), and both halves hold exact zeros for l < m0 + m (E.vector_zero_mask)."""
    plan, m0 = _plan(grid, nlat, nlon, L, M, m0, vector=True)
    assert plan.vector and plan.query(2) == L
    if prec == TF32:
        assert plan.umma_ok, "tensor-core path unavailable"
    L2, R = 2 * L, 2 * C
    kp, cp = plan.kp, (R + 3) // 4 * 4
    tf32 = prec == TF32
    st = _stream(DEV)
    gen = torch.Generator(device=DEV).manual_seed(4242)
    T = plan.table().permute(1, 0, 2, 3).reshape(M, L2, kp)   # [2][M][L][kp] (D, Q) -> the engine's [M][2L][kp]
    T = E.tf32_rna(T) if tf32 else T
    rnd = (lambda *s: E.rand_tf32(*s, device=DEV, generator=gen)) if tf32 else (lambda *s: torch.randn(*s, device=DEV, generator=gen))
    tag = f"vector {case} {'tf32' if tf32 else 'fp32'}"
    c = E.C_ACC if tf32 else E.C_FMA
    want_ana, want_syn = leg_engine_kernels(widths, prec)
    zm = E.vector_zero_mask(L, M, m0, device=DEV)

    lat = torch.full((plan.latspec_elems(B, R),), float("nan"), device=DEV)
    X = lat[: M * 2 * B * R * kp].view(M, 2, B, R, kp)
    X[..., :nlat] = rnd(M, 2, B, R, nlat)
    spec = sentinel(plan.spec_elems(B, R))
    assert_engine_ran(tag, "analysis", lambda: call("b200sht_vector_legendre_analysis", plan.handle, _ptr(lat), _ptr(spec), B, C, prec, st), want_ana)
    ref, mag = E.legendre_analysis_ref(T, X, nlat, cp, m0)
    check_spec(tag, "analysis", spec.view(L2, M, 2, B, cp), ref, mag, nlat, R, m0, r=E.R_TF32 if tf32 else 0.0,
               floor=E.underflow_floor(nlat, X[..., :nlat]), c=c, zero_mask=zm)

    S = rnd(L2, M, 2, B, cp)
    S[..., R:] = 0
    S[zm] = 0
    S[~E.stored_mask(L2, M, m0, device=DEV)] = float("nan")
    ref, mag, K = E.legendre_synthesis_ref(T, S, R, m0)
    n = M * 2 * B * R * kp
    Z = sentinel(plan.latspec_elems(B, R))
    assert_engine_ran(tag, "synthesis", lambda: call("b200sht_vector_legendre_synthesis", plan.handle, _ptr(S), _ptr(Z), B, C, prec, st), want_syn)
    assert untouched(Z[n:]), f"{tag}: the padding orders of the standard layout must not be written"
    Zv = Z[:n].view(M, 2, B, R, kp)
    assert (Zv[..., nlat:] == 0).all(), f"{tag}: latitude padding rows must be exact zeros"
    floor = E.underflow_floor(L2, S)
    check(tag, "synthesis", Zv, ref, mag, K, floor=floor, c=c)
    if tf32 and plan.dft_ok and m0 == 0:
        Zt = sentinel(plan.latspec_elems(B, R))
        assert_engine_ran(tag, "synthesis-tiled", lambda: call("b200sht_vector_legendre_synthesis_tiled", plan.handle, _ptr(S), _ptr(Zt), B, C, st), want_syn)
        tK = E.to_tiled(K.expand(M, 2, B, R, kp).reshape(M, 2, B * R, kp))
        check(tag, "synthesis-tiled", Zt, E.to_tiled(ref.view(M, 2, B * R, kp)), E.to_tiled(mag.view(M, 2, B * R, kp)), tK, floor=floor)


# ------------------------------------------------------------------------------------------------------------ mix
# id, L, M, B, G, Ci, Co, dense, tile widths NB (forward, dgrad, wgrad): see mix_engine_kernels
MIX_CASES = [
    ("M-crosses-32", 33, 33, 1, 1, 8, 8, False, (4, 4, 4)),
    ("raggedK-73-cppad", 65, 65, 2, 1, 73, 73, False, (12, 12, 12)),
    ("G2-B4-Mt32", 64, 65, 4, 2, 16, 24, False, (4, 4, 4)),
    ("G2-B4-Mt32-dense", 64, 65, 4, 2, 16, 24, True, (4, 4, 4)),
    ("G3-B8-crossgroupK-wgradstride4", 40, 41, 8, 3, 36, 12, False, (4, 4, 4)),
    ("B32-Mt4-one-order-per-wgrad-kblock", 32, 33, 32, 1, 8, 12, False, (4, 4, 4)),
    ("B32-Mt4-dense", 32, 33, 32, 1, 8, 12, True, (4, 4, 4)),
    ("wgrad-rowtiles-dgrad-coltiles-200-136", 64, 65, 1, 1, 200, 136, False, (12, 12, 12)),
    ("three-ragged-coltiles-300-330", 64, 65, 1, 1, 300, 330, False, (12, 12, 12)),
    ("headline-240x241-73", 240, 241, 1, 1, 73, 73, False, (12, 12, 12)),
    ("cols64-C64", 64, 65, 1, 1, 64, 64, False, (8, 8, 8)),
    ("two-coltiles-of-64-C128-B2", 64, 65, 2, 1, 128, 128, False, (8, 8, 8)),
    ("G2-ragged-slices-48-44", 64, 65, 1, 2, 96, 88, False, (8, 8, 8)),
    ("G2-ragged-slices-48-44-dense", 64, 65, 1, 2, 96, 88, True, (8, 8, 8)),
    # 33 x 128 row tiles (Mt = 4) of one K-block each: the 5-stage rings of the forward (mma.sync) and dgrad (wgmma) wrap many times
    ("ring-wrap-B32-Mt4-1kblock-L128", 128, 129, 32, 1, 8, 8, False, (4, 4, 4)),
]
OPS = {"dhconv": _lib.OP_DHCONV, "ldep": _lib.OP_LDEP, "shared": _lib.OP_SHARED}
MIX_PARAMS = [pytest.param(*c, op, id=f"{c[0]}-{op}") for c in MIX_CASES for op in OPS if c[4] == 1 or op == "dhconv"]


def mix_engine_kernels(widths):
    """the umma_kernel instantiations (b200sht_mix_forward, b200sht_mix_backward) of a mix case on the tensor cores"""
    f, d, w = widths
    return {("MixFwdTraits", f, False)}, {("MixDgradTraits", d, False), ("MixWgradTraits", w, False)}


def _native_weight(op, L, G, Ci, Co, gen):
    shape = {"dhconv": (G, Ci // G, Co // G, L), "ldep": (L, Ci, Co), "shared": (Ci, Co)}[op]
    return torch.randn(*shape, dtype=torch.complex64, device=DEV, generator=gen)


def _spec_input(L, M, B, C, dense, rnd):
    cp = (C + 3) // 4 * 4
    s = rnd(L, M, 2, B, cp)
    s[..., C:] = 0
    s[E.zero_mask(L, M, 0, dense, device=DEV)] = 0
    s[~E.stored_mask(L, M, 0, dense, device=DEV)] = float("nan")
    return s


def _run_mix(case, L, M, B, G, Ci, Co, dense, op, widths):
    """forward (without and with cbias) and backward (gx, gw, gcbias) of one shape through b200sht_mix_* at PREC_TF32, every output
    against the fp64 reference.  `widths` (a MIX_CASES column): TF32 operands and weight packed at TF32, and the calls launch the
    instantiations mix_engine_kernels names; None: the shape is served by the fp32 kernels (no umma_kernel), so fp32 operands and a
    weight packed at fp32 (as include/b200sht.h advises for such shapes)"""
    lib = _lib.load()
    code = OPS[op]
    opf = code | (_lib.DENSE_FLAG if dense else 0)
    st = _stream(DEV)
    gen = torch.Generator(device=DEV).manual_seed(4321)
    tf32 = widths is not None
    want_fwd, want_bwd = mix_engine_kernels(widths) if tf32 else (set(), set())
    rnd = (lambda *s: E.rand_tf32(*s, device=DEV, generator=gen)) if tf32 else (lambda *s: torch.randn(*s, device=DEV, generator=gen))
    Cig, Cog = Ci // G, Co // G
    cpi, cpo, cop = (Ci + 3) // 4 * 4, (Co + 3) // 4 * 4, (Cog + 3) // 4 * 4
    r = E.R_TF32 if tf32 else 0.0   # the tensor-core forward / dgrad epilogues round to TF32

    wn = _native_weight(op, L, G, Ci, Co, gen)
    wp = sentinel(int(lib.b200sht_mix_weight_elems(code, L, M, G, Ci, Co)))
    call("b200sht_mix_weight_pack", code, _ptr(wn), _ptr(wp), L, G, Ci, Co, TF32 if tf32 else FP32, st)
    wu = torch.empty_like(wn)
    call("b200sht_mix_weight_unpack", code, _ptr(wp), _ptr(wu), L, G, Ci, Co, st)
    want = E.tf32_rna(torch.view_as_real(wn)) if tf32 else torch.view_as_real(wn)
    assert torch.equal(torch.view_as_real(wu).view(torch.int32), want.view(torch.int32)), f"{case}: packed weight != tf32_rna(w)"
    assert (wp.view(-1, G, Cig, 2, cop)[..., Cog:] == 0).all(), f"{case}: packed-weight padding must be exact zeros"

    x = _spec_input(L, M, B, Ci, dense, rnd)
    gy = _spec_input(L, M, B, Co, dense, rnd)
    cb = torch.randn(Co, dtype=torch.complex64, device=DEV, generator=gen)
    for bias in (None, cb):
        y = sentinel(L * M * 2 * B * cpo)
        assert_engine_ran(case, "forward", lambda: call("b200sht_mix_forward", L, M, opf, _ptr(x), _ptr(wp), _ptr(bias), _ptr(y), B, G, Ci, Co, TF32, st),
                          want_fwd)
        ref, mag, K = E.mix_forward_ref(x, wp, G, Ci, Co, cbias=bias, dense=dense)
        check_spec(case, "forward" + ("+cbias" if bias is not None else ""), y.view(L, M, 2, B, cpo), ref, mag, K, Co, dense=dense, r=r,
                   zeros=bias is None)

    gx = sentinel(L * M * 2 * B * cpi)
    gw = sentinel(wp.numel())
    gcb = sentinel(2 * Co)
    assert_engine_ran(case, "backward", lambda: call("b200sht_mix_backward", L, M, opf, _ptr(x), _ptr(wp), _ptr(gy), _ptr(gx), _ptr(gw), _ptr(gcb), B, G, Ci,
                                                     Co, TF32, st), want_bwd)
    ref, mag, K = E.mix_dgrad_ref(gy, wp, G, Ci, Co, dense=dense)
    check_spec(case, "dgrad", gx.view(L, M, 2, B, cpi), ref, mag, K, Ci, dense=dense, r=r)
    ref, mag, K = E.mix_wgrad_ref(x, gy, G, Ci, Co, shared=(op == "shared"), dense=dense)
    check(case, "wgrad", gw.view(ref.shape), ref, mag, K)   # channel padding [Cog, cop): reference and bound 0 -> exact zeros
    ref, mag, K = E.mix_cbias_grad_ref(gy, Co, dense=dense)
    check(case, "cbias-grad", torch.view_as_complex(gcb.view(Co, 2)), ref, mag, K)


@pytest.mark.parametrize("case,L,M,B,G,Ci,Co,dense,widths,op", MIX_PARAMS)
def test_mix_engine(case, L, M, B, G, Ci, Co, dense, widths, op):
    assert _lib.load().b200sht_mix_uses_tensor_cores(OPS[op], B, G, Ci, Co, TF32) == 1, f"{case}: not on the tensor cores"
    _run_mix(f"{case}-{op}", L, M, B, G, Ci, Co, dense, op, widths)


@pytest.mark.parametrize("case,L,M,B,G,Ci,Co", [("B3", 33, 33, 3, 1, 8, 8), ("G2-slices5to6", 33, 33, 1, 2, 10, 12)], ids=["B3", "G2-slices5to6"])
def test_mix_shapes_outside_the_tensor_cores(case, L, M, B, G, Ci, Co):
    """shapes the tensor-core mix cannot address are served by the fp32 CUDA-core kernels (the route query says so): unrounded fp32
    weight and operands, no TF32 rounding of the output, same reference and bound"""
    assert _lib.load().b200sht_mix_uses_tensor_cores(_lib.OP_DHCONV, B, G, Ci, Co, TF32) == 0
    _run_mix(f"fallback-{case}", L, M, B, G, Ci, Co, False, "dhconv", None)


# ------------------------------------------------------------------------------------------------ SHT forward
def _workspace(plan, B, C):
    nbytes = int(_lib.load().b200sht_sht_workspace_bytes(plan.handle, B, C))
    return sentinel(nbytes // 4)


# id, grid, nlat, nlon, lmax, mmax, B, C, dtype (the tensor-core DFT takes fp32 rows when nlon % 32 == 0, bf16 otherwise), tile width NB
# of the TF32 Legendre analysis (umma_kernel<AnaTraits, NB, false>)
FORWARD_GRIDS = [
    ("181x360-bf16", "legendre-gauss", 181, 360, 181, 181, 1, 4, torch.bfloat16, 4),
    ("721x1440", "equiangular", 721, 1440, 240, 241, 1, 3, torch.float32, 4),
    ("721x1440-cols128-C64", "equiangular", 721, 1440, 240, 241, 1, 64, torch.float32, 16),
]


@pytest.mark.parametrize("case,grid,nlat,nlon,L,M,B,C,dtype,nb", FORWARD_GRIDS, ids=[c[0] for c in FORWARD_GRIDS])
def test_sht_forward_analysis(case, grid, nlat, nlon, L, M, B, C, dtype, nb):
    """b200sht_sht_forward at TF32: the (longitude analysis -> Legendre analysis) pair through the workspace.  Operands: the latspec the
    longitude stage left in the workspace (the same rows as one plain b200sht_fft_analysis) and the TF32 table."""
    plan = mb.get_plan(nlat, nlon, L, M, grid, True, DEV)
    assert plan.umma_ok and plan.dft_ok
    kp, cp = plan.kp, (C + 3) // 4 * 4
    st = _stream(DEV)
    torch.manual_seed(99)
    x = torch.randn(B, C, nlat, nlon, device=DEV).to(dtype)
    code = mb.sht._dtype_code(dtype)
    nl = M * 2 * B * C * kp
    lat0 = torch.full((plan.latspec_elems(B, C),), float("nan"), device=DEV)
    call("b200sht_fft_analysis", plan.handle, _ptr(x), code, B, C, _ptr(lat0), 0 | 2, st)
    ws = _workspace(plan, B, C)
    coeffs = torch.empty(B, C, L, M, dtype=torch.complex64, device=DEV)
    assert_engine_ran(case, "analysis", lambda: call("b200sht_sht_forward", plan.handle, _ptr(x), code, B, C, _ptr(coeffs), _ptr(ws), TF32, st),
                      {("AnaTraits", nb, False)})
    X = ws[:nl].view(M, 2, B, C, kp)
    X0 = lat0[:nl].view(M, 2, B, C, kp)
    assert torch.equal(X[..., :nlat].view(torch.int32), X0[..., :nlat].view(torch.int32)), "latspec rows != plain fft_analysis"
    spec_off = (4 * plan.latspec_elems(B, C) + 255) // 256 * 256 // 4
    sv = ws[spec_off : spec_off + plan.spec_elems(B, C)].view(L, M, 2, B, cp)
    ref, mag = E.legendre_analysis_ref(E.tf32_rna(plan.table()), E.tf32_trunc(X), nlat, cp)
    check_spec(case, "analysis", sv, ref, mag, nlat, C, r=E.R_TF32, floor=E.underflow_floor(nlat, X[..., :nlat]))
    tri = torch.tril(torch.ones(L, M, dtype=torch.bool, device=DEV))
    want = torch.where(tri, torch.complex(sv[:, :, 0, :, :C], sv[:, :, 1, :, :C]).permute(2, 3, 0, 1), 0)
    assert torch.equal(coeffs, want), "coefficients != the packed spectrum in the workspace"

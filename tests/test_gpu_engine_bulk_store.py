"""The bulk-store epilogue of the tensor-core Legendre synthesis (csrc/umma.cu, SynTraits::epilogue_staged) at the tile widths that
stage a tile in 32-column pieces (more than 20 fragments: C = 384 and a 184-column tile).  Every case ends inside its last 128-row
latitude box (kp = 72, 136 and 40), where the store map clips the boxes.  Same conventions as tests/test_gpu_engine.py: outputs start as
NaN sentinels, stored entries are checked against the fp64 reference of the exact operands, padding rows and orders must be exact zeros,
nothing else may be written."""
import pytest
import torch

import engine_ref as E
import makani_b200 as mb
from makani_b200 import _lib
from makani_b200.sht import _ptr, _stream

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SENTINEL = 0x7FC05EED
TF32 = _lib.PREC_TF32


def sentinel(n):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)


def untouched(t):
    return bool((t.contiguous().view(torch.int32) == SENTINEL).all())


def call(name, *args):
    _lib.call(name, *args)
    torch.cuda.synchronize()


def check(case, got, ref, mag, K, floor):
    ratio = E.bound_ratio(got, ref, mag, K, floor=floor)
    assert ratio <= 1.0, f"{case}: |got - ref| exceeds the bound by {ratio:.3g}x"


# id, grid, nlat, nlon, lmax, mmax, B, C
WIDE = [
    ("C384-N256-pieces", "equiangular", 65, 128, 40, 45, 1, 384),
    ("C90-N192-pieces", "legendre-gauss", 129, 256, 129, 129, 1, 90),
    ("B2-C100-JP400", "equiangular", 33, 64, 33, 33, 2, 100),
]


@pytest.mark.parametrize("case,grid,nlat,nlon,L,M,B,C", WIDE, ids=[c[0] for c in WIDE])
def test_synthesis_staged_in_pieces(case, grid, nlat, nlon, L, M, B, C):
    plan = mb.get_plan(nlat, nlon, L, M, grid, True, DEV)
    assert plan.umma_ok, "tensor-core path unavailable"
    kp, cp = plan.kp, (C + 3) // 4 * 4
    st = _stream(DEV)
    gen = torch.Generator(device=DEV).manual_seed(4321)
    T = E.tf32_rna(plan.table())
    S = E.rand_tf32(L, M, 2, B, cp, device=DEV, generator=gen)
    S[..., C:] = 0
    S[E.zero_mask(L, M, 0, device=DEV)] = 0
    S[~E.stored_mask(L, M, 0, device=DEV)] = float("nan")
    ref, mag, K = E.legendre_synthesis_ref(T, S, C, 0)
    floor = E.underflow_floor(L, S)
    n = M * 2 * B * C * kp
    Z = sentinel(plan.latspec_elems(B, C))
    call("b200sht_legendre_synthesis", plan.handle, _ptr(S), _ptr(Z), B, C, TF32, st)
    assert untouched(Z[n:]), f"{case}: the padding orders of the standard layout must not be written"
    Zv = Z[:n].view(M, 2, B, C, kp)
    assert (Zv[..., nlat:] == 0).all(), f"{case}: latitude padding rows must be exact zeros"
    check(f"{case} synthesis", Zv, ref, mag, K, floor)
    if plan.dft_ok:
        Zt = sentinel(plan.latspec_elems(B, C))
        call("b200sht_legendre_synthesis_tiled", plan.handle, _ptr(S), _ptr(Zt), B, C, st)
        R = B * C
        tK = E.to_tiled(K.expand(M, 2, B, C, kp).reshape(M, 2, R, kp))
        check(f"{case} synthesis-tiled", Zt, E.to_tiled(ref.view(M, 2, R, kp)), E.to_tiled(mag.view(M, 2, R, kp)), tK, floor)
        assert (Zt.view(R, kp // 8, 2, -1, 8, 8).permute(3, 4, 2, 0, 1, 5).reshape(-1, 2, R, kp)[M:] == 0).all()


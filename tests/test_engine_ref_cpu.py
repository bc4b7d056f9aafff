"""CPU checks of the fp64 references and the bound that tests/test_gpu_engine.py holds the tensor-core engine to (tests/engine_ref.py):
the TF32 conversions bit for bit, the stored-region convention against csrc/common.cuh, the mix references against the reference's own
contraction outputs (and PyTorch autograd for the gradients), the Legendre references against oracle einsums."""
import os
import re

import numpy as np
import pytest
import torch

import engine_ref as E
from oracle import makani_oracle as O
from oracle import makani_vector_oracle as V

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "contractions_golden.npz")


def _f(bits):
    return torch.tensor(bits, dtype=torch.int64).to(torch.int32).view(torch.float32)


def _bits(t):
    return [int(b) & 0xFFFFFFFF for b in t.view(torch.int32).tolist()]


# ------------------------------------------------------------------------------------------------ TF32 conversions
# (input bits, rna bits, trunc bits)
TF32_CASES = [
    (0x3F800000, 0x3F800000, 0x3F800000),   # 1.0 is TF32
    (0x3F800FFF, 0x3F800000, 0x3F800000),   # just below half an ulp: down
    (0x3F801000, 0x3F802000, 0x3F800000),   # tie: away from zero
    (0x3F803000, 0x3F804000, 0x3F802000),   # tie with an odd kept mantissa: still away from zero (not to even)
    (0x3F801001, 0x3F802000, 0x3F800000),   # above the tie
    (0xBF801000, 0xBF802000, 0xBF800000),   # negative tie: away from zero, i.e. more negative
    (0xBF800FFF, 0xBF800000, 0xBF800000),
    (0x3FFFF000, 0x40000000, 0x3FFFE000),   # tie at the top of a binade: carries into the exponent (2.0)
    (0xBFFFFFFF, 0xC0000000, 0xBFFFE000),   # negative binade edge
    (0x007FF000, 0x00800000, 0x007FE000),   # largest subnormals round up to the smallest normal
    (0x00000FFF, 0x00000000, 0x00000000),   # subnormal below half an ulp
    (0x00001000, 0x00002000, 0x00000000),   # subnormal tie
    (0x80001000, 0x80002000, 0x80000000),   # negative subnormal tie
    (0x00000000, 0x00000000, 0x00000000),   # +0
    (0x80000000, 0x80000000, 0x80000000),   # -0 keeps its sign
    (0x7F800000, 0x7F800000, 0x7F800000),   # +inf
    (0xFF800000, 0xFF800000, 0xFF800000),   # -inf
]


@pytest.mark.parametrize("x,rna,trunc", TF32_CASES, ids=[f"{c[0]:08x}" for c in TF32_CASES])
def test_tf32_conversions_bit_patterns(x, rna, trunc):
    t = _f([x])
    assert _bits(E.tf32_rna(t)) == [rna]
    assert _bits(E.tf32_trunc(t)) == [trunc]


def test_tf32_rna_nan_and_random_values():
    assert torch.isnan(E.tf32_rna(torch.tensor([float("nan")]))).all()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(100000, generator=g) * torch.exp2(torch.randint(-60, 60, (100000,), generator=g).float())
    r = E.tf32_rna(x)
    assert (r.view(torch.int32) & 0x1FFF == 0).all(), "13 low mantissa bits must be clear"
    assert torch.equal(E.tf32_rna(r), r), "TF32 values are fixed points"
    # nearest: within half a TF32 ulp of x, and no other TF32 value is closer (the neighbours are one ulp away)
    ulp = torch.exp2(torch.floor(torch.log2(x.double().abs())) - 10)
    assert ((r.double() - x.double()).abs() <= ulp / 2).all()
    assert ((r.double() - x.double()).abs() <= E.R_TF32 * x.double().abs()).all()


# ----------------------------------------------------------------------------------------------- storage convention
def _common_cuh():
    with open(os.path.join(ROOT, "makani_b200", "csrc", "common.cuh")) as f:
        return f.read()


def test_stored_mask_follows_common_cuh():
    src = _common_cuh()
    # the convention as the kernels state it; these lines are restated below
    assert "constexpr int kTriBlock = 32;" in src and E.TRI == 32
    assert re.search(r"HD int lstart\(int m\) \{ return \(m / kTriBlock\) \* kTriBlock; \}", src)
    assert re.search(r"HD int mend\(int l, int M\) \{ int e = \(l / kTriBlock \+ 1\) \* kTriBlock; return e < M \? e : M; \}", src)
    assert re.search(r"HD int mend_d\(int l, int M, int dense\) \{ return dense \? M : mend\(l, M\); \}", src)

    def mend(l, M):
        e = (l // 32 + 1) * 32
        return e if e < M else M

    for L, M in ((7, 8), (33, 33), (40, 41), (64, 65), (129, 129), (240, 241), (20, 70)):
        st = E.stored_mask(L, M)
        rows = torch.tensor([[m < mend(l, M) for m in range(M)] for l in range(L)])
        assert torch.equal(st, rows), (L, M)   # the mix kernels walk rows m < mend(l)
        assert E.stored_mask(L, M, dense=True).all()
        z = E.zero_mask(L, M)
        assert torch.equal(z, torch.tensor([[E.lstart(m) <= l < m for m in range(M)] for l in range(L)]))
        assert not E.zero_mask(L, M, dense=True).any()
    # with an order offset the Legendre kernels start order m at degree lstart(m0 + m)
    for m0 in (23, 32, 45):
        st = E.stored_mask(40, 22, m0)
        assert torch.equal(st, torch.tensor([[l >= 32 * ((m0 + m) // 32) for m in range(22)] for l in range(40)]))
        z = E.zero_mask(40, 22, m0)
        assert torch.equal(z, st & torch.tensor([[l < m0 + m for m in range(22)] for l in range(40)]))


@pytest.mark.parametrize("L,M,m0", [(9, 10, 0), (40, 41, 0), (91, 40, 51), (40, 22, 23)])
def test_vector_zero_mask_is_where_the_stacked_tables_vanish(L, M, m0):
    """the stacked vector spec (rows D_l, then Q_l) as the Legendre stages store it: the 2L rows from lstart(m0 + m); exact zeros where
    l < m0 + m in either half, which is exactly where the analysis of the stacked fp64 tables of the vector oracle vanishes (besides the
    rows that are zero for every order: D_0, and Q of order 0)"""
    z = E.vector_zero_mask(L, M, m0)
    st = E.stored_mask(2 * L, M, m0)
    want = torch.tensor([[2 * L > r >= E.lstart(m0 + m) and r % L < m0 + m for m in range(M)] for r in range(2 * L)])
    assert torch.equal(z, want)
    assert torch.equal(z[:L], E.zero_mask(L, M, m0)), "the D half follows the scalar convention"
    assert st[L:].all(), "the whole Q half is stored"

    nlat = 33
    th, _ = O.precompute_latitudes(nlat, "equiangular")
    D, Q = V.vector_legpoly(m0 + M, L, th)
    T = torch.from_numpy(np.concatenate([D, Q], axis=1)[m0:])               # [M][2L][nlat]
    X = torch.randn(M, 2, 1, 3, nlat, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    ref, mag = E.legendre_analysis_ref(T, X, nlat, 4, m0)
    assert (ref[z] == 0).all() and (mag[z] == 0).all()
    r = torch.arange(2 * L)[:, None]
    m = torch.arange(M)[None, :]
    always0 = (r == 0) | ((r >= L) & (m0 + m == 0))
    assert (mag[st & ~z & ~always0][..., :3] > 0).all()


def test_to_tiled_index_map():
    """latspec[r][k / 8][plane][m / 8][m % 8][k % 8] (include/b200sht.h), orders padded with zeros to a multiple of 8"""
    M, R, kp = 13, 3, 24
    Z = torch.arange(M * 2 * R * kp, dtype=torch.float64).view(M, 2, R, kp) + 1
    t = E.to_tiled(Z)
    M2 = 2
    assert t.numel() == 8 * M2 * 2 * R * kp
    v = t.view(R, kp // 8, 2, M2, 8, 8)
    for m, p, r, k in ((0, 0, 0, 0), (12, 1, 2, 23), (5, 1, 1, 9), (8, 0, 2, 16)):
        assert v[r, k // 8, p, m // 8, m % 8, k % 8] == Z[m, p, r, k]
    assert (v[:, :, :, 1, M - 8:] == 0).all()


# ------------------------------------------------------------------------------------------------ mix vs golden
def _pack_spec(z, cp):
    """complex (B, C, L, M) -> packed [L][M][2][B][cp] float64"""
    return E.complex_to_spec(z.to(torch.complex128).permute(2, 3, 0, 1), cp)


def _unpack_spec(s, C):
    """packed [L][M][2][B][cp] -> complex (B, C, L, M)"""
    return torch.complex(s[:, :, 0, :, :C], s[:, :, 1, :, :C]).permute(2, 3, 0, 1)


def _golden():
    return {k: torch.from_numpy(v) for k, v in np.load(GOLD).items()}


def test_mix_references_match_reference_contractions():
    g = _golden()
    x = g["x"]                                                 # (B, G, Cig, L, M)
    B, G, Cig, L, M = x.shape
    w = g["w_dhconv"]                                          # (G, Cig, Cog, L)
    Cog = w.shape[2]
    Ci, Co = G * Cig, G * Cog
    xs = _pack_spec(x.reshape(B, Ci, L, M), Ci + (-Ci) % 4)
    wp = E.complex_to_weight(w.to(torch.complex128).permute(3, 0, 1, 2), Cog + (-Cog) % 4)
    y, mag, K = E.mix_forward_ref(xs, wp, G, Ci, Co)
    gold = g["y_dhconv"].reshape(B, Co, L, M).to(torch.complex128)
    assert torch.allclose(_unpack_spec(y, Co), gold, rtol=1e-5, atol=1e-6)
    # the reference output is fp32: inside the fp32 accumulation bound of the fp64 result
    assert E.bound_ratio(torch.view_as_real(gold.permute(2, 3, 0, 1)), torch.view_as_real(_unpack_spec(y, Co).permute(2, 3, 0, 1)),
                         _unpack_spec(mag, Co).real.permute(2, 3, 0, 1)[..., None].expand(L, M, B, Co, 2), K, c=1.0) <= 1.0
    assert K == 2 * Cig
    xa, cb = g["xa"], g["cbias"].reshape(-1)                   # (B, Ci, L, M), (Co,)
    Ci = xa.shape[1]
    xs = _pack_spec(xa, Ci + (-Ci) % 4)
    for name, wn in (("shared", g["w_shared"][None]), ("ldep", g["w_ldep"])):   # -> [Lw][Ci][Co]
        Co = wn.shape[-1]
        wp = E.complex_to_weight(wn.to(torch.complex128)[:, None], Co + (-Co) % 4)
        y, _, _ = E.mix_forward_ref(xs, wp, 1, Ci, Co)
        assert torch.allclose(_unpack_spec(y, Co), g[f"y_{name}"].to(torch.complex128), rtol=1e-5, atol=1e-6), name
        y, _, _ = E.mix_forward_ref(xs, wp, 1, Ci, Co, cbias=cb)
        assert torch.allclose(_unpack_spec(y, Co), g[f"y_{name}_bias"].to(torch.complex128), rtol=1e-5, atol=1e-6), name + "+bias"


@pytest.mark.parametrize("G,shared,dense", [(1, False, False), (3, False, False), (1, True, False), (2, False, True)])
def test_mix_gradient_references_match_autograd(G, shared, dense):
    """dgrad / wgrad / cbias-grad references = PyTorch's complex gradients of the forward reference; 40 x 41 crosses the 32-row
    triangle blocks, so the stored rows of each l matter."""
    gen = torch.Generator().manual_seed(7)
    L, M, B, Cig, Cog = 40, 41, 2, 3, 5
    Ci, Co = G * Cig, G * Cog
    cpi, cpo, cop = Ci + (-Ci) % 4, Co + (-Co) % 4, Cog + (-Cog) % 4
    st = E.stored_mask(L, M, dense=dense)

    def spec(C, cp):
        s = torch.randn(L, M, 2, B, cp, generator=gen, dtype=torch.float64)
        s[..., C:] = 0
        s[~st] = float("nan")
        return s

    x, gy = spec(Ci, cpi), spec(Co, cpo)
    Lw = 1 if shared else L
    wc = torch.randn(Lw, G, Cig, Cog, dtype=torch.complex128, generator=gen)
    cb = torch.randn(Co, dtype=torch.complex128, generator=gen)
    xc = E.spec_to_complex(x, Ci, dense).requires_grad_(True)
    wr = wc.clone().requires_grad_(True)
    cbr = cb.clone().requires_grad_(True)
    y = torch.einsum("lmbgi,lgio->lmbgo", xc.view(L, M, B, G, Cig), wr.expand(L, G, Cig, Cog)).reshape(L, M, B, Co) + cbr
    y.backward(E.spec_to_complex(gy, Co, dense))
    wp = E.complex_to_weight(wc, cop)
    yref, _, _ = E.mix_forward_ref(x, wp, G, Ci, Co, cbias=cb, dense=dense)
    keep = st[:, :, None, None]
    assert torch.allclose(_unpack_spec(yref, Co).permute(2, 3, 0, 1), torch.where(keep, y.detach(), 0))
    gx, gxmag, K = E.mix_dgrad_ref(gy, wp, G, Ci, Co, dense=dense)
    assert K == 2 * Cog
    got = E.complex_to_spec(torch.where(keep, xc.grad, 0), cpi)
    assert torch.allclose(gx, got)
    assert (gxmag >= gx.abs()).all()
    gw, gwmag, Kw = E.mix_wgrad_ref(x, gy, G, Ci, Co, shared=shared, dense=dense)
    assert torch.allclose(gw, E.complex_to_weight(wr.grad, cop))
    assert (gwmag >= gw.abs()).all()
    rows = st.sum(1) * B
    assert torch.equal(Kw.view(-1), 2 * (rows.sum().view(1) if shared else rows).double())
    gcb, _, _ = E.mix_cbias_grad_ref(gy, Co, dense=dense)
    assert torch.allclose(gcb, cbr.grad)


# ------------------------------------------------------------------------------------------- Legendre vs oracle
@pytest.mark.parametrize("grid,nlat,L,M,m0,B,C", [("legendre-gauss", 32, 32, 17, 0, 1, 4), ("equiangular", 65, 40, 22, 23, 2, 5),
                                                   ("equiangular", 33, 33, 33, 0, 2, 5)])
def test_legendre_references_match_oracle_einsums(grid, nlat, L, M, m0, B, C):
    gen = torch.Generator().manual_seed(3)
    kp, cp = nlat + (-nlat) % 8, C + (-C) % 4
    th, _ = O.precompute_latitudes(nlat, grid)
    P = torch.from_numpy(O.legpoly(m0 + M, L, np.cos(th)))[m0:]          # [M][L][nlat], orders m0 .. m0 + M - 1
    T = torch.zeros(M, L, kp, dtype=torch.float64)
    T[..., :nlat] = P
    # analysis: X [M][2][B][C][kp], padding rows NaN (not part of the sum)
    X = torch.randn(M, 2, B, C, kp, generator=gen, dtype=torch.float64)
    X[..., nlat:] = float("nan")
    ref, mag = E.legendre_analysis_ref(T, X, nlat, cp, m0)
    Xc = torch.complex(X[:, 0, ..., :nlat], X[:, 1, ..., :nlat]).permute(1, 2, 3, 0)          # (B, C, k, m)
    want = torch.einsum("...km,mlk->...lm", Xc, P.to(torch.complex128))                        # (B, C, l, m)
    st = E.stored_mask(L, M, m0)
    got = torch.complex(ref[:, :, 0, :, :C], ref[:, :, 1, :, :C]).permute(2, 3, 0, 1)
    assert torch.allclose(got, torch.where(st, want, 0), rtol=1e-12, atol=1e-12)
    assert (ref[..., C:] == 0).all() and (mag[..., C:] == 0).all()
    assert (ref[E.zero_mask(L, M, m0)].abs() < 1e-12).all(), "P[m][l] = 0 for l < m"
    assert (mag >= ref.abs()).all()
    # synthesis from a spec with NaN in the unstored region
    S = torch.randn(L, M, 2, B, cp, generator=gen, dtype=torch.float64)
    S[~st] = float("nan")
    Z, zmag, K = E.legendre_synthesis_ref(T, S, C, m0)
    Sc = torch.where(st, torch.complex(S[:, :, 0, :, :C], S[:, :, 1, :, :C]).permute(2, 3, 0, 1), 0)   # (B, C, l, m)
    want = torch.einsum("...lm,mlk->...km", Sc, P.to(torch.complex128))                                  # (B, C, k, m)
    got = torch.complex(Z[:, 0, ..., :nlat], Z[:, 1, ..., :nlat]).permute(1, 2, 3, 0)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    assert (Z[..., nlat:] == 0).all()
    assert torch.equal(K.view(-1), st.sum(0).double())
    assert torch.isfinite(zmag).all() and (zmag >= Z.abs()).all()


def test_bound_rejects_one_dropped_term():
    """the bound at the calibrated constant accepts an fp32 evaluation of a 721-term TF32 contraction and rejects the same sum
    with one term of average size left out"""
    gen = torch.Generator().manual_seed(11)
    K, N = 721, 64
    a = E.rand_tf32(N, K, generator=gen)
    b = E.rand_tf32(K, generator=gen)
    ref = a.double() @ b.double()
    mag = a.double().abs() @ b.double().abs()
    got = a @ b                                       # fp32 accumulation
    assert E.bound_ratio(got, ref, mag, K) <= 1.0
    assert E.bound_ratio(E.tf32_rna(got), ref, mag, K, r=E.R_TF32) <= 1.0
    k = int(torch.argsort((a[0] * b).abs())[K // 2])   # a median-size term of row 0
    dropped = got.clone()
    dropped[0] -= a[0, k] * b[k]
    assert E.bound_ratio(dropped, ref, mag, K) > 1.0
    assert E.bound_ratio(E.tf32_rna(dropped), ref, mag, K, r=E.R_TF32) > 1.0
    exact0 = torch.zeros(3, dtype=torch.float64)
    assert E.bound_ratio(torch.tensor([0.0, 0.0, 1e-30]), exact0, exact0, K) == float("inf"), "exact zeros are exact"


# ------------------------------------------------------------------------------------------------ per-mode mixes
# op, L, M, B, G, Ci, Co, dense
PERMODE_REF_CASES = [("diagonal", 9, 9, 2, 2, 4, 6, False), ("diagonal", 9, 9, 3, 1, 3, 5, True), ("sep_diagonal", 9, 9, 2, 2, 6, 6, False),
                     ("sep_dhconv", 40, 35, 3, 1, 5, 5, False), ("sep_dhconv", 9, 9, 2, 2, 6, 6, True)]


@pytest.mark.parametrize("op,L,M,B,G,Ci,Co,dense", PERMODE_REF_CASES)
def test_permode_refs_match_oracle_contraction_and_autograd(op, L, M, B, G, Ci, Co, dense):
    """forward against contractions.py's einsum (oracle.contract_dense) in the native weight layout, dgrad and wgrad against its autograd"""
    g = torch.Generator().manual_seed(17)
    Cig, Cog = Ci // G, Co // G
    shape = {"diagonal": (G, Cig, Cog, L, M), "sep_diagonal": (G, Cig, L, M), "sep_dhconv": (G, Cig, L)}[op]
    w = torch.randn(*shape, dtype=torch.complex128, generator=g)
    cpi, cpo = (Ci + 3) // 4 * 4, (Co + 3) // 4 * 4
    x = torch.randn(L, M, 2, B, cpi, dtype=torch.float64, generator=g)
    gy = torch.randn(L, M, 2, B, cpo, dtype=torch.float64, generator=g)
    keep = E.stored_mask(L, M, 0, dense)[:, :, None, None]
    xo = E.spec_to_complex(x, Ci, dense).permute(2, 3, 0, 1).reshape(B, G, Cig, L, M).requires_grad_(True)
    wo = w.clone().requires_grad_(True)
    y = O.contract_dense(xo, wo, separable=op != "diagonal", operator_type="dhconv" if op == "sep_dhconv" else "diagonal")
    y = torch.where(keep, y.reshape(B, Co, L, M).permute(2, 3, 0, 1), torch.zeros((), dtype=y.dtype))     # [L][M][B][Co]
    ref, mag, K = E.permode_forward_ref(op, x, w, G, Ci, Co, dense)
    assert K == (2 * Cig if op == "diagonal" else 2)
    assert torch.allclose(E.spec_to_complex(ref, Co, dense), y.detach(), atol=1e-12)
    assert (mag >= ref.abs() - 1e-12).all() and (ref[..., Co:] == 0).all()
    gx, gw = torch.autograd.grad(y, [xo, wo], grad_outputs=E.spec_to_complex(gy, Co, dense))
    ref, mag, K = E.permode_dgrad_ref(op, gy, w, G, Ci, Co, dense)
    assert torch.allclose(E.spec_to_complex(ref, Ci, dense), gx.reshape(B, Ci, L, M).permute(2, 3, 0, 1), atol=1e-12)
    assert (mag >= ref.abs() - 1e-12).all()
    ref, mag, K = E.permode_wgrad_ref(op, x, gy, G, Ci, Co, dense)
    assert ref.shape == w.shape and torch.allclose(ref, gw, atol=1e-12)
    assert (mag >= ref.abs() - 1e-12).all()
    if op == "sep_dhconv":
        assert torch.equal(K.view(-1), 2 * B * E.stored_mask(L, M, 0, dense).sum(1).double())


# ---------------------------------------------------------------------------------------------------- ComplexReLU
@pytest.mark.parametrize("mode", E.RELU_MODES)
@pytest.mark.parametrize("bias_kind", ["channel", "scalar", "none"])
def test_complex_relu_ref_matches_finite_differences(mode, bias_kind):
    """the autograd reference against central differences of the oracle's forward, away from its kinks; modulus at z = 0 gives 0 and no gradient"""
    g = torch.Generator().manual_seed(5)
    L, M, B, C, slope = 6, 5, 2, 3, 0.1
    x = torch.randn(L, M, 2, B, 4, dtype=torch.float64, generator=g)
    x[2, 1, :, 0, 1] = 0.0
    gy = torch.randn(L, M, 2, B, 4, dtype=torch.float64, generator=g)
    bias = {"channel": torch.randn(C, dtype=torch.float64, generator=g) * 0.5, "scalar": torch.tensor([0.3], dtype=torch.float64), "none": None}[bias_kind]
    y, gx, gb = E.complex_relu_ref(mode, x, bias, slope, gy, C)
    assert y[2, 1, 0, 1] == 0 and (gx[2, 1, 0, 1] == 0 or mode != "modulus")
    z = E.spec_to_complex(x, C)
    gc = E.spec_to_complex(gy, C)
    bb = 0.0 if bias is None else (bias if bias.numel() > 1 else bias.reshape(()))

    def loss(zz, b):
        zero = (z == 0) & (mode == "modulus")
        return (torch.where(zero, torch.zeros((), dtype=zz.dtype), O.complex_relu(zz, mode, b, slope)) * gc.conj()).real.sum()

    h = 1e-6 * (z != 0)    # along every nonzero entry (z = 0 is a kink of every mode)
    fd = (loss(z + h, bb) - loss(z - h, bb)) / 2e-6 + 1j * (loss(z + 1j * h, bb) - loss(z - 1j * h, bb)) / 2e-6
    assert torch.allclose(gx[z != 0].sum(), fd.to(gx.dtype), rtol=1e-6, atol=1e-6)
    if bias is not None and mode == "modulus":
        fdb = torch.stack([(loss(z, bias + 1e-6 * e) - loss(z, bias - 1e-6 * e)) / 2e-6 for e in torch.eye(bias.numel(), dtype=torch.float64)])
        assert torch.allclose(gb, fdb, rtol=1e-6, atol=1e-6)
    elif bias is not None:
        assert (gb == 0).all()


# --------------------------------------------------------------------------------------------------- instance norm
def test_norm_refs_match_torch():
    g = torch.Generator().manual_seed(9)
    x = torch.randn(3, 4, 50, dtype=torch.float64, generator=g) * 2 + 1
    mean, var = E.norm_stats_ref(x.view(12, 50))
    ref = torch.nn.functional.instance_norm(x, eps=1e-6)
    assert torch.allclose(((x.view(12, 50) - mean[:, None]) / torch.sqrt(var[:, None] + 1e-6)).view(3, 4, 50), ref, atol=1e-12)
    z = torch.linspace(-6, 6, 101, dtype=torch.float64, requires_grad=True)
    assert torch.allclose(E.gelu_ref(z), torch.nn.functional.gelu(z), atol=1e-14)
    (gz,) = torch.autograd.grad(torch.nn.functional.gelu(z).sum(), z)
    assert torch.allclose(E.gelu_grad_ref(z.detach()), gz, atol=1e-14)

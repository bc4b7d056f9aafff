"""CPU checks of the fp64 DFT references (tests/dft_ref.py) the GPU tests of csrc/dft.cu rely on: with exact tables they are numpy's
rfft / irfft, with the tables the plan stores they stay inside the TF32 rounding of those tables, and the analysis bound holds for a
simulation of the kernel's operand rounding (compensated truncation), adversarial inputs included."""
import numpy as np
import pytest
import torch

import dft_ref as D
import engine_ref as E

# (nlon, mmax): every length class of the GPU tests -- N2 = 180, 90, 60 (compile-time analysis kernels), 156, 182, 189 (largest),
# 16, 32, 12, 2, 9, 45, 39 (odd); Nyquist (mmax = nlon / 2 + 1), mmax % 8 != 0, mmax < 8
CASES = [(1440, 241), (720, 121), (480, 241), (1248, 189), (1456, 256), (1512, 256), (128, 65), (256, 100), (96, 49), (16, 9),
         (72, 37), (360, 100), (312, 149), (64, 5), (96, 7)]
R, NLAT = 2, 3


def _rows(nlon, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(R, NLAT, nlon, generator=g, dtype=torch.float64)


def _spec(mmax, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(mmax, 2, R, NLAT, generator=g, dtype=torch.float64)


def _np_analysis(x, mmax, mode, rs):
    X = np.fft.rfft(x.numpy(), axis=-1)[..., :mmax]
    if mode == 0:
        return torch.from_numpy(X * rs.numpy()[None, :, None])
    sc = np.full(mmax, 2.0)
    sc[0] = 1.0
    if mmax - 1 == x.shape[-1] // 2:
        sc[-1] = 1.0
    return torch.from_numpy(X * sc)


def _np_synthesis(Z, nlon, mode, rs, bias):
    mmax = Z.shape[0]
    zc = (Z[:, 0] + 1j * Z[:, 1]).permute(1, 2, 0).numpy()   # [R][K][mmax]
    if mode == 0:
        full = np.zeros(zc.shape[:-1] + (nlon // 2 + 1,), dtype=np.complex128)
        full[..., :mmax] = zc
        return torch.from_numpy(np.fft.irfft(full, n=nlon, axis=-1) * nlon + bias.numpy()[:, None, None])
    j = np.arange(nlon)
    ph = np.exp(2j * np.pi * np.arange(mmax)[:, None] * j[None, :] / nlon)
    return torch.from_numpy((zc @ ph).real * rs.numpy()[None, :, None])


@pytest.mark.parametrize("nlon,mmax", CASES)
@pytest.mark.parametrize("mode", [0, 1])
def test_references_are_rfft_irfft_with_exact_tables(nlon, mmax, mode):
    rs = torch.linspace(0.3, 1.7, NLAT, dtype=torch.float64)
    bias = torch.tensor([0.25, -1.5], dtype=torch.float64)
    x = _rows(nlon, nlon + mode)
    ref, _, _ = D.analysis_ref(x, mmax, mode, rs, rounded=False)
    want = _np_analysis(x, mmax, mode, rs)
    assert (ref - want).abs().max() <= 1e-12 * want.abs().max()
    Z = _spec(mmax, 3 * nlon + mode)
    y, _ = D.synthesis_ref(Z, nlon, mode, rs, bias if mode == 0 else None, C=2, rounded=False)
    want = _np_synthesis(Z, nlon, mode, rs, bias)
    assert (y - want).abs().max() <= 1e-12 * want.abs().max()


@pytest.mark.parametrize("nlon,mmax", CASES)
@pytest.mark.parametrize("mode", [0, 1])
def test_rounded_tables_stay_within_their_tf32_rounding(nlon, mmax, mode):
    """E rounded to TF32 (relative 2^-11) and fp32 twiddles (2^-24): the rounded-table references differ from rfft / irfft by at
    most (2^-11 + 2^-22) times the sum of magnitudes -- and they do differ (the GPU bounds could not tell them apart otherwise)"""
    rs = torch.linspace(0.3, 1.7, NLAT, dtype=torch.float64)
    extra = 2.0 ** -11 + 2.0 ** -22
    x = _rows(nlon, 5 * nlon + mode)
    ref, mag, _ = D.analysis_ref(x, mmax, mode, rs)
    exact = _np_analysis(x, mmax, mode, rs)
    assert E.bound_ratio(ref, exact, mag, 0, extra=extra) <= 1.0
    Z = _spec(mmax, 7 * nlon + mode)
    bias = torch.tensor([0.5, 2.0], dtype=torch.float64)
    y, ymag = D.synthesis_ref(Z, nlon, mode, rs, bias if mode == 0 else None, C=2)
    exact = _np_synthesis(Z, nlon, mode, rs, bias)
    assert E.bound_ratio(y, exact, ymag, 0, extra=extra) <= 1.0
    if nlon >= 64:
        assert not torch.equal(y, exact)


def _adversarial_rows(nlon, seed):
    """rows whose GEMM operands sit just below a TF32 step after the compensation (the worst truncation), plus rows of mixed
    binades with a strong mean (large class-0 operands next to small ones)"""
    N2 = nlon // 8
    g = torch.Generator().manual_seed(seed)
    steps = torch.randint(0, 1024, (N2,), generator=g).double()
    e = torch.randint(-3, 4, (N2,), generator=g).double()
    v = (1.0 + steps * 2.0 ** -10 + (2.0 ** -10 - 2.0 ** -22) / D.TRUNC_COMP) * torch.exp2(e) / 8.0
    v[N2 // 2 + 1 :] = 0.0   # partner columns zero: Ye = Yo = 8 v (class 0 only)
    per = v.repeat(8)                                                         # period N2: only orders m = 0 mod 8
    mixed = torch.randn(nlon, generator=g, dtype=torch.float64) * torch.exp2(torch.randint(-8, 8, (nlon,), generator=g).double()) + 3.0
    return torch.stack([per.float().double(), mixed.float().double()]).view(2, 1, nlon)


@pytest.mark.parametrize("nlon,mmax", CASES)
@pytest.mark.parametrize("mode", [0, 1])
def test_analysis_bound_holds_for_the_simulated_rounding(nlon, mmax, mode):
    rs = torch.linspace(0.3, 1.7, NLAT, dtype=torch.float32).double()
    for kind, x in (("random", _rows(nlon, 11 * nlon + mode).float().double()), ("adversarial", _adversarial_rows(nlon, nlon + mode))):
        r = rs[: x.shape[1]]
        ref, mag, tmag = D.analysis_ref(x, mmax, mode, r)
        sim = D.simulate_analysis(x, mmax, mode, r)
        ratio = E.bound_ratio(sim, ref, mag, D.gemm_len(mmax), r=D.R_OUT, c=D.C_DFT, floor=D.analysis_floor(ref, tmag))
        assert ratio <= 1.0, (kind, ratio)
        assert torch.equal(E.tf32_trunc(torch.view_as_real(sim).float()).double(), torch.view_as_real(sim))


@pytest.mark.parametrize("nlon,mmax", [(1440, 241), (480, 241), (128, 65), (72, 37), (1512, 256)])
def test_simulated_rounding_is_unbiased(nlon, mmax):
    """the compensated truncation has gain 1 within 1e-4 per class; leaving out the compensation (plain truncation) or keeping the
    scaled fp32 value (the stored value without the final truncation) moves it by about -3.5e-4 / +3.3e-4"""
    x = torch.randn(8, 16, nlon, generator=torch.Generator().manual_seed(nlon), dtype=torch.float32).double()
    for mode in (0, 1):
        rs = torch.linspace(0.3, 1.7, 16, dtype=torch.float32).double()
        ref, _, _ = D.analysis_ref(x, mmax, mode, rs)
        sim = D.simulate_analysis(x, mmax, mode, rs)
        for c in range(8):
            gn = D.gain(sim[..., c::8], ref[..., c::8])
            assert abs(gn - 1.0) <= 1e-4, (mode, c, gn)
        assert abs(D.gain(ref * D.TRUNC_COMP, ref) - 1.0 - (D.TRUNC_COMP - 1.0)) < 1e-12
        plain = torch.complex(E.tf32_trunc(ref.real.float()).double(), E.tf32_trunc(ref.imag.float()).double())
        assert D.gain(plain, ref) - 1.0 < -2e-4

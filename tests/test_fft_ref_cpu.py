"""The fp64 references of the longitude FFT (tests/fft_ref.py) on the CPU: against numpy's rfft / irfft and an explicit sum, against the
adjoint identity between the mode-0 analysis and the mode-1 synthesis, and on the run-time kernels' own butterfly and split arithmetic
(b200sht_debug_fft_host runs `stage_butterfly` / `split_pair` of csrc/fft.cu on the host) at the lengths the GPU rows use: the pair bound
holds for it, the own-row bound does not when a small row shares a pair with a large one, and the DC order of constant rows is exact for
every radix."""
import ctypes

import numpy as np
import pytest
import torch

import engine_ref as E
import fft_ref as F
from makani_b200 import _lib
from test_gpu_fft import ROWS, nstages

RT_LENGTHS = sorted({r[2] for r in ROWS if r[8] not in ("T", "F")})


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _rs(nlat, gen):
    return (torch.rand(nlat, generator=gen, dtype=torch.float64) * 0.01 + 1e-4).float()


@pytest.mark.parametrize("N,mmax", [(2, 1), (2, 2), (3, 1), (3, 2), (4, 3), (15, 8), (16, 9), (16, 5), (45, 23), (210, 106), (1440, 241), (1440, 721)])
@pytest.mark.parametrize("mode", [0, 1])
def test_analysis_ref_matches_numpy(N, mmax, mode):
    gen = torch.Generator().manual_seed(N + mmax)
    x = torch.randn(2, 5, N, generator=gen)
    rs = _rs(5, gen)
    ref, mag = F.analysis_ref(x, mmax, mode, rs)
    X = np.fft.rfft(x.double().numpy(), axis=-1)[..., :mmax]
    if mode == 0:
        X = X * rs.double().numpy()[:, None]
    else:
        s = np.full(mmax, 2.0)
        s[0] = 1.0
        if N % 2 == 0 and mmax == N // 2 + 1:
            s[-1] = 1.0
        X = X * s
    assert np.abs(ref.numpy() - X).max() <= 1e-12 * np.abs(X).max()
    # the magnitude bounds every part of the result; the pair magnitude bounds the own-row one
    _, pmag = F.analysis_ref(x, mmax, mode, rs, paired=True)
    assert ref.shape == mag.shape == pmag.shape
    assert (ref.real.abs() <= mag * (1 + 1e-12)).all() and (ref.imag.abs() <= mag * (1 + 1e-12)).all()
    assert (pmag >= mag).all()
    assert torch.equal(pmag[:, 4], mag[:, 4])   # the last row of an odd count pairs with a zero row


def _explicit_synthesis(Z, N, mode, rs, bias, C):
    """y[r][k][j] = sum_m w_m f_m (Re Z_m cos(2 pi m j / N) - Im Z_m sin(2 pi m j / N)) (+ bias): f_m = 1 at DC and Nyquist (Im ignored),
    2 otherwise; w_m = 1/2 for 0 < m < N/2 in mode 1, times rs[k]"""
    mmax, _, R, K = Z.shape
    m = np.arange(mmax)[:, None]
    j = np.arange(N)[None, :]
    selfc = ((m == 0) | (2 * m == N))[:, 0]
    f = np.where(selfc, 1.0, 2.0) * (np.where(selfc, 1.0, 0.5) if mode == 1 else 1.0)
    zr = Z[:, 0].double().numpy()
    zi = np.where(selfc[:, None, None], 0.0, Z[:, 1].double().numpy())
    cs, sn = np.cos(2 * np.pi * m * j / N), np.sin(2 * np.pi * m * j / N)
    y = np.einsum("m,mrk,mj->rkj", f, zr, cs) - np.einsum("m,mrk,mj->rkj", f, zi, sn)
    if mode == 1:
        y = y * rs.double().numpy()[None, :, None]
    if bias is not None:
        y = y + np.tile(bias.double().numpy(), R // C)[:, None, None]
    return y


@pytest.mark.parametrize("N,mmax", [(2, 1), (2, 2), (3, 2), (4, 3), (15, 8), (16, 9), (16, 5), (45, 23), (210, 106), (1440, 241)])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("with_bias", [False, True])
def test_synthesis_ref_matches_an_explicit_sum(N, mmax, mode, with_bias):
    gen = torch.Generator().manual_seed(3 * N + mmax)
    R, K, C = 6, 3, 3
    Z = torch.randn(mmax, 2, R, K, generator=gen)
    rs = _rs(K, gen)
    bias = torch.randn(C, generator=gen) if with_bias else None
    ref, mag = F.synthesis_ref(Z, N, mode, rs, bias, C)
    want = _explicit_synthesis(Z, N, mode, rs, bias, C)
    assert np.abs(ref.numpy() - want).max() <= 1e-12 * max(1.0, np.abs(want).max())
    assert (ref.abs() <= mag * (1 + 1e-12)).all()
    # numpy's irfft (norm="forward") in mode 0 without a bias
    if mode == 0 and not with_bias:
        z = (Z[:, 0].double() + 1j * Z[:, 1].double()).permute(1, 2, 0).numpy()
        full = np.zeros((R, K, N // 2 + 1), dtype=np.complex128)
        full[..., :mmax] = z
        full[..., 0] = full[..., 0].real
        if N % 2 == 0 and mmax == N // 2 + 1:
            full[..., -1] = full[..., -1].real
        assert np.abs(ref.numpy() - np.fft.irfft(full, n=N, axis=-1, norm="forward")).max() <= 1e-12 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("N,mmax", [(2, 2), (3, 2), (15, 8), (16, 9), (16, 5), (210, 106), (1440, 241), (1440, 721)])
def test_mode1_synthesis_is_the_adjoint_of_mode0_analysis(N, mmax):
    """<A x, Z> = <x, A^T Z> with A the mode-0 analysis and A^T the mode-1 synthesis (real inner products over re / im planes)"""
    gen = torch.Generator().manual_seed(N)
    R, K = 2, 5
    x = torch.randn(R, K, N, generator=gen, dtype=torch.float64)
    Z = torch.randn(mmax, 2, R, K, generator=gen, dtype=torch.float64)
    rs = _rs(K, gen)
    X, _ = F.analysis_ref(x, mmax, 0, rs)
    lhs = (X.real * Z[:, 0].permute(1, 2, 0) + X.imag * Z[:, 1].permute(1, 2, 0)).sum()
    y, _ = F.synthesis_ref(Z, N, 1, rs)
    rhs = (x * y).sum()
    assert abs(float(lhs - rhs)) <= 1e-12 * max(1.0, float((X.abs() * Z.abs().amax()).sum()))


# ------------------------------------------------------------------------------------ the run-time kernels' host arithmetic
def host_analysis(a, b, mmax):
    """b200sht_debug_fft_host direction 0: two rows packed as a + i b -> their unscaled half spectra (complex64 [2][mmax])"""
    N = a.shape[-1]
    out = np.zeros((2, 2 * mmax), dtype=np.float32)
    a, b = np.ascontiguousarray(a, dtype=np.float32), np.ascontiguousarray(b, dtype=np.float32)
    o0, o1 = out[0].copy(), out[1].copy()
    assert _lib.load().b200sht_debug_fft_host(N, mmax, 0, _p(a), _p(b), _p(o0), _p(o1)) == 0
    return np.stack([o0.view(np.complex64), o1.view(np.complex64)])


def host_synthesis(za, zb, N):
    """direction 1: two half spectra (complex64 [mmax]) -> rows (float32 [2][N]), irfft(norm="forward")"""
    ya, yb = np.zeros(N, dtype=np.float32), np.zeros(N, dtype=np.float32)
    za, zb = np.ascontiguousarray(za, dtype=np.complex64), np.ascontiguousarray(zb, dtype=np.complex64)
    assert _lib.load().b200sht_debug_fft_host(N, za.shape[0], 1, _p(za.view(np.float32)), _p(zb.view(np.float32)), _p(ya), _p(yb)) == 0
    return np.stack([ya, yb])


def _host_needs(N, sa, sb, seed):
    """(needed c with the pair magnitude, with the own-row magnitude) of the host analysis and synthesis on rows of scales sa, sb"""
    rng = np.random.default_rng(seed)
    mmax = N // 2 + 1
    K = F.fft_len(nstages(N)[0])
    x = torch.from_numpy((rng.standard_normal((1, 2, N)) * np.array([sa, sb])[None, :, None]).astype(np.float32))
    got = torch.from_numpy(host_analysis(x[0, 0].numpy(), x[0, 1].numpy(), mmax))[None]
    ana = []
    for paired in (True, False):
        ref, mag = F.analysis_ref(x, mmax, 1, paired=paired)
        ref, mag = ref / F.mode_scale(N, mmax), mag / F.mode_scale(N, mmax)   # the host emulation does not scale
        ana.append(E.needed_c(got, ref, mag, K))
    Z = torch.from_numpy((rng.standard_normal((mmax, 2, 1, 2)) * np.array([sa, sb])).astype(np.float32))
    zc = (Z[:, 0, 0].numpy() + 1j * Z[:, 1, 0].numpy()).astype(np.complex64)   # [mmax][2 rows]
    y = torch.from_numpy(host_synthesis(zc[:, 0], zc[:, 1], N))[None]
    syn = []
    for paired in (True, False):
        ref, mag = F.synthesis_ref(Z, N, 0, paired=paired)
        syn.append(E.needed_c(y, ref, mag, K))
    return ana, syn


@pytest.mark.parametrize("N", RT_LENGTHS)
def test_host_arithmetic_within_the_pair_bound(N):
    for sa, sb in ((1.0, 1.0), (1.0, 2.0 ** -20), (2.0 ** -20, 1.0)):
        (ana, _), (syn, _) = _host_needs(N, sa, sb, N)
        print(f"[fft host] N={N} scales {sa:g}/{sb:g}: pair bound needs c >= {ana:.3e} (analysis), {syn:.3e} (synthesis)")
        assert ana <= F.C_FFT and syn <= F.C_FFT


@pytest.mark.parametrize("N", [1001, 2002, 8192])
def test_host_arithmetic_breaks_the_own_row_bound_of_a_small_partner(N):
    """a row of scale 2^-20 packed with a row of scale 1: its spectrum carries the rounding error of the large row, far beyond a bound
    on its own magnitude; that is why the run-time kernels are held to the pair magnitude"""
    (_, own), (_, own_s) = _host_needs(N, 1.0, 2.0 ** -20, 5 * N)
    print(f"[fft host] N={N}: own-row bound of the small row needs c >= {own:.3e} (analysis), {own_s:.3e} (synthesis)")
    assert own > 100 * F.C_FFT and own_s > 100 * F.C_FFT


def _lengths_for_every_radix():
    rad = {}
    for N in RT_LENGTHS:
        for r in nstages(N)[1]:
            rad.setdefault(r, N)
    return sorted(set(rad.values()))


@pytest.mark.parametrize("N", _lengths_for_every_radix())
def test_host_dc_of_constant_rows_is_exact(N):
    """constant rows of small integers: order 0 is N c exactly (a sum of integers, twiddle 1 only) and has no imaginary part; DC-only
    spectra give constant rows c exactly"""
    for ca, cb in ((3.0, -4.0), (-1.0, 2.0), (4.0, 4.0)):
        X = host_analysis(np.full(N, ca), np.full(N, cb), 1)
        assert X[0, 0] == np.complex64(N * ca) and X[1, 0] == np.complex64(N * cb), (N, ca, cb, X[:, 0])
        y = host_synthesis(np.array([ca + 7j]), np.array([cb - 5j]), N)
        assert (y[0] == ca).all() and (y[1] == cb).all(), (N, ca, cb)

"""makani_b200.noise on the GPU (csrc/noise.cu) against makani's own classes (tests/golden/noise_golden.npz) and torch's elementwise sequences:

* the update kernel on the golden (state, xi) gives makani's state bit for bit in the AR step, in the memoryless update and in the stationary
  redraw of T = 1; the stationary redraw of T > 1 (an fp32 FMA discount sum) against fp64 of the same operands, per element within
  (T + 4) 2^-24 sum_q |discount[t][q] w[q]|: the T - 1 FMA roundings of the sum, the rounding of sigma xi, and the ~3 of sqrt and the division
  that step 0 carries;
* the module draws makani's shapes in makani's order from its generator (a same-seeded generator replaying them ends in the same state), and its
  state is the kernel applied to those draws, and for T = 1 torch's elementwise sequence of makani;
* the spectrum is bit for bit torch's `torch.complex(...) * sigma_l` (CUDA divides by math.sqrt(2) as a multiply by the fp32 reciprocal)
  followed by the pack, compared as int32 bit patterns so that signed zeros count, at the golden geometries and at the shipped one;
* a CUDA module cast to another dtype is refused before it draws;
* forward() against the golden fields: rtol 2e-5 at fp32, relative L2 2e-3 at TF32;
* the learnable isotropic sigma's gradient against fp64 of the operands the kernel reads (the packed gradient of the synthesis backward and
  state / sqrt 2), per element within 2 K 2^-24 sum |terms| (K = B T C: one FMA chain of 2 K terms), and bit-identical on a rerun;
* at the shipped shape (721 x 1440, lmax 721, 8 channels) what makani's tests/test_noise.py asserts: the isotropic field's variance sigma^2 and
  zero mean, the diffusion noise's lag-one correlation phi; and the diffusion state's stationary variance sigma_l^2 / (1 - phi^2) after the
  redraw and after AR steps;
* h x w on virtual ranks (2 x 1, 1 x 2, 2 x 2): every rank's sigma / phi is the slice of the serial module's, and the ranks' spectra of a
  scattered global state, through the virtual-rank inverse SHT of tests/test_gpu_distributed_sht.py, give the serial forward at fp32: bit for
  bit when the latitudes are not split (h = 1), else within that file's single-GPU bound (rtol 2e-5), because nlon = 32 runs on the runtime
  FFT plan, which transforms two real rows as one complex sequence, and a latitude shard of 17 rows pairs different rows than the whole grid.
Run with -s to see the worst ratio of every bounded comparison.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

import makani_b200 as mb
import makani_b200.distributed as mbd
from makani_b200 import _lib
from makani_b200 import noise as mn
from makani_b200.sht import _SpecPack, _ptr, _stream
from test_gpu_distributed_sht import _vs_single, emulated_isht
from test_gpu_parity import close
from test_gpu_vector_sht import rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "noise_golden.npz"))
CASES = sorted({k.split("/")[0] for k in GOLD.files})
SHIPPED_KT = [3.0806e-5, 1.2322e-4, 4.9289e-4, 1.9716e-3, 7.8862e-3, 3.1545e-2, 1.2618e-1, 5.0472e-1]
U = 2.0 ** -24


def meta(case):
    return json.loads(str(GOLD[f"{case}/meta"]))


def gold(case, key):
    return torch.from_numpy(GOLD[f"{case}/{key}"])


def build(case):
    m = meta(case)
    kw = dict(m["kwargs"])
    kw["img_shape"] = tuple(kw["img_shape"])
    return (mn.build_noise(**kw) if m["how"] == "build_noise" else getattr(mn, m["how"])(**kw)).to(DEV)


SPECTRAL = [c for c in CASES if meta(c)["cls"] != "DummyNoiseS2"]
UPDATES = [(c, k.split("/")[2]) for c in SPECTRAL for k in GOLD.files if k.startswith(f"{c}/upd/") and k.endswith("/after")]


def kernel_update(state, xi, mode, reflect, sigma=None, phi=None, discount=None):
    """b200sht_noise_update on a copy of `state`"""
    s = state.to(DEV).contiguous().clone()
    B, T, C, L, M, _ = s.shape
    args = [None if t is None else t.to(DEV).contiguous() for t in (xi, sigma, phi, discount)]
    _lib.call("b200sht_noise_update", _ptr(s), *[_ptr(t) for t in args], B, T, C, L, M, mode, int(reflect), _stream(DEV))
    return s


def golden_update(case, mode):
    m, s0, xi = meta(case), gold(case, "state0"), gold(case, f"upd/{mode}/xi")
    reflect = m["attrs"]["reflect"]
    if mode == "base":
        return kernel_update(s0, xi, _lib.NOISE_BASE, reflect)
    disc = gold(case, "t/discount") if f"{case}/t/discount" in GOLD.files else None
    code = _lib.NOISE_STATIONARY if mode == "stationary" else _lib.NOISE_AR
    return kernel_update(s0, xi, code, reflect, gold(case, "t/sigma_l"), gold(case, "t/phi"), disc if code == _lib.NOISE_STATIONARY else None)


@pytest.mark.parametrize("case,mode", UPDATES)
def test_update_kernel_matches_makani(case, mode):
    after = golden_update(case, mode).cpu()
    want = gold(case, f"upd/{mode}/after")
    T = want.shape[1]
    if mode != "stationary" or T == 1:
        assert torch.equal(after, want), f"{case} {mode}: not bit-identical to makani's update"
        return
    # T > 1 stationary redraw: fp64 of the same operands
    s, p, D = gold(case, "t/sigma_l").double(), gold(case, "t/phi").double(), gold(case, "t/discount").double()
    r = -1.0 if meta(case)["attrs"]["reflect"] else 1.0
    w = r * s * gold(case, f"upd/{mode}/xi").double()
    w[:, 0] = w[:, 0] / torch.sqrt(1.0 - p**2)
    ref = torch.einsum("ctr,brclmu->btclmu", D, w)
    terms = torch.einsum("ctr,brclmu->btclmu", D.abs(), w.abs())
    ratio = ((after.double() - ref).abs() / ((T + 4) * U * terms).clamp_min(1e-300)).max().item()
    print(f"[noise] {case} stationary T={T}: worst error / bound {ratio:.3f}")
    assert ratio <= 1.0
    close(after, want, 1e-6, f"{case} stationary vs makani's CPU einsum")


def _torch_update(state, xi, replace, sigma, phi, reflect):
    """makani's DiffusionNoiseS2.update of T = 1, as torch computes it on the GPU"""
    eta = sigma * xi
    if reflect:
        eta = -eta
    if not replace:
        return phi * state + eta
    eta[:, 0, ...] = eta[:, 0, ...] / torch.sqrt(1.0 - phi**2)
    return eta


@pytest.mark.parametrize("reflect", [False, True])
def test_module_draws_and_state(reflect):
    """a sequence of updates (with a batch resize) against a same-seeded CUDA generator drawing makani's shapes in makani's order"""
    n = mn.DiffusionNoiseS2((17, 32), 2, 8, kT=SHIPPED_KT, lambd=1.0, seed=333, reflect=reflect).to(DEV)
    g = mn.IsotropicGaussianRandomFieldS2((17, 32), 2, 3, alpha=2.0, seed=335, reflect=reflect).to(DEV)
    rn, rg = torch.Generator(device=DEV), torch.Generator(device=DEV)
    rn.manual_seed(333)
    rg.manual_seed(335)
    L, M = n.lmax_local, n.mmax_local
    for step, (replace, B) in enumerate([(True, 2), (False, 2), (False, 2), (True, 3), (False, 3)]):
        before_n = n.get_tensor_state()
        n.update(replace_state=replace, batch_size=B)
        g.update(replace_state=replace, batch_size=B)
        if before_n.shape[0] != B:
            before_n = torch.zeros_like(n.state)
        xi_n = torch.empty((B, 1, 8, L, M, 2) if not replace else tuple(n.state.shape), device=DEV).normal_(mean=0.0, std=1.0, generator=rn)
        xi_g = torch.empty(tuple(g.state.shape), device=DEV).normal_(mean=0.0, std=1.0, generator=rg)
        code = _lib.NOISE_STATIONARY if replace else _lib.NOISE_AR
        assert torch.equal(n.state, kernel_update(before_n, xi_n, code, reflect, n.sigma_l, n.phi)), f"step {step}: diffusion state"
        assert torch.equal(n.state, _torch_update(before_n, xi_n, replace, n.sigma_l, n.phi, reflect)), f"step {step}: vs torch's sequence"
        assert torch.equal(g.state, -xi_g if reflect else xi_g), f"step {step}: isotropic state"
    assert torch.equal(n.get_rng_state()[1], rn.get_state()) and torch.equal(g.get_rng_state()[1], rg.get_state())


def _torch_spectrum(m):
    """makani's forward up to the synthesis input, as torch computes it on the GPU: complex (B, T C, L, M)"""
    if isinstance(m, mn.IsotropicGaussianRandomFieldS2):
        _s = m.state / math.sqrt(2)
        c = torch.complex(_s[..., 0], _s[..., 1]) * m.sigma_l
    else:
        c = torch.complex(m.state[..., 0], m.state[..., 1])
    return c.reshape(m.state.shape[0], m.num_time_steps * m.num_channels, m.lmax_local, m.mmax_local)


def _written(L, M, B, cp):
    """mask of the packed entries the pack writes: l >= lstart(m), every channel slot"""
    l, m = torch.arange(L).reshape(-1, 1), torch.arange(M)
    return (l >= (m // 32) * 32).reshape(L, M, 1, 1, 1).expand(L, M, 2, B, cp).to(DEV)


def _check_spectrum(m, tag):
    ref = _torch_spectrum(m)
    B, TC, L, M = ref.shape
    cp = (TC + 3) // 4 * 4
    sigma = m.sigma_l if isinstance(m, mn.IsotropicGaussianRandomFieldS2) else None
    spec = mn._NoiseSpectrum.apply(m.state, sigma, True).view(L, M, 2, B, cp)
    want = _SpecPack.apply(ref).view(L, M, 2, B, cp)
    mask = _written(L, M, B, cp)
    # int32 bit patterns: the sign of the zeros where sigma_l = 0 (m > l) counts too
    assert torch.equal(spec.view(torch.int32)[mask], want.view(torch.int32)[mask]), f"{tag}: packed spectrum not torch's bits"
    coeffs = mn._NoiseSpectrum.apply(m.state, sigma, False)
    assert torch.equal(torch.view_as_real(coeffs).view(torch.int32), torch.view_as_real(ref).view(torch.int32)), f"{tag}: complex spectrum"


@pytest.mark.parametrize("case", SPECTRAL)
def test_spectrum_matches_torch(case):
    m = build(case)
    m.set_tensor_state(gold(case, "state0"))
    _check_spectrum(m, case)


@pytest.mark.parametrize("cast", ["half", "double"])
def test_cast_cuda_module_is_refused(cast):
    n = getattr(mn.DiffusionNoiseS2((17, 32), 2, 8, kT=SHIPPED_KT, seed=333).to(DEV), cast)()
    rng = n.get_rng_state()[1]
    for call in (lambda: n.update(), lambda: n.update(replace_state=True), lambda: n()):
        with pytest.raises(mb.B200ShtError, match="float32 only"):
            call()
    assert torch.equal(n.get_rng_state()[1], rng) and bool((n.state == 0).all())


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("case", SPECTRAL)
def test_forward_matches_golden(case, precision):
    m = build(case)
    m.isht.precision = precision
    m.set_tensor_state(gold(case, "state0"))
    y = m()
    want = gold(case, "y")
    assert y.dtype == torch.float32 and tuple(y.shape) == tuple(want.shape)
    if precision == "fp32":
        close(y, want, 2e-5, f"{case} forward fp32")
    else:
        r = rel_l2(y, want)
        print(f"[noise] {case} forward TF32 relative L2 {r:.3e}")
        assert r < 2e-3
    with torch.autocast("cuda", dtype=torch.bfloat16):
        assert m().dtype == torch.float32


@pytest.mark.parametrize("packed", [True, False])
@pytest.mark.parametrize("case", [c for c in SPECTRAL if f"{c}/dsigma" in GOLD.files])
def test_sigma_grad(case, packed):
    m = build(case)
    m.isht.precision = "fp32"
    s0, g = gold(case, "state0").to(DEV), gold(case, "g").to(DEV)
    m.set_tensor_state(s0)
    B, T, C, L, M, _ = s0.shape
    TC, K = T * C, B * T * C
    if packed:
        y = m()
        y.backward(g)
        dsigma = m.sigma_l.grad.clone()
        # the operand the kernel read: the packed gradient of the synthesis backward
        spec = mn._NoiseSpectrum.apply(m.state, m.sigma_l.detach(), True).detach().requires_grad_(True)
        m.isht.forward_packed(spec, B, TC, torch.float32).backward(g.reshape(B, TC, *g.shape[-2:]))
        cp = (TC + 3) // 4 * 4
        gs = spec.grad.view(L, M, 2, B, cp)[..., :TC].permute(3, 4, 0, 1, 2).double()       # (B, TC, L, M, 2)
        tri = torch.tril(torch.ones(L, M, device=DEV, dtype=torch.bool)).reshape(1, 1, L, M, 1)
        gs = torch.where(tri, gs, 0.0)     # l < m: not stored (l < lstart(m)) or zero; the kernel writes 0 there
        close(dsigma, gold(case, "dsigma"), 2e-5, f"{case} dsigma vs makani")
        m.sigma_l.grad = None
        m().backward(g)
        assert torch.equal(m.sigma_l.grad, dsigma), f"{case}: dsigma not bit-identical on a rerun"
    else:
        gs = torch.randn(B, TC, L, M, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(3))
        dsigma = torch.empty(1, 1, 1, L, M, device=DEV)
        _lib.call("b200sht_noise_sigma_grad", _ptr(m.state), _ptr(gs), _ptr(dsigma), B, TC, L, M, 0, _stream(DEV))
        gs = gs.double()
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(math.sqrt(2), dtype=torch.float32)
    z = (m.state * inv.to(DEV)).reshape(B, TC, L, M, 2).double()
    ref = (gs * z).sum(dim=(0, 1, 4))
    bound = 2 * K * U * (gs * z).abs().sum(dim=(0, 1, 4))
    ratio = ((dsigma.reshape(L, M).double() - ref).abs() / bound.clamp_min(1e-300)).max().item()
    print(f"[noise] {case} dsigma ({'packed' if packed else 'complex'} gradient): worst error / bound {ratio:.3f}")
    assert ratio <= 1.0


def test_shipped_shape_statistics():
    """721 x 1440, lmax 721, 8 channels: the FCN3 input noise runs with makani_b200 alone; makani's statistical assertions"""
    n = mn.DiffusionNoiseS2((721, 1440), 1, 8, kT=SHIPPED_KT, lambd=1.0, seed=333).to(DEV)
    n.update(replace_state=True)
    y = n()
    assert y.dtype == torch.float32 and tuple(y.shape) == (1, 1, 8, 721, 1440) and bool(torch.isfinite(y).all())
    _check_spectrum(n, "shipped diffusion")
    # stationary variance of the state, sigma_l^2 / (1 - phi^2) per (c, l) over m <= l, after the redraw and after AR steps
    # (m > l entries carry the same law; the synthesis ignores them)
    var = n.sigma_l.double() ** 2 / (1 - n.phi.double() ** 2)
    # sigma_l underflows at high degrees of the smooth channels: only coefficients of a normal fp32 sigma_l^2 count
    tri = torch.tril(torch.ones(721, 721, device=DEV, dtype=torch.bool)).reshape(1, 1, 1, 721, 721, 1) & (var > 1e-60)
    tri = tri.expand_as(n.state)
    for k in range(3):
        z = (n.state.double() ** 2 / var)[tri]
        print(f"[noise] shipped diffusion after {k} AR steps: normalised state variance {z.mean().item():.4f}")
        assert abs(z.mean().item() - 1.0) < 0.01
        before = n.get_tensor_state()
        n.update()
    x, yv = before.reshape(-1), n.state.reshape(-1)
    corr = torch.corrcoef(torch.stack([x, yv]))[0, 1].item()
    print(f"[noise] shipped diffusion lag-one correlation {corr:.4f} (phi {math.exp(-1.0):.4f})")
    assert abs(corr - math.exp(-1.0)) < 0.05

    g = mn.IsotropicGaussianRandomFieldS2((721, 1440), 4, 8, sigma=2.0, seed=333).to(DEV)
    g.isht.precision = "fp32"
    g.update()
    _check_spectrum(g, "shipped isotropic")
    out = g()
    print(f"[noise] shipped isotropic field: variance {out.var().item():.4f} (sigma^2 4), mean {out.mean().item():.2e}")
    assert abs(out.var().item() - 4.0) < 0.5 and abs(out.mean().item()) < 0.2


# ------------------------------------------------------------------------------------------------------------------ h x w virtual ranks
class _VirtualGrid:
    """makani_b200.distributed answering as rank (ih, iw) of an h x w grid"""

    def __init__(self, monkeypatch, h, w, ih, iw):
        mbd.init(object(), object())
        for name, v in (("polar_group_size", h), ("azimuth_group_size", w), ("polar_group_rank", ih), ("azimuth_group_rank", iw)):
            monkeypatch.setattr(mbd, name, lambda v=v: v)


GRIDS = [(2, 1), (1, 2), (2, 2)]
VR_CASES = ["diffusion_shipped", "diffusion_t3", "grf_alpha2_learnable_lg", "grf_alpha2_lmax12"]


@pytest.mark.parametrize("hw", GRIDS, ids=lambda hw: f"{hw[0]}x{hw[1]}")
@pytest.mark.parametrize("case", VR_CASES)
def test_virtual_ranks(case, hw, monkeypatch):
    h, w = hw
    serial = build(case)
    serial.isht.precision = "fp32"
    s0 = gold(case, "state0").to(DEV)
    serial.set_tensor_state(s0)
    want = serial()
    B, T, C, L, M, _ = s0.shape
    isotropic = isinstance(serial, mn.IsotropicGaussianRandomFieldS2)
    ls, ms = mbd.compute_split_shapes(L, h), mbd.compute_split_shapes(M, w)
    cols = []
    try:
        for iw in range(w):
            col = []
            for ih in range(h):
                with monkeypatch.context() as mp:
                    _VirtualGrid(mp, h, w, ih, iw)
                    r = build(case)
                assert isinstance(r.isht, mbd.DistributedInverseRealSHT) and r._distributed
                assert (r.lmax_local, r.mmax_local) == (ls[ih], ms[iw]) and (r.lmax, r.mmax) == (L, M)
                l0, m0 = sum(ls[:ih]), sum(ms[:iw])
                if isotropic:
                    assert torch.equal(r.sigma_l, serial.sigma_l[..., l0:l0 + ls[ih], m0:m0 + ms[iw]])
                else:
                    assert torch.equal(r.sigma_l, serial.sigma_l[..., l0:l0 + ls[ih], :, :]) and torch.equal(r.phi, serial.phi)
                    assert r.sigma_l.shape[-3] == ls[ih]
                r.set_tensor_state(s0[..., l0:l0 + ls[ih], m0:m0 + ms[iw], :])
                col.append(mn._NoiseSpectrum.apply(r.state, r.sigma_l if isotropic else None, False))
            cols.append(torch.cat(col, dim=-2))
    finally:
        mbd.finalize()
    coeffs = torch.cat(cols, dim=-1)
    grid = serial.isht.grid
    y = emulated_isht(coeffs, serial.nlat, serial.nlon, L, M, grid, "fp32", h, w).reshape(want.shape)
    _vs_single(y, want, "fp32", f"noise {case} {h}x{w} vs serial forward", h == 1)

"""The quadrature-weighted instance norm on the GPU (csrc/norm.cu, makani_b200.norm.GeometricInstanceNormS2, the distributed class's stages):

* the kernels through the C ABI against fp64 evaluations of their exact operands, per element: the partials (sum q, mean, M2) against fp64 sums of
  the float32 weights and the input; mu / r against fp64 of the kernel's partials; y against fp64 of the kernel's stats; S1 / S2 against fp64 of x,
  dy and the stats; dx against fp64 of the kernel's stats and sums.  fp32: |got - ref| <= 1e-5 max(1, |ref|); bf16 outputs within one bf16 ulp; the
  sums S1 / S2 (whose terms are fp32) within 1e-5 of the larger of max(1, |ref|) and the 2-norm of their terms.
  Shapes: 240 x 480 x 384 (the SFNO inner grid), 721 x 1440 x 8 (zero-weight pole rows of `naive`), 49 x 95 (the scalar path), a partial crop of a
  Legendre-Gauss grid and a full one; GELU on and off, affine off; one row offset by 1e4 (the pivot);
* the module against the fp64 oracle (output, dx, dgamma, dbeta at 1e-5 in fp32; bf16 inputs);
* the forward and backward launch only the new kernels (no aten reduction);
* h x w virtual ranks in one process: per-rank partials combined in rank order give bit-identical statistics on every rank, and each rank's dx
  matches its slice of the single-GPU distributed formula within the bound above;
* makani's own SFNO with instance_norm_s2 (tests/golden/sfno_s2norm_golden.npz) on the CUDA path, fp32 and TF32."""
import pytest
import torch

from makani_b200 import _lib
from makani_b200 import norm as N
from makani_b200.quadrature import crop_quadrature_np
from oracle import makani_norm_oracle as O
from test_gpu_engine import DEV, launched_kernels

pytestmark = pytest.mark.gpu

# id, dtype, B, C, img_shape, crop_shape, crop_offset, grid
SHAPES = [
    ("sfno-inner-240x480x384", torch.float32, 1, 384, (240, 480), (240, 480), (0, 0), "legendre-gauss"),
    ("bf16-240x480x384", torch.bfloat16, 1, 384, (240, 480), (240, 480), (0, 0), "legendre-gauss"),
    ("naive-721x1440x8", torch.float32, 1, 8, (721, 1440), (721, 1440), (0, 0), "equiangular"),
    ("bf16-naive-721x1440x8", torch.bfloat16, 1, 8, (721, 1440), (721, 1440), (0, 0), "equiangular"),
    ("scalar-49x95", torch.float32, 2, 3, (49, 95), (49, 95), (0, 0), "clenshaw-curtiss"),
    ("bf16-scalar-49x95", torch.bfloat16, 2, 3, (49, 95), (49, 95), (0, 0), "clenshaw-curtiss"),
    ("partial-crop-lg", torch.float32, 2, 4, (180, 360), (120, 200), (30, 100), "legendre-gauss"),
    ("lg-180x360", torch.float32, 2, 6, (180, 360), (180, 360), (0, 0), "legendre-gauss"),
]
TOL = 1e-5


def _bf16_ulp(ref):
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126)))
    return torch.pow(2.0, e - 7)


def _check(name, got, ref, dtype, scale=None):
    """per element |got - ref| <= 1e-5 max(1, |ref|) (fp32) or one bf16 ulp of ref; a sum of many terms also by 1e-5 of `scale`, the 2-norm of its
    terms: its terms are rounded to fp32 one by one, so on a row whose terms cancel the error is a random walk of that size, not of |sum|"""
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    if dtype == torch.bfloat16:
        bound = _bf16_ulp(ref) + 1e-6 * ref.abs().clamp_min(1.0)
    else:
        bound = TOL * ref.abs().clamp_min(1.0)
    if scale is not None:
        bound = torch.maximum(bound, TOL * scale.double())
    worst = (err / bound).max().item()
    print(f"{name}: worst err / bound {worst:.3f}")
    assert torch.isfinite(got).all() and worst <= 1.0, name


def _inputs(B, C, H, W, dtype, gen):
    x = 0.5 + torch.randn(B, C, H, W, dtype=torch.float64, device=DEV, generator=gen)
    x[0, min(1, C - 1)] += 1e4                        # the pivot: a row far from zero
    return x.to(dtype), torch.randn(B, C, H, W, device=DEV, generator=gen).to(dtype)


@pytest.mark.parametrize("case", SHAPES, ids=[s[0] for s in SHAPES])
@pytest.mark.parametrize("mode", ["gelu", "plain", "no-affine"])
def test_kernels_against_fp64_of_their_operands(case, mode):
    _, dtype, B, C, img, cs, co, grid = case
    H, W = cs
    gen = torch.Generator(device=DEV).manual_seed(7)
    x, dy = _inputs(B, C, H, W, dtype, gen)
    q = torch.from_numpy(crop_quadrature_np(grid, img, cs, co)).float().to(DEV)
    gelu = mode == "gelu"
    w32 = b32 = None
    if mode != "no-affine":
        w32 = (1.0 + 0.3 * torch.randn(C, device=DEV, generator=gen)).float()
        b32 = (0.2 * torch.randn(C, device=DEV, generator=gen)).float()
    st = N.CudaGeometricNormStages()
    rows = B * C
    x64, q64 = x.double().view(rows, H, W), q.double().view(1, H, 1)

    # partials: (sum q, mean, M2) against fp64 of the operands
    parts = st.partials(x, q)
    sq = (q64.sum() * W).expand(rows)
    mean = (q64 * x64).sum(dim=(1, 2)) / sq
    m2 = (q64 * (x64 - mean.view(-1, 1, 1)) ** 2).sum(dim=(1, 2))
    _check("sum q", parts[:, 0], sq, torch.float32)
    _check("mean", parts[:, 1], mean, torch.float32)
    assert ((parts[:, 2] - m2).abs() <= TOL * m2.abs().clamp_min(1e-3 * sq)).all(), "M2"

    # finalize (serial: R = 1, D = 1) against fp64 of the kernel's partials
    stats = st.finalize(parts.unsqueeze(0), 1.0, 1e-5)
    p = parts.double()
    mu = p[:, 0] * p[:, 1]
    var = p[:, 2] + p[:, 0] * (p[:, 1] - mu) ** 2
    r = 1.0 / torch.sqrt(var + 1e-5)
    _check("mu", stats[:, 0], mu, torch.float32)
    _check("r", stats[:, 1], r, torch.float32)
    _check("corr", stats[:, 2], r * mu * (1.0 - p[:, 0]), torch.float32)

    # apply against fp64 of the stats
    y = st.apply(x, w32, b32, stats, gelu)
    s = stats.double().view(B, C, 3, 1, 1)
    xh = (x.double() - s[:, :, 0]) * s[:, :, 1]
    gam = w32.double().view(1, C, 1, 1) if w32 is not None else 1.0
    z = xh * gam + (b32.double().view(1, C, 1, 1) if b32 is not None else 0.0)
    _check("y", y, torch.nn.functional.gelu(z) if gelu else z, dtype)

    # backward sums against fp64 of x, dy and the stats
    sums = st.backward_sums(x, dy, w32, b32, stats, gelu)
    g = dy.double()
    if gelu:
        g = g * (0.5 * (1.0 + torch.erf(z / 2 ** 0.5)) + z * torch.exp(-0.5 * z * z) / (2 * torch.pi) ** 0.5)
    norm1, norm2 = g.square().sum(dim=(2, 3)).sqrt().flatten(), (g * xh).square().sum(dim=(2, 3)).sqrt().flatten()
    _check("S1", sums[:, 0], g.sum(dim=(2, 3)).flatten(), torch.float32, norm1)
    _check("S2", sums[:, 1], (g * xh).sum(dim=(2, 3)).flatten(), torch.float32, norm2)

    # backward apply against fp64 of the stats and sums
    dx = st.backward_apply(x, dy, w32, b32, stats, sums.unsqueeze(0), q, 1.0, gelu)
    tot = sums.double().view(B, C, 2, 1, 1)
    ref = gam * s[:, :, 1] * (g - q.double().view(1, 1, H, 1) * (tot[:, :, 0] + xh * tot[:, :, 1] - s[:, :, 2] * tot[:, :, 1]))
    _check("dx", dx, ref, dtype)

    dg, db = st.param_grads(sums, B, C)
    _check("dgamma", dg, sums.double().view(B, C, 2)[:, :, 1].sum(0), torch.float32, sums.double().view(B, C, 2)[:, :, 1].abs().sum(0))
    _check("dbeta", db, sums.double().view(B, C, 2)[:, :, 0].sum(0), torch.float32, sums.double().view(B, C, 2)[:, :, 0].abs().sum(0))


def test_refusals():
    st = N.CudaGeometricNormStages()
    x = torch.randn(2, 40000, 2, 4, device=DEV)
    q = torch.ones(2, device=DEV)
    with pytest.raises(_lib.B200ShtError, match="65535"):
        st.partials(x, q)
    with pytest.raises(_lib.B200ShtError):
        st.finalize(torch.zeros(1, 4, 3, dtype=torch.float64, device=DEV), 0.0, 1e-5)


MODULE_CASES = [((240, 480), (240, 480), (0, 0), "legendre-gauss", 16), ((181, 360), (181, 360), (0, 0), "equiangular", 8),
                ((180, 360), (120, 200), (30, 100), "weatherbench2", 4), ((49, 95), (49, 95), (0, 0), "clenshaw-curtiss", 3)]


@pytest.mark.parametrize("case", MODULE_CASES, ids=lambda c: f"{c[3]}-{c[1][0]}x{c[1][1]}")
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_module_against_oracle(case, dtype):
    img, cs, co, grid, C = case
    m = N.GeometricInstanceNormS2(img, cs, co, grid, C, eps=1e-6, affine=True).to(DEV)
    gen = torch.Generator().manual_seed(3)
    with torch.no_grad():
        m.weight.copy_(1.0 + 0.3 * torch.randn(C, generator=gen))
        m.bias.copy_(0.2 * torch.randn(C, generator=gen))
    x = (1.0 + torch.randn(2, C, *cs, generator=gen)).to(dtype)
    dy = torch.randn(2, C, *cs, generator=gen).to(dtype)
    qg = O.grid_quadrature(grid, img, cs, co)
    rel = lambda a, b: ((a.double().cpu() - b).abs().max() / b.abs().max()).item()   # noqa: E731
    for gelu in (False, True):
        m.zero_grad()
        xd = x.to(DEV).requires_grad_(True)
        y = m(xd, gelu=gelu)
        y.backward(dy.to(DEV))
        xr = x.double().requires_grad_(True)
        pr = [p.detach().cpu().double().requires_grad_(True) for p in m.parameters()]
        yr = O.serial(xr, qg, 1e-6, *pr, gelu=gelu)
        yr.backward(dy.double())
        tol = 1e-5 if dtype == torch.float32 else 1e-2
        assert y.dtype == dtype
        assert rel(y.detach(), yr.detach()) < tol
        assert rel(xd.grad, xr.grad) < (tol if dtype == torch.float32 else 2e-2)
        for p, r in zip(m.parameters(), pr):
            assert rel(p.grad, r.grad) < tol


def test_launches_only_the_new_kernels():
    m = N.GeometricInstanceNormS2((240, 480), (240, 480), (0, 0), "legendre-gauss", 32, affine=True).to(DEV)
    x = torch.randn(1, 32, 240, 480, device=DEV, requires_grad=True)
    dy = torch.randn_like(x)
    m(x, gelu=True).backward(dy)     # warm the weight cache

    def run():
        x.grad = None
        m(x, gelu=True).backward(dy)

    want = ["geo_finalize_kernel", "geo_param_grad_kernel"] + [f"geo_norm_kernel<float, {m}, true" for m in range(4)]
    names = launched_kernels(run, done=lambda n: all(any(w in s for s in n) for w in want))
    assert all(any(w in s for s in names) for w in want), names
    assert all("geo_" in s for s in names), names
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    every = {e.name for e in prof.events()}
    assert not any("reduce_kernel" in s for s in every), every


@pytest.mark.parametrize("h,w", [(2, 1), (1, 2), (2, 2), (4, 2)])
@pytest.mark.parametrize("case", [((181, 360), (181, 360), (0, 0), "equiangular"), ((180, 360), (120, 200), (30, 100), "legendre-gauss")],
                         ids=["eq-181x360", "lg-crop"])
def test_virtual_ranks(h, w, case):
    img, cs, co, grid = case
    B, C = 2, 5
    gen = torch.Generator(device=DEV).manual_seed(21)
    x, dy = _inputs(B, C, *cs, torch.float32, gen)
    w32 = (1.0 + 0.3 * torch.randn(C, device=DEV, generator=gen)).float()
    b32 = (0.2 * torch.randn(C, device=DEV, generator=gen)).float()
    st = N.CudaGeometricNormStages()
    qfull = torch.from_numpy(crop_quadrature_np(grid, img, cs, co)).float().to(DEV)
    D = float(qfull.double().sum() * cs[1])
    hs, ws = O.split_shapes(cs[0], h), O.split_shapes(cs[1], w)
    shards, qs, parts = [], [], []
    for ih in range(h):
        for iw in range(w):
            xs = x[:, :, sum(hs[:ih]):sum(hs[:ih + 1]), sum(ws[:iw]):sum(ws[:iw + 1])].contiguous()
            dys = dy[:, :, sum(hs[:ih]):sum(hs[:ih + 1]), sum(ws[:iw]):sum(ws[:iw + 1])].contiguous()
            qk = qfull[sum(hs[:ih]):sum(hs[:ih + 1])].contiguous()
            shards.append((xs, dys))
            qs.append(qk)
            parts.append(st.partials(xs, qk))
    gathered = torch.stack(parts)
    stats = [st.finalize(gathered, D, 1e-5) for _ in shards]
    assert all(torch.equal(s, stats[0]) for s in stats)

    # the single-GPU distributed formula on the whole crop
    stats1 = st.finalize(st.partials(x, qfull).unsqueeze(0), D, 1e-5)
    y1 = st.apply(x, w32, b32, stats1, True)
    sums1 = st.backward_sums(x, dy, w32, b32, stats1, True)
    dx1 = st.backward_apply(x, dy, w32, b32, stats1, sums1.unsqueeze(0), qfull, D, True)
    _check("stats", stats[0][:, :2], stats1[:, :2].double(), torch.float32)

    sums = torch.stack([st.backward_sums(xs, dys, w32, b32, stats[k], True) for k, (xs, dys) in enumerate(shards)])
    for k, (xs, dys) in enumerate(shards):
        ih, iw = divmod(k, w)
        sl = (slice(None), slice(None), slice(sum(hs[:ih]), sum(hs[:ih + 1])), slice(sum(ws[:iw]), sum(ws[:iw + 1])))
        _check(f"y rank {k}", st.apply(xs, w32, b32, stats[k], True), y1[sl], torch.float32)
        _check(f"dx rank {k}", st.backward_apply(xs, dys, w32, b32, stats[k], sums, qs[k], D, True), dx1[sl], torch.float32)


@pytest.fixture
def torch_tf32():
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("name", ["s2norm_eq", "s2norm_lg"])
@pytest.mark.parametrize("precision,rtol,grtol", [("fp32", 2e-4, 5e-4), ("tf32", 4e-3, 1.5e-2)])
def test_sfno_instance_norm_s2_matches_reference_network(name, precision, rtol, grtol, torch_tf32):
    """makani's own SFNO with instance_norm_s2 (tests/golden/sfno_s2norm_golden.npz) on the CUDA path, at the tolerances of test_gpu_sfno.py"""
    import os
    import sys

    import numpy as np

    from makani_b200.sfno import SphericalFourierNeuralOperatorNet
    from test_gpu_parity import close
    from test_sfno_cpu import golden_state_dict

    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "golden"))
    from make_sfno_s2norm_golden import GRAD_KEYS, SFNO_S2NORM_GOLDEN_CASES

    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = (precision == "tf32")
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "sfno_s2norm_golden.npz"))
    net = SphericalFourierNeuralOperatorNet(**SFNO_S2NORM_GOLDEN_CASES[name], precision=precision)
    net.load_state_dict(golden_state_dict(g, name), strict=True)
    net = net.to(DEV)
    x = torch.from_numpy(g[f"{name}/x"]).to(DEV).requires_grad_(True)

    def run():
        return net(x)

    names = launched_kernels(lambda: run(), done=lambda n: any("geo_norm_kernel" in s for s in n))
    assert any("geo_norm_kernel" in s for s in names), names      # the norms run on the new kernels
    y = run()
    close(y, torch.from_numpy(g[f"{name}/y"]), rtol, f"SFNO-S2norm[{name},{precision}] y")
    (y * torch.from_numpy(g[f"{name}/g"]).to(DEV)).sum().backward()
    close(x.grad, torch.from_numpy(g[f"{name}/dx"]), grtol, f"SFNO-S2norm[{name},{precision}] dx")
    params = dict(net.named_parameters())
    for k in GRAD_KEYS:
        ref = torch.from_numpy(g[f"{name}/grad/{k}"])
        got = params[k].grad
        got = torch.view_as_real(got) if got.is_complex() else got
        close(got, ref, grtol, f"SFNO-S2norm[{name},{precision}] d{k}")

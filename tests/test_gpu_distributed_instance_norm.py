"""makani's DistributedInstanceNorm2d on the GPU (makani_b200.distributed.DistributedInstanceNorm2d): the quadrature-weighted norm stages of
csrc/norm.cu with every latitude weight 1 and the global point count as normaliser.

* h x w virtual ranks in one process: the CUDA partials of every shard, gathered in rank order, give statistics bit-identical on every rank and
  within 1e-5 max(1, |ref|) of fp64 of the whole field; every rank's partials, y, S1 / S2 and dx are held to the criteria of DESIGN.md section
  4.6b against fp64 evaluations of their exact operands (fp32 within 1e-5 max(1, |ref|), bf16 outputs within one bf16 ulp, the sums S1 / S2 also
  within 1e-5 of the 2-norm of their terms), and the gathered y and dx are compared with fp64 `F.instance_norm` of the whole field.
  Shapes: 384 x 240 x 480 at 2 x 2, 8 x 721 x 1440 at 4 x 2, 181 x 360 at 4 x 2 and at 2 x 4 (W_loc = 90: the scalar path); one plane offset by 1e4;
* the module at world size 1 against fp64 nn.InstanceNorm2d, fp32 and bf16, and replayed from a CUDA graph after its first call;
* the forward and backward launch only the geo_* kernels: no aten reduction, no Triton kernel."""
import pytest
import torch
import torch.nn.functional as F

import makani_b200.distributed as mbd
from makani_b200 import norm as N
from oracle import makani_norm_oracle as O
from test_gpu_engine import DEV, launched_kernels
from test_gpu_norm_s2 import _check

pytestmark = pytest.mark.gpu

EPS = 1e-5
# id, B, C, H, W, h, w
SHARDINGS = [("384x240x480-2x2", 1, 384, 240, 480, 2, 2), ("8x721x1440-4x2", 1, 8, 721, 1440, 4, 2), ("181x360-4x2", 2, 5, 181, 360, 4, 2),
             ("181x360-2x4-scalar", 2, 5, 181, 360, 2, 4)]


def _inputs(B, C, H, W, dtype, gen):
    x = 0.5 + torch.randn(B, C, H, W, dtype=torch.float64, device=DEV, generator=gen)
    x[0, min(1, C - 1)] += 1e4                        # one plane far from zero: the pivot carries it
    return x.to(dtype), torch.randn(B, C, H, W, device=DEV, generator=gen).to(dtype)


@pytest.mark.parametrize("affine", [True, False], ids=["affine", "plain"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("case", SHARDINGS, ids=[s[0] for s in SHARDINGS])
def test_virtual_ranks_against_fp64(case, dtype, affine):
    _, B, C, H, W, h, w = case
    gen = torch.Generator(device=DEV).manual_seed(11)
    x, dy = _inputs(B, C, H, W, dtype, gen)
    w32 = b32 = None
    if affine:
        w32 = (1.0 + 0.3 * torch.randn(C, device=DEV, generator=gen)).float()
        b32 = (0.2 * torch.randn(C, device=DEV, generator=gen)).float()
    st = N.CudaGeometricNormStages()
    D = float(H * W)
    hs, ws = O.split_shapes(H, h), O.split_shapes(W, w)
    if case[0].endswith("scalar"):
        assert all(wl % 4 for wl in ws)             # no 16-byte packet fits a row: the scalar path in both dtypes
    rows = B * C
    slices, parts = [], []
    for ih in range(h):
        for iw in range(w):
            sl = (slice(None), slice(None), slice(sum(hs[:ih]), sum(hs[:ih + 1])), slice(sum(ws[:iw]), sum(ws[:iw + 1])))
            xs = x[sl].contiguous()
            p = st.partials(xs, torch.ones(hs[ih], device=DEV))
            # partials against fp64 of the shard: the count exactly, the mean and M2 within 1e-5
            x64 = xs.double().view(rows, -1)
            mean = x64.mean(dim=1)
            m2 = ((x64 - mean[:, None]) ** 2).sum(dim=1)
            assert torch.equal(p[:, 0], torch.full_like(p[:, 0], float(hs[ih] * ws[iw]))), "count"
            _check(f"mean {ih},{iw}", p[:, 1], mean, torch.float32)
            assert ((p[:, 2] - m2).abs() <= 1e-5 * m2.abs().clamp_min(1e-3 * x64.shape[1])).all(), "M2"
            slices.append(sl)
            parts.append(p)
    gathered = torch.stack(parts)
    stats = [st.finalize(gathered, D, EPS) for _ in slices]
    assert all(torch.equal(s, stats[0]) for s in stats)

    # the statistics against fp64 of the whole field; the correction term vanishes (S = D exactly)
    x64 = x.double().view(rows, -1)
    mu64 = x64.mean(dim=1)
    r64 = 1.0 / torch.sqrt(((x64 - mu64[:, None]) ** 2).mean(dim=1) + EPS)
    _check("mu", stats[0][:, 0], mu64, torch.float32)
    _check("r", stats[0][:, 1], r64, torch.float32)
    assert torch.equal(stats[0][:, 2], torch.zeros_like(stats[0][:, 2]))

    s = stats[0].double().view(B, C, 3, 1, 1)
    gam = w32.double().view(1, C, 1, 1) if affine else 1.0
    bet = b32.double().view(1, C, 1, 1) if affine else 0.0
    y = torch.empty_like(x)
    sums = []
    for k, sl in enumerate(slices):
        xs, dys = x[sl].contiguous(), dy[sl].contiguous()
        xh = (xs.double() - s[:, :, 0]) * s[:, :, 1]
        y[sl] = ys = st.apply(xs, w32, b32, stats[k], False)
        _check(f"y rank {k}", ys, xh * gam + bet, dtype)
        sk = st.backward_sums(xs, dys, w32, b32, stats[k], False)
        g = dys.double()
        _check(f"S1 rank {k}", sk[:, 0], g.sum(dim=(2, 3)).flatten(), torch.float32, g.square().sum(dim=(2, 3)).sqrt().flatten())
        _check(f"S2 rank {k}", sk[:, 1], (g * xh).sum(dim=(2, 3)).flatten(), torch.float32, (g * xh).square().sum(dim=(2, 3)).sqrt().flatten())
        sums.append(sk)
    gsums = torch.stack(sums)
    tot = gsums.double().sum(dim=0).view(B, C, 2, 1, 1)
    dx = torch.empty_like(x)
    for k, sl in enumerate(slices):
        xs, dys = x[sl].contiguous(), dy[sl].contiguous()
        dx[sl] = dxs = st.backward_apply(xs, dys, w32, b32, stats[k], gsums, torch.ones(xs.shape[2], device=DEV), D, False)
        xh = (xs.double() - s[:, :, 0]) * s[:, :, 1]
        ref = gam * s[:, :, 1] * (dys.double() - (tot[:, :, 0] + xh * tot[:, :, 1] - s[:, :, 2] * tot[:, :, 1]) / D)
        _check(f"dx rank {k}", dxs, ref, dtype)

    # the gathered field against fp64 F.instance_norm of the whole (dtype-rounded) input; the fp32 rounding of mu on the offset plane
    # (half an ulp of 1e4, 5e-4) dominates the fp32 error
    xr = x.double().requires_grad_(True)
    yr = F.instance_norm(xr, weight=w32.double() if affine else None, bias=b32.double() if affine else None, eps=EPS)
    yr.backward(dy.double())
    rel = lambda a, b: ((a.double() - b).abs().max() / b.abs().max()).item()   # noqa: E731
    ey, edx = rel(y, yr.detach()), rel(dx, xr.grad)
    print(f"end to end: y {ey:.2e}, dx {edx:.2e}")
    tol = 3e-4 if dtype == torch.float32 else 1e-2
    assert ey < tol and edx < tol


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("shape", [(2, 16, 181, 360), (1, 384, 240, 480), (2, 3, 17, 33)], ids=lambda s: "x".join(map(str, s)))
def test_module_at_world_size_one_matches_instance_norm(shape, dtype):
    B, C, H, W = shape
    mbd.init(None, None)
    try:
        m = mbd.DistributedInstanceNorm2d(C, eps=EPS, affine=True).to(DEV)
        gen = torch.Generator().manual_seed(4)
        with torch.no_grad():
            m.weight.copy_(1.0 + 0.3 * torch.randn(C, generator=gen))
            m.bias.copy_(0.2 * torch.randn(C, generator=gen))
        x = (1.0 + torch.randn(B, C, H, W, generator=gen)).to(dtype)
        dy = torch.randn(B, C, H, W, generator=gen).to(dtype)
        xd = x.to(DEV).requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = m(xd)
        y.backward(dy.to(DEV))
        assert y.dtype == dtype
        ref = torch.nn.InstanceNorm2d(C, eps=EPS, affine=True).double()
        with torch.no_grad():
            ref.weight.copy_(m.weight.detach().cpu())
            ref.bias.copy_(m.bias.detach().cpu())
        xr = x.detach().double().requires_grad_(True)
        yr = ref(xr)
        yr.backward(dy.double())
        rel = lambda a, b: ((a.double().cpu() - b).abs().max() / b.abs().max()).item()   # noqa: E731
        tol = 1e-5 if dtype == torch.float32 else 1e-2
        assert rel(y.detach(), yr.detach()) < tol
        assert rel(xd.grad, xr.grad) < (tol if dtype == torch.float32 else 2e-2)
        assert rel(m.weight.grad, ref.weight.grad) < tol and rel(m.bias.grad, ref.bias.grad) < tol
        assert m._points == {(H, W): float(H * W)}
    finally:
        mbd.finalize()


def test_module_replays_from_a_cuda_graph():
    """after its first call the layer copies nothing to the host, so forward and backward capture in a CUDA graph; replays on new data equal
    eager calls bit for bit"""
    m = mbd.DistributedInstanceNorm2d(32, affine=True).to(DEV)
    with torch.no_grad():
        m.weight.add_(0.3 * torch.randn(32, device=DEV))
    x = torch.randn(1, 32, 120, 240, device=DEV, requires_grad=True)
    dy = torch.randn_like(x)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            x.grad = m.weight.grad = m.bias.grad = None
            m(x).backward(dy)
    torch.cuda.current_stream().wait_stream(side)
    x.grad = m.weight.grad = m.bias.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = m(x)
        y.backward(dy)
    with torch.no_grad():
        x.copy_(3.0 + 2.0 * torch.randn_like(x))
        dy.copy_(torch.randn_like(dy))
    graph.replay()
    torch.cuda.synchronize()
    got = [t.clone() for t in (y, x.grad, m.weight.grad, m.bias.grad)]
    xe = x.detach().clone().requires_grad_(True)
    m.weight.grad = m.bias.grad = None
    ye = m(xe)
    ye.backward(dy)
    for a, b in zip(got, (ye, xe.grad, m.weight.grad, m.bias.grad)):
        assert torch.equal(a, b.detach())


def test_launches_only_the_geo_kernels():
    m = mbd.DistributedInstanceNorm2d(32, affine=True).to(DEV)
    x = torch.randn(1, 32, 240, 480, device=DEV, requires_grad=True)
    dy = torch.randn_like(x)
    m(x).backward(dy)     # the first call exchanges the point count and makes the weights

    def run():
        x.grad = m.weight.grad = m.bias.grad = None
        m(x).backward(dy)

    want = ["geo_finalize_kernel", "geo_param_grad_kernel"] + [f"geo_norm_kernel<float, {mode}, true" for mode in range(4)]
    names = launched_kernels(run, done=lambda n: all(any(w in s for s in n) for w in want))
    assert all(any(w in s for s in names) for w in want), names
    assert all("geo_" in s for s in names), names
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    every = {e.name for e in prof.events()}
    assert not any("reduce_kernel" in s or "triton" in s.lower() for s in every), every

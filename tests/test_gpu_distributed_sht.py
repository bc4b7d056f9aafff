"""The CUDA local stages of DistributedRealSHT / DistributedInverseRealSHT on one GPU, at the shard geometries of h x w model parallelism:

A. a scalar plan with an order offset holds exactly (bit for bit) the order slice of the table of the plan of all orders;
B. the Legendre stages of CudaLocalOps on an order shard (latspec_pack -> analysis -> spec_unpack_ex, spec_pack_ex -> synthesis ->
   latspec_unpack) give bit for bit the order slice of the same stages on the plan of all orders, at FP32, TF32 and 3 x TF32: the tiles
   of order m start at lstart(m_offset + m) in the engine and in the CUDA-core kernels, so every per-order sum runs over the same rows;
C. the longitude stages of CudaLocalOps on every latitude slice (an FFT-only plan of nlat_local rows) give bit for bit the rows of the same
   call on the plan of all rows: the row scale is the same float, computed from the same quad_w[k], and every kernel that serves these
   plans (the tensor-core DFT, the compile-time CUDA-core FFT) transforms each row on its own;
D. h x w virtual ranks emulated in one process (each rank's CudaLocalOps on its shard geometry, the transposes as split / cat): values and
   both gradients against the single-GPU RealSHT / InverseRealSHT, equal wherever both run the same kernels on the same rows, and against
   the fp64 oracle;
E. the distributed spectral filter (dense packed spectra of each (l, m) shard, the dense channel mix on the rank's weight slice) against the
   single-GPU SpectralConv and the oracle.

Every buffer a stage must not read holds NaN and every output of a direct C-ABI call starts as a sentinel.  Run with -s to see the kernel
that served each longitude analysis and the worst ratio of every bounded comparison.
"""
import functools

import pytest
import torch

import makani_b200 as mb
import makani_b200.distributed as mbd
from makani_b200 import _lib
from makani_b200.quadrature import _grid_np
from makani_b200.sht import Plan, _SpecPackEx, _SpecUnpackEx, _ptr, _stream
from makani_b200.spectral_convolution import _op_code, mix_packed
from oracle import makani_oracle as O
from test_gpu_distributed_vector import ORACLE, SINGLE_GPU, _bits_equal, _split, close, rel_l2
from test_gpu_engine import SENTINEL, launched_kernels, sentinel, untouched

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
NAN = float("nan")
PRECS = {"fp32": _lib.PREC_FP32, "tf32": _lib.PREC_TF32, "fp32x3": _lib.PREC_FP32X3}


def _no_sentinel(t):
    t = torch.view_as_real(t) if t.is_complex() else t
    return not bool((t.contiguous().view(torch.int32) == SENTINEL).any())


def splits(n, parts):
    """(offset, size) of every shard of compute_split_shapes(n, parts)"""
    s = mbd.compute_split_shapes(n, parts)
    return [(sum(s[:i]), s[i]) for i in range(parts)]


def local_ops(cls, nlat, nlon, L, M, grid, precision, lat=(0, None), orders=(0, None), csphase=True):
    """CudaLocalOps of the module of world size 1 given the shard geometry: latitude rows [lat[0], lat[0] + lat[1]) and orders
    [orders[0], orders[0] + orders[1]) (None: all)"""
    t = cls(nlat, nlon, L, M, grid, csphase=csphase, precision=precision)
    t.lat_offset, t.nlat_local = lat[0], lat[1] or t.nlat
    t.m_offset, t.mmax_local = orders[0], orders[1] or t.mmax
    return t, mbd.CudaLocalOps(t)


# ------------------------------------------------------------------------------------------------------------- A. tables
def splan(nlat, nlon, L, M, m_offset, grid="equiangular", csphase=True):
    cost, w = _grid_np(nlat, grid)
    return Plan.create_ex(nlat, nlon, L, M, m_offset, 0, cost, w, csphase, DEV)


@pytest.mark.parametrize("csphase", [True, False])
def test_offset_scalar_plan_tables_are_the_order_slice(csphase):
    # on and off the 32-order tiles, a shard of one order, shards ending at mmax
    nlat, nlon, L, M = 91, 192, 91, 97
    tfull = splan(nlat, nlon, L, M, 0, csphase=csphase).table()
    for off, mloc in ((0, 40), (13, 20), (32, 32), (33, 31), (64, 33), (90, 1), (96, 1), (40, 57)):
        p = splan(nlat, nlon, L, mloc, off, csphase=csphase)
        assert not p.vector and p.query(7) == off and p.query(3) == mloc and p.query(2) == L
        assert _bits_equal(p.table(), tfull[off:off + mloc]), (off, mloc, csphase)
    # the order shards of the 721 x 1440, L = 240 grid
    nlat, nlon, L, M = 721, 1440, 240, 241
    tfull = splan(nlat, nlon, L, M, 0, csphase=csphase).table()
    for w in (2, 3, 4, 8):
        for off, mloc in splits(M, w):
            assert _bits_equal(splan(nlat, nlon, L, mloc, off, csphase=csphase).table(), tfull[off:off + mloc]), (w, off, mloc, csphase)
    del tfull
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------- B. Legendre stages on order shards
def _legendre_direct(plan, prec, xc, direction):
    """the chain of makani_b200.distributed._legendre_call with sentinel intermediate and output buffers: every output entry written,
    every intermediate entry a later stage reads written (a sentinel read shows as a NaN)"""
    B, C = xc.shape[:2]
    st = _stream(DEV)
    lat, spec = sentinel(plan.latspec_elems(B, C)), sentinel(plan.spec_elems(B, C))
    if direction == 0:
        out = sentinel(B * C * plan.lmax * plan.mmax * 2).view(torch.complex64).view(B, C, plan.lmax, plan.mmax)
        _lib.call("b200sht_latspec_pack", plan.handle, _ptr(xc), _ptr(lat), B, C, st)
        _lib.call("b200sht_legendre_analysis", plan.handle, _ptr(lat), _ptr(spec), B, C, prec, st)
        _lib.call("b200sht_spec_unpack_ex", plan.lmax, plan.mmax, plan.m_offset, 0, _ptr(spec), _ptr(out), B, C, st)
        # the analysis writes the stored entries l >= lstart(m_offset + m) of the packed spec, and only those
        sv = spec.view(plan.lmax, plan.mmax, -1)
        stored = torch.arange(plan.lmax, device=DEV)[:, None] >= _lstart(plan.m_offset + torch.arange(plan.mmax, device=DEV))[None, :]
        assert untouched(sv[~stored]) and _no_sentinel(sv[stored]), "the analysis must write exactly the stored spec entries"
    else:
        out = sentinel(B * C * plan.nlat * plan.mmax * 2).view(torch.complex64).view(B, C, plan.nlat, plan.mmax)
        _lib.call("b200sht_spec_pack_ex", plan.lmax, plan.mmax, plan.m_offset, 0, _ptr(xc), _ptr(spec), B, C, st)
        _lib.call("b200sht_legendre_synthesis", plan.handle, _ptr(spec), _ptr(lat), B, C, prec, st)
        _lib.call("b200sht_latspec_unpack", plan.handle, _ptr(lat), _ptr(out), B, C, st)
    assert _no_sentinel(out), "an output entry was not written"
    return out


def _lstart(m):
    return (m // 32) * 32


def _synthesis_input(B, C, L, M, gen):
    """complex (B, C, L, M) twice: NaN for l < lstart(m) (spec_pack_ex drops these, nothing may read them), random values for l >= m, and
    for lstart(m) <= l < m finite junk in the first tensor, zeros in the second"""
    c = torch.randn(B, C, L, M, dtype=torch.complex64, device=DEV, generator=gen)
    l, m = torch.arange(L, device=DEV)[:, None], torch.arange(M, device=DEV)[None, :]
    band, nan = (l >= _lstart(m)) & (l < m), torch.full_like(c, complex(NAN, NAN))
    return (torch.where(l < _lstart(m), nan, torch.where(band, 7.0 * c, c)),
            torch.where(l < _lstart(m), nan, torch.where(band, torch.zeros_like(c), c)))


LEG_GRIDS = [("equiangular", 91, 180, 91, 91, 2, 3), ("legendre-gauss", 721, 1440, 240, 241, 1, 2)]


@pytest.mark.parametrize("precision", ["fp32", "tf32", "fp32x3"])
@pytest.mark.parametrize("grid,nlat,nlon,L,M,B,C", LEG_GRIDS, ids=["91x180", "721x1440"])
def test_order_shard_legendre_stages_are_the_order_slice(precision, grid, nlat, nlon, L, M, B, C):
    """analysis, synthesis and both backward passes of CudaLocalOps on every shard of compute_split_shapes(M, w), w = 2, 3, 4 (8 on the
    large grid), plus shards on a tile boundary and of one order: bit for bit the order slice of the plan of all orders.

    Synthesis input contract (the same as the single-GPU InverseRealSHT, whose spec_pack keeps l >= lstart(m)): entries l < lstart(m_offset
    + m) are dropped by spec_pack_ex and never read (NaN here); entries lstart(m_offset + m) <= l < m_offset + m are read but meet exact
    zeros of the table, so finite values there change nothing (junk here gives the output of zeros, bit for bit)."""
    gen = torch.Generator(device=DEV).manual_seed(333 + nlat)
    prec = PRECS[precision]
    _, full = local_ops(mbd.DistributedRealSHT, nlat, nlon, L, M, grid, precision)
    xc = torch.randn(B, C, nlat, M, dtype=torch.complex64, device=DEV, generator=gen)
    c, c0 = _synthesis_input(B, C, L, M, gen)
    pf = full._leg_plan(DEV)
    ya, ys = _legendre_direct(pf, prec, xc, 0), _legendre_direct(pf, prec, c, 1)
    assert torch.isfinite(torch.view_as_real(ya)).all() and torch.isfinite(torch.view_as_real(ys)).all()
    assert _bits_equal(ys, _legendre_direct(pf, prec, c0, 1)), "finite entries lstart(m) <= l < m must not change the synthesis"
    # the single-GPU inverse transform has the same contract
    isht = mb.InverseRealSHT(nlat, nlon, L, M, grid, precision=precision)
    assert _bits_equal(isht(c), isht(c0)), "InverseRealSHT: finite entries lstart(m) <= l < m must not change the output"

    shards = sorted({s for w in ((2, 3, 4, 8) if M > 200 else (2, 3, 4)) for s in splits(M, w)} | {(32, 32), (M - 1, 1)})
    lo = torch.arange(L, device=DEV)[:, None]
    for off, mloc in shards:
        _, ops = local_ops(mbd.DistributedRealSHT, nlat, nlon, L, M, grid, precision, orders=(off, mloc))
        sl = slice(off, off + mloc)
        tag = f"{grid} {nlat}x{nlon} {precision} orders {off}..{off + mloc - 1}"
        p = ops._leg_plan(DEV)
        assert p.m_offset == off and p.mmax == mloc
        # direct chain on sentinels
        a = _legendre_direct(p, prec, xc[..., sl].contiguous(), 0)
        assert _bits_equal(a, ya[..., sl]), f"{tag}: analysis"
        below = lo < (off + torch.arange(mloc, device=DEV))[None, :]
        assert (a[..., below] == 0).all(), f"{tag}: analysis l < m_offset + m must be exact zeros"
        s = _legendre_direct(p, prec, c[..., sl].contiguous(), 1)
        assert _bits_equal(s, ys[..., sl]), f"{tag}: synthesis"
        # the autograd stages of CudaLocalOps: forward and backward of legendre / ilegendre
        xs = xc[..., sl].clone().requires_grad_(True)
        y = ops.legendre(xs)
        assert _bits_equal(y, a), f"{tag}: CudaLocalOps.legendre"
        y.backward(c[..., sl])
        assert _bits_equal(xs.grad, s), f"{tag}: legendre backward"
        cs = c[..., sl].clone().requires_grad_(True)
        z = ops.ilegendre(cs)
        assert _bits_equal(z, ys[..., sl]), f"{tag}: CudaLocalOps.ilegendre"
        z.backward(xc[..., sl])
        assert _bits_equal(cs.grad, a), f"{tag}: ilegendre backward"
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ C. longitude stages on latitude slices
def _want_analysis_kernel(nlon, dtype, precision):
    """the kernel b200sht_fft_analysis runs for an FFT-only plan (csrc/fft.cu fft_analysis): the tensor-core DFT at TF32 for bf16 rows
    or nlon % 32 == 0, else the compile-time CUDA-core FFT"""
    N2 = nlon // 8
    if precision == "tf32" and (dtype == torch.bfloat16 or nlon % 32 == 0):
        return f"dft_analysis_kernel<{'float' if dtype == torch.float32 else '__nv_bfloat16'}, {N2 if N2 in (180, 90, 60) else 0}>"
    return "fft_analysis_ct_kernel<"


FFT_GRIDS = [(721, 1440, 241), (11, 1440, 241), (45, 360, 181), (13, 72, 37)]


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("nlat,nlon,M", FFT_GRIDS, ids=[f"{g[0]}x{g[1]}" for g in FFT_GRIDS])
def test_latitude_slice_longitude_stages_are_the_row_slice(nlat, nlon, M, dtype, precision):
    """fft, ifft and their backward passes on every slice of compute_split_shapes(nlat, h), h = 2, 3, 4, 8 (slices of 1 .. 7 rows on the
    small grids): bit for bit rows [lat_offset, lat_offset + nlat_local) of the same stage on the FFT-only plan of all rows.  Every
    analysis asserts its kernel; the direct call into a sentinel latspec also checks that the latitude padding of a slice holds zeros."""
    gen = torch.Generator(device=DEV).manual_seed(nlat + nlon)
    B, C = 1, 3
    x = torch.randn(B, C, nlat, nlon, device=DEV, generator=gen).to(dtype)
    z = torch.randn(B, C, nlat, M, dtype=torch.complex64, device=DEV, generator=gen)
    gy = torch.randn(B, C, nlat, nlon, device=DEV, generator=gen).to(dtype)
    want = _want_analysis_kernel(nlon, dtype, precision)

    def stages(ops, rows):
        xs = x[..., rows, :].clone().requires_grad_(True)
        X = ops.fft(xs)
        X.backward(z[..., rows, :])
        zs = z[..., rows, :].clone().requires_grad_(True)
        y = ops.ifft(zs, dtype)
        y.backward(gy[..., rows, :])
        return X, xs.grad, y, zs.grad

    _, fops = local_ops(mbd.DistributedRealSHT, nlat, nlon, None, M, "equiangular", precision)
    ref = stages(fops, slice(0, nlat))
    for t in ref:
        assert torch.isfinite(torch.view_as_real(t) if t.is_complex() else t.float()).all()
    seen = set()
    for h in (2, 3, 4, 8):
        for off, n in splits(nlat, h):
            rows = slice(off, off + n)
            _, ops = local_ops(mbd.DistributedRealSHT, nlat, nlon, None, M, "equiangular", precision, lat=(off, n))
            tag = f"{nlat}x{nlon} {dtype} {precision} h={h} rows {off}..{off + n - 1}"
            for name, a, b in zip(("fft", "fft backward", "ifft", "ifft backward"), stages(ops, rows), ref):
                assert _bits_equal(a, b[..., rows, :]), f"{tag}: {name}"
            xs = x[..., rows, :].contiguous()
            names = launched_kernels(lambda: ops.fft(xs), lambda nm: any(want in s for s in nm))
            assert any(want in s for s in names), f"{tag}: expected {want}, ran {names}"
            names_b = launched_kernels(lambda: mbd._LocalIFFT.backward(_Ctx(ops, precision), xs), lambda nm: any(want in s for s in nm))
            assert any(want in s for s in names_b), f"{tag}: ifft backward expected {want}, ran {names_b}"
            seen.update(s for s in names if "analysis" in s)
            # the slice plan's latspec: rows [n, kp) exact zeros
            p = ops._fft_plan(DEV)
            lat = sentinel(p.latspec_elems(B, C))
            mode = 2 if precision == "tf32" else 0
            _lib.call("b200sht_fft_analysis", p.handle, _ptr(xs), mb.sht._dtype_code(dtype), B, C, _ptr(lat), mode, _stream(DEV))
            X = lat[: M * 2 * B * C * p.kp].view(M, 2, B * C, p.kp)
            assert (X[..., n:] == 0).all() and torch.isfinite(X).all(), f"{tag}: latitude padding of the slice"
            if "dft" in want:
                assert untouched(lat[M * 2 * B * C * p.kp:]), f"{tag}: the DFT wrote a padding order [mmax, mmax8)"
    print(f"[dist-sht] {nlat}x{nlon} {dtype} {precision}: analysis served by {sorted(seen)}")


class _Ctx:
    """stand-in for the autograd context of _LocalIFFT: runs its backward (the adjoint longitude analysis) on its own"""

    def __init__(self, ops, precision):
        self.plan, self.prec = ops._fft_plan(DEV), PRECS[precision]


# ------------------------------------------------------------------------------------------------------ D. virtual h x w ranks
def _rank(cls, nlat, nlon, L, M, grid, precision, h, w, ih, iw):
    lat, ms = splits(nlat, h)[ih], splits(M, w)[iw]
    return local_ops(cls, nlat, nlon, L, M, grid, precision, lat=lat, orders=ms)


def emulated_sht(x, nlat, nlon, L, M, grid, precision, h, w):
    """x (B, C, nlat, nlon) -> (B, C, L, M): the stages of every virtual rank, the transposes as split / cat"""
    X = []
    for ih, xh in enumerate(_split(x, -2, h)):                  # polar shard of the input
        row = []
        for iw, xw in enumerate(_split(xh, 1, w)):               # azimuth transpose: channels split, all longitudes
            _, ops = _rank(mbd.DistributedRealSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            row.append(ops.fft(xw))
        X.append(torch.cat(row, dim=1))
    X = torch.cat(X, dim=-2)
    out = []
    for iw, Xw in enumerate(_split(X, -1, w)):                   # order shards
        col = []
        for ih, Xh in enumerate(_split(Xw, 1, h)):               # polar transpose: channels split, all latitudes
            _, ops = _rank(mbd.DistributedRealSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            col.append(ops.legendre(Xh))
        out.append(torch.cat(col, dim=1))
    return torch.cat(out, dim=-1)


def emulated_isht(c, nlat, nlon, L, M, grid, precision, h, w, dtype=torch.float32):
    Z = []
    for iw, cw in enumerate(_split(c, -1, w)):
        col = []
        for ih, ch in enumerate(_split(cw, 1, h)):
            _, ops = _rank(mbd.DistributedInverseRealSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            col.append(ops.ilegendre(ch))
        Z.append(torch.cat(col, dim=1))
    Z = torch.cat(Z, dim=-1)
    y = []
    for ih, Zh in enumerate(_split(Z, -2, h)):
        row = []
        for iw, Zw in enumerate(_split(Zh, 1, w)):
            _, ops = _rank(mbd.DistributedInverseRealSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            row.append(ops.ifft(Zw, dtype))
        y.append(torch.cat(row, dim=1))
    return torch.cat(y, dim=-2)


def _cmp(a, b, precision, name, bounds):
    """fp32 / 3 x TF32: the element bound close(rtol = bounds[0]); TF32: relative L2 below bounds[1].  Prints the worst ratio."""
    if precision in ("fp32", "fp32x3"):
        close(a, b, bounds[0], name)
    else:
        r = rel_l2(a, b)
        print(f"[dist-sht] TF32 rel-L2 {name}: {r:.3e} (ratio {r / bounds[1]:.3f})")
        assert r < bounds[1], (name, r)


def _equal(a, b, name):
    a, b = a.detach(), b.detach()
    same = torch.equal(a.view(torch.int16), b.view(torch.int16)) if a.dtype == torch.bfloat16 else _bits_equal(a, b)
    assert a.dtype == b.dtype and same, f"{name}: not bit-identical to the single-GPU transform"


def _vs_single(a, b, precision, name, same):
    """`same`: both run the same kernels on the same rows, so bit for bit; else the SINGLE_GPU bound"""
    if same:
        _equal(a, b, name)
    else:
        _cmp(a, b, precision, name, SINGLE_GPU)


@functools.lru_cache(maxsize=None)
def _oracle(grid, nlat, nlon, L, M, B, C, dtype):
    """inputs and fp64 oracle results (forward values and dx, inverse values and dcoeffs) of one grid, shared by every (h, w, precision)"""
    gen = torch.Generator().manual_seed(nlat * 7 + nlon)
    x = torch.randn(B, C, nlat, nlon, generator=gen).to(dtype)
    g = torch.randn(B, C, L, M, dtype=torch.complex64, generator=gen) * torch.tril(torch.ones(L, M))
    c = torch.randn(B, C, L, M, dtype=torch.complex64, generator=gen) * torch.tril(torch.ones(L, M))
    gy = torch.randn(B, C, nlat, nlon, generator=gen)
    of = O.RealSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    oi = O.InverseRealSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    xr = x.double().requires_grad_(True)
    cr = of(xr)
    cr.backward(g.to(torch.complex128))
    cc = c.to(torch.complex128).requires_grad_(True)
    yr = oi(cc)
    yr.backward(gy.double())
    return x, g, c, gy, (cr.detach(), xr.grad, yr.detach(), cc.grad)


# channels >= h and >= w: the transposes split them
VR_GRIDS = [("equiangular", 91, 180, 91, 91, 2, 8), ("legendre-gauss", 90, 180, 70, 20, 2, 4), ("equiangular", 721, 1440, 240, 241, 1, 4)]
VR_PARAMS = [pytest.param(*g, hw, id=f"{g[1]}x{g[2]}-{hw[0]}x{hw[1]}") for g in VR_GRIDS for hw in ((2, 1), (1, 2), (2, 2), (4, 2))]
VR_PARAMS.append(pytest.param(*VR_GRIDS[0], (8, 4), id="91x180-8x4"))


@pytest.mark.parametrize("precision", ["fp32", "tf32", "fp32x3"])
@pytest.mark.parametrize("grid,nlat,nlon,L,M,B,C,hw", VR_PARAMS)
def test_virtual_ranks_match_single_gpu_and_oracle(precision, grid, nlat, nlon, L, M, B, C, hw):
    """Same kernels on the same rows as the single-GPU transforms (makani_b200/sht.py), so torch.equal: the forward transform and the
    inverse's dcoeffs (longitude analysis, DFT or FFT by the same rule, then Legendre analysis) at every precision, everything at FP32 and
    3 x TF32, and at TF32 too where the grid has no tensor-core DFT (nlon 180).  At TF32 on a DFT grid (nlon 1440) the single-GPU synthesis
    runs the tiled layout and the tensor-core DFT, the distributed one the standard layout and the CUDA-core FFT: the forward's dx and the
    inverse's values are held to SINGLE_GPU there."""
    h, w = hw
    x, g, c, gy, (cr, dxr, yr, dcr) = _oracle(grid, nlat, nlon, L, M, B, C, torch.float32)
    sht = mb.RealSHT(nlat, nlon, L, M, grid, precision=precision)
    isht = mb.InverseRealSHT(nlat, nlon, L, M, grid, precision=precision)
    tag = f"{h}x{w} {grid} {nlat}x{nlon} L={L} M={M} {precision}"
    # the single-GPU synthesis leaves the standard chain only at TF32 on a grid the tensor-core DFT covers (sht._synthesis_pair)
    same_syn = not (precision == "tf32" and sht.plan(DEV).dft_ok)

    xd, xs = x.to(DEV).requires_grad_(True), x.to(DEV).requires_grad_(True)
    cd, cs = emulated_sht(xd, nlat, nlon, L, M, grid, precision, h, w), sht(xs)
    for a in (cd, cs):
        a.backward(g.to(DEV))
    _equal(cd, cs, f"sht {tag}")
    _vs_single(xd.grad, xs.grad, precision, f"sht dx vs single GPU {tag}", same_syn)
    _cmp(cd, cr, precision, f"sht vs oracle {tag}", ORACLE)
    _cmp(xd.grad, dxr, precision, f"sht dx vs oracle {tag}", ORACLE)

    cd, cs = c.to(DEV).requires_grad_(True), c.to(DEV).requires_grad_(True)
    yd, ys = emulated_isht(cd, nlat, nlon, L, M, grid, precision, h, w), isht(cs)
    assert yd.dtype == torch.float32
    for a in (yd, ys):
        a.backward(gy.to(DEV))
    _vs_single(yd, ys, precision, f"isht vs single GPU {tag}", same_syn)
    _equal(cd.grad, cs.grad, f"isht dcoeffs {tag}")
    _cmp(yd, yr, precision, f"isht vs oracle {tag}", ORACLE)
    _cmp(cd.grad, dcr, precision, f"isht dcoeffs vs oracle {tag}", ORACLE)


def test_virtual_ranks_bf16_input():
    """bf16 rows on 2 x 2 ranks at FP32 and TF32: values and the bf16 dx bit for bit the single-GPU transform's (nlon 180 has no
    tensor-core DFT, so both run the same kernels at TF32 too), and the fp64 oracle of the bf16 values bounds both"""
    grid, nlat, nlon, L, M, B, C = "equiangular", 91, 180, 91, 91, 2, 8
    x, g, _, _, (cr, dxr, _, _) = _oracle(grid, nlat, nlon, L, M, B, C, torch.bfloat16)
    for precision in ("fp32", "tf32"):
        sht = mb.RealSHT(nlat, nlon, L, M, grid, precision=precision)
        xd, xs = x.to(DEV).requires_grad_(True), x.to(DEV).requires_grad_(True)
        cd, cs = emulated_sht(xd, nlat, nlon, L, M, grid, precision, 2, 2), sht(xs)
        for a in (cd, cs):
            a.backward(g.to(DEV))
        assert xd.grad.dtype == torch.bfloat16
        _equal(cd, cs, f"bf16 sht {precision}")
        _vs_single(xd.grad, xs.grad, precision, f"bf16 sht dx {precision}", not (precision == "tf32" and sht.plan(DEV).dft_ok))
        _cmp(cd, cr, precision, f"bf16 sht vs oracle {precision}", ORACLE)
        close(xd.grad.float(), dxr, 1e-2, f"bf16 sht dx vs oracle {precision} (bf16 output)")


# -------------------------------------------------------------------------------------------- E. the distributed spectral filter
def emulated_spectral_conv(x, weight, bias, op, nlat, nlon, L, M, grid, precision, h, w):
    """SHT on the virtual ranks; each rank (ih, iw) packs its (l, m) shard densely (_SpecPackEx(., 0, 1)), mixes it with its weight
    slice (dhconv: the l slice; diagonal: the l x m slice) and unpacks it; the inverse on the virtual ranks, plus the bias"""
    B, Ci = x.shape[:2]
    Co = bias.shape[1]
    X = emulated_sht(x, nlat, nlon, L, M, grid, precision, h, w)
    code = _op_code(op, False) | _lib.DENSE_FLAG
    Y = []
    for (lo, nl), Xl in zip(splits(L, h), _split(X, -2, h)):
        row = []
        for (mo, nm), Xlm in zip(splits(M, w), _split(Xl, -1, w)):
            wr = weight[..., lo:lo + nl] if op == "dhconv" else weight[..., lo:lo + nl, mo:mo + nm]
            spec = _SpecPackEx.apply(Xlm.contiguous(), 0, 1)
            ys = mix_packed(spec, wr, code, nl, nm, B, 1, Ci, Co, precision)
            row.append(_SpecUnpackEx.apply(ys, nl, nm, B, Co, 0, 1))
        Y.append(torch.cat(row, dim=-1))
    Y = torch.cat(Y, dim=-2)
    return emulated_isht(Y, nlat, nlon, L, M, grid, precision, h, w) + bias


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("op", ["dhconv", "diagonal"])
@pytest.mark.parametrize("h,w", [(2, 2), (4, 2)])
def test_distributed_spectral_filter(h, w, op, precision):
    grid, nlat, nlon, L, M, B, C = "equiangular", 91, 180, 91, 91, 2, 8
    torch.manual_seed(333)
    sht = mb.RealSHT(nlat, nlon, L, M, grid, precision=precision)
    isht = mb.InverseRealSHT(nlat, nlon, L, M, grid, precision=precision)
    conv = mb.SpectralConv(sht, isht, C, C, operator_type=op, bias=True, precision=precision).to(DEV)
    with torch.no_grad():
        conv.bias.copy_(torch.randn(1, C, 1, 1))
    x, gy = torch.randn(B, C, nlat, nlon), torch.randn(B, C, nlat, nlon)
    tag = f"{h}x{w} {op} {precision}"

    xd, xs = x.to(DEV).requires_grad_(True), x.to(DEV).requires_grad_(True)
    wd = conv.weight.detach().clone().requires_grad_(True)
    bd = conv.bias.detach().clone().requires_grad_(True)
    yd = emulated_spectral_conv(xd, wd, bd, op, nlat, nlon, L, M, grid, precision, h, w)
    ys, _ = conv(xs)
    yd.backward(gy.to(DEV))
    ys.backward(gy.to(DEV))

    of, oi = O.RealSHT(nlat, nlon, L, M, grid, dtype=torch.float64), O.InverseRealSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    xr = x.double().requires_grad_(True)
    wr = conv.weight.detach().cpu().to(torch.complex128).requires_grad_(True)
    br = conv.bias.detach().cpu().double().requires_grad_(True)
    yr, _ = O.spectral_conv_forward(xr, wr, of, oi, operator_type=op, bias=br)
    yr.backward(gy.double())
    for name, a, b, r in (("y", yd, ys, yr), ("dx", xd.grad, xs.grad, xr.grad), ("dweight", wd.grad, conv.weight.grad, wr.grad),
                          ("dbias", bd.grad, conv.bias.grad, br.grad)):
        _cmp(a, b, precision, f"filter {name} vs single GPU {tag}", SINGLE_GPU)
        _cmp(a, r, precision, f"filter {name} vs oracle {tag}", ORACLE)

"""The CUDA local stages of DistributedRealVectorSHT / DistributedInverseRealVectorSHT on one GPU:

* a vector plan with an order offset holds exactly (bit for bit) the order slice of the tables of the plan of all orders;
* its Legendre stages and converters, run through ctypes with NaN sentinels in everything they must not read, give bit for bit the order slice
  of the full plan's outputs, at FP32 and TF32: every per-order sum runs over the same latitude rows and degree tiles (the tiles of order m
  start at lstart(m_offset + m) on both plans), so only the order index of the launch differs;
* h x w virtual ranks emulated in one process: each rank's CudaLocalOps stages on its shard geometry, the transposes done with split and cat,
  against the single-GPU RealVectorSHT / InverseRealVectorSHT and the fp64 oracle, values and both gradients;
* the refusals: the one-call b200sht_vsht_* entries and the tiled synthesis on an order shard, VECTOR | FFT_ONLY plans, and 3 x TF32.
"""
import ctypes

import pytest
import torch

import makani_b200 as mb
import makani_b200.distributed as mbd
from makani_b200 import _lib
from makani_b200.quadrature import _grid_np
from makani_b200.sht import Plan
from oracle import makani_vector_oracle as V
from test_gpu_parity import close
from test_gpu_vector_sht import TF32_REL_L2, rel_l2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
VP = ctypes.c_void_p
NAN = float("nan")


def _p(t):
    return VP(t.data_ptr())


def _stream():
    return VP(torch.cuda.current_stream(DEV).cuda_stream)


def vplan(nlat, nlon, L, M, m_offset, grid="equiangular", csphase=True):
    cost, w = _grid_np(nlat, grid)
    return Plan.create_ex(nlat, nlon, L, M, m_offset, _lib.PLAN_VECTOR, cost, w, csphase, DEV)


def _bits_equal(a, b):
    a = torch.view_as_real(a) if a.is_complex() else a
    b = torch.view_as_real(b) if b.is_complex() else b
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


# ------------------------------------------------------------------------------------------------------------- tables
@pytest.mark.parametrize("csphase", [True, False])
def test_offset_vector_plan_tables_are_the_order_slice(csphase):
    nlat, nlon, L, M = 91, 192, 91, 91
    full = vplan(nlat, nlon, L, M, 0, csphase=csphase)
    tfull = full.table()
    # offsets off the 32-order tiles, a shard ending at mmax, one starting at 0
    for off, mloc in ((0, 40), (13, 20), (33, 31), (40, 51), (64, 27), (90, 1)):
        p = vplan(nlat, nlon, L, mloc, off, csphase=csphase)
        assert p.vector and p.query(7) == off and p.query(3) == mloc and p.query(2) == L
        assert p.query(5) == 2 * mloc * L * p.kp * 4
        assert _bits_equal(p.table(), tfull[:, off:off + mloc]), (off, mloc, csphase)


# ---------------------------------------------------------------------------------------------- stages on an order shard
def _analysis(plan, xc, prec):
    """complex (B, C, 2, nlat, m) -> (B, C, 2, L, m) through latspec_pack -> vector_legendre_analysis -> vector_spec_unpack(1), NaN-filled buffers"""
    lib, st = _lib.load(), _stream()
    B, C = xc.shape[:2]
    lat = torch.full((plan.latspec_elems(B, 2 * C),), NAN, device=DEV)
    spec = torch.full((plan.spec_elems(B, 2 * C),), NAN, device=DEV)
    out = torch.full((B, C, 2, plan.lmax, plan.mmax), NAN, dtype=torch.complex64, device=DEV)
    _lib.check(lib.b200sht_latspec_pack(plan.handle, _p(xc), _p(lat), B, 2 * C, st), "latspec_pack")
    _lib.check(lib.b200sht_vector_legendre_analysis(plan.handle, _p(lat), _p(spec), B, C, prec, st), "vector_legendre_analysis")
    _lib.check(lib.b200sht_vector_spec_unpack(plan.handle, _p(spec), _p(out), B, C, 1, st), "vector_spec_unpack")
    return out


def _synthesis(plan, c, prec):
    """complex (B, C, 2, L, m) -> (B, C, 2, nlat, m) through vector_spec_pack(0) -> vector_legendre_synthesis -> latspec_unpack"""
    lib, st = _lib.load(), _stream()
    B, C = c.shape[:2]
    lat = torch.full((plan.latspec_elems(B, 2 * C),), NAN, device=DEV)
    spec = torch.full((plan.spec_elems(B, 2 * C),), NAN, device=DEV)
    out = torch.full((B, C, 2, plan.nlat, plan.mmax), NAN, dtype=torch.complex64, device=DEV)
    _lib.check(lib.b200sht_vector_spec_pack(plan.handle, _p(c), _p(spec), B, C, 0, st), "vector_spec_pack")
    _lib.check(lib.b200sht_vector_legendre_synthesis(plan.handle, _p(spec), _p(lat), B, C, prec, st), "vector_legendre_synthesis")
    _lib.check(lib.b200sht_latspec_unpack(plan.handle, _p(lat), _p(out), B, 2 * C, st), "latspec_unpack")
    return out


@pytest.mark.parametrize("prec", [_lib.PREC_FP32, _lib.PREC_TF32])
@pytest.mark.parametrize("grid,nlat,nlon,L,M,B,C", [("equiangular", 91, 192, 91, 91, 2, 3), ("legendre-gauss", 130, 260, 100, 131, 1, 5)])
def test_offset_stages_are_the_order_slice(prec, grid, nlat, nlon, L, M, B, C):
    torch.manual_seed(333)
    full = vplan(nlat, nlon, L, M, 0, grid)
    xc = torch.randn(B, C, 2, nlat, M, dtype=torch.complex64, device=DEV)
    l = torch.arange(L, device=DEV)[:, None]
    c = torch.randn(B, C, 2, L, M, dtype=torch.complex64, device=DEV)
    c = torch.where(l >= torch.arange(M, device=DEV)[None, :], c, torch.full_like(c, complex(NAN, NAN)))   # l < m: never read
    ya, ys = _analysis(full, xc, prec), _synthesis(full, c, prec)
    assert torch.isfinite(torch.view_as_real(ya)).all() and torch.isfinite(torch.view_as_real(ys)).all()
    shards = [(0, 37), (37, 45), (82, M - 82)] if M > 91 else [(0, 40), (13, 20), (40, 51)]
    for off, mloc in shards:
        p = vplan(nlat, nlon, L, mloc, off, grid)
        sl = slice(off, off + mloc)
        a = _analysis(p, xc[..., sl].contiguous(), prec)
        assert _bits_equal(a, ya[..., sl]), (off, mloc, "analysis")
        below = l < (off + torch.arange(mloc, device=DEV))[None, :]
        assert (a.abs()[..., below] == 0).all(), "l < m_offset + m must be exact zeros"
        s = _synthesis(p, c[..., sl].contiguous(), prec)
        assert _bits_equal(s, ys[..., sl]), (off, mloc, "synthesis")


# ------------------------------------------------------------------------------------------------- virtual h x w ranks
def _rank_ops(cls, nlat, nlon, L, M, grid, precision, h, w, ih, iw):
    """CudaLocalOps of virtual rank (ih, iw): the module of world size 1 given this rank's shard geometry"""
    t = cls(nlat, nlon, L, M, grid, precision=precision)
    lat, ms = mbd.compute_split_shapes(nlat, h), mbd.compute_split_shapes(t.mmax, w)
    t.nlat_local, t.lat_offset = lat[ih], sum(lat[:ih])
    t.mmax_local, t.m_offset = ms[iw], sum(ms[:iw])
    return t, mbd.CudaLocalOps(t)


def _split(x, dim, n):
    return torch.split(x, mbd.compute_split_shapes(x.shape[dim], n), dim=dim)


def emulated_vsht(x, nlat, nlon, L, M, grid, precision, h, w):
    """x (B, C, 2, nlat, nlon) -> (B, C, 2, L, M): the stages of every virtual rank, the transposes as split / cat"""
    B, C = x.shape[:2]
    X = []
    for ih, xh in enumerate(_split(x, -2, h)):                  # polar shard of the input
        row = []
        for iw, xw in enumerate(_split(xh, 1, w)):               # azimuth transpose: channels split, all longitudes
            t, ops = _rank_ops(mbd.DistributedRealVectorSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            Cw = xw.shape[1]
            row.append(ops.fft(xw.reshape(B, 2 * Cw, t.nlat_local, nlon)).reshape(B, Cw, 2, t.nlat_local, t.mmax))
        X.append(torch.cat(row, dim=1))                          # back: all channels (of this latitude slice)
    X = torch.cat(X, dim=-2)
    out = []
    for iw, Xw in enumerate(_split(X, -1, w)):                   # order shards
        col = []
        for ih, Xh in enumerate(_split(Xw, 1, h)):               # polar transpose: channels split, all latitudes
            _, ops = _rank_ops(mbd.DistributedRealVectorSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            col.append(ops.vlegendre(Xh))
        out.append(torch.cat(col, dim=1))
    return torch.cat(out, dim=-1)


def emulated_ivsht(c, nlat, nlon, L, M, grid, precision, h, w):
    B = c.shape[0]
    Z = []
    for iw, cw in enumerate(_split(c, -1, w)):
        col = []
        for ih, ch in enumerate(_split(cw, 1, h)):
            _, ops = _rank_ops(mbd.DistributedInverseRealVectorSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            col.append(ops.ivlegendre(ch))
        Z.append(torch.cat(col, dim=1))
    Z = torch.cat(Z, dim=-1)
    y = []
    for ih, Zh in enumerate(_split(Z, -2, h)):
        row = []
        for iw, Zw in enumerate(_split(Zh, 1, w)):
            t, ops = _rank_ops(mbd.DistributedInverseRealVectorSHT, nlat, nlon, L, M, grid, precision, h, w, ih, iw)
            Cw = Zw.shape[1]
            row.append(ops.ifft(Zw.reshape(B, 2 * Cw, t.nlat_local, t.mmax), torch.float32).reshape(B, Cw, 2, t.nlat_local, nlon))
        y.append(torch.cat(row, dim=1))
    return torch.cat(y, dim=-2)


SINGLE_GPU = (2e-5, 3e-3)       # (fp32 rtol, TF32 relative L2) against the single-GPU modules
ORACLE = (1e-5, TF32_REL_L2)     # against the fp64 oracle: the bounds of tests/test_gpu_vector_sht.py


def _cmp(a, b, precision, name, bounds):
    if precision == "fp32":
        close(a, b, bounds[0], name)
    else:
        r = rel_l2(a, b)
        print(f"TF32 rel-L2 {name}: {r:.3e}")
        assert r < bounds[1], (name, r)


@pytest.mark.parametrize("h,w", [(2, 1), (1, 2), (2, 2), (4, 2)])
@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("grid,nlat,nlon,L,M", [("equiangular", 91, 180, None, None), ("legendre-gauss", 90, 180, 70, 20)])
def test_virtual_ranks_match_single_gpu_and_oracle(h, w, precision, grid, nlat, nlon, L, M):
    torch.manual_seed(333)
    B, C = 2, 5
    vsht = mb.RealVectorSHT(nlat, nlon, L, M, grid, precision=precision)
    ivsht = mb.InverseRealVectorSHT(nlat, nlon, L, M, grid, precision=precision)
    ov = V.RealVectorSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    oiv = V.InverseRealVectorSHT(nlat, nlon, L, M, grid, dtype=torch.float64)
    L, M = vsht.lmax, vsht.mmax
    tag = f"{h}x{w} {grid} {nlat}x{nlon} L={L} M={M} {precision}"

    x = torch.randn(B, C, 2, nlat, nlon)
    g = torch.randn(B, C, 2, L, M, dtype=torch.complex64) * torch.tril(torch.ones(L, M))
    xd, xs, xr = (x.to(DEV).requires_grad_(True), x.to(DEV).requires_grad_(True), x.double().requires_grad_(True))
    cd, cs, cr = emulated_vsht(xd, nlat, nlon, L, M, grid, precision, h, w), vsht(xs), ov(xr)
    for a, b in ((cd, g.to(DEV)), (cs, g.to(DEV)), (cr, g.to(torch.complex128))):
        a.backward(b)
    _cmp(cd, cs, precision, f"vsht vs single GPU {tag}", SINGLE_GPU)
    _cmp(xd.grad, xs.grad, precision, f"vsht grad vs single GPU {tag}", SINGLE_GPU)
    _cmp(cd, cr, precision, f"vsht vs oracle {tag}", ORACLE)
    _cmp(xd.grad, xr.grad, precision, f"vsht grad vs oracle {tag}", ORACLE)

    c = torch.randn(B, C, 2, L, M, dtype=torch.complex64) * torch.tril(torch.ones(L, M))
    gy = torch.randn(B, C, 2, nlat, nlon)
    cd, cs, cr = c.to(DEV).requires_grad_(True), c.to(DEV).requires_grad_(True), c.to(torch.complex128).requires_grad_(True)
    yd, ys, yr = emulated_ivsht(cd, nlat, nlon, L, M, grid, precision, h, w), ivsht(cs), oiv(cr)
    assert yd.dtype == torch.float32
    for a, b in ((yd, gy.to(DEV)), (ys, gy.to(DEV)), (yr, gy.double())):
        a.backward(b)
    _cmp(yd, ys, precision, f"ivsht vs single GPU {tag}", SINGLE_GPU)
    _cmp(cd.grad, cs.grad, precision, f"ivsht grad vs single GPU {tag}", SINGLE_GPU)
    _cmp(yd, yr, precision, f"ivsht vs oracle {tag}", ORACLE)
    _cmp(cd.grad, cr.grad, precision, f"ivsht grad vs oracle {tag}", ORACLE)


def test_world1_modules_bf16_and_6d_shape():
    """world size 1 on the CUDA stages: the 6-D (B, E, C, 2, H, W) shape of VortDivCRPSLoss, bf16 input, == the single-GPU modules"""
    torch.manual_seed(333)
    nlat, nlon = 46, 90
    dv, div = mbd.DistributedRealVectorSHT(nlat, nlon, precision="fp32"), mbd.DistributedInverseRealVectorSHT(nlat, nlon, precision="fp32")
    v, iv = mb.RealVectorSHT(nlat, nlon, precision="fp32"), mb.InverseRealVectorSHT(nlat, nlon, precision="fp32")
    x = torch.randn(2, 3, 2, 2, nlat, nlon).to(torch.bfloat16)
    xd, xs = x.to(DEV).requires_grad_(True), x.to(DEV).requires_grad_(True)
    yd, ys = div(dv(xd)), iv(v(xs))
    assert yd.shape == x.shape and yd.dtype == torch.float32
    close(yd, ys, 2e-5, "world 1 6-D bf16 round trip")
    gy = torch.randn(x.shape, device=DEV)
    yd.backward(gy)
    ys.backward(gy)
    assert xd.grad.dtype == torch.bfloat16
    close(xd.grad.float(), xs.grad.float(), 1e-2, "world 1 6-D bf16 gradient")


# ---------------------------------------------------------------------------------------------------------- refusals
def test_refusals_on_order_shards():
    lib = _lib.load()
    nlat, nlon, L, B, C = 32, 64, 32, 1, 2
    p = vplan(nlat, nlon, L, 17, 16)
    st = _stream()
    x = torch.zeros(B, C, 2, nlat, nlon, device=DEV)
    coeffs = torch.zeros(B, C, 2, L, 17, dtype=torch.complex64, device=DEV)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    spec = torch.zeros(p.spec_elems(B, 2 * C), device=DEV)
    lat = torch.zeros(p.latspec_elems(B, 2 * C), device=DEV)
    assert lib.b200sht_vsht_workspace_bytes(p.handle, B, C) == -1
    for prec in (_lib.PREC_FP32, _lib.PREC_TF32):
        assert lib.b200sht_vsht_forward(p.handle, _p(x), _lib.F32, B, C, _p(coeffs), _p(ws), prec, st) == -1
        assert lib.b200sht_vsht_inverse(p.handle, _p(coeffs), _p(x), _lib.F32, B, C, _p(ws), prec, st) == -1
        assert lib.b200sht_vsht_forward_adjoint(p.handle, _p(coeffs), _p(x), _lib.F32, B, C, _p(ws), prec, st) == -1
        assert lib.b200sht_vsht_inverse_adjoint(p.handle, _p(x), _lib.F32, B, C, _p(coeffs), _p(ws), prec, st) == -1
    assert lib.b200sht_vector_legendre_synthesis_tiled(p.handle, _p(spec), _p(lat), B, C, st) == -1
    assert lib.b200sht_vector_legendre_analysis(p.handle, _p(lat), _p(spec), B, C, _lib.PREC_FP32X3, st) == -3
    # the plan of all orders still serves the one-call entries; VECTOR | FFT_ONLY is refused
    assert lib.b200sht_vsht_workspace_bytes(vplan(nlat, nlon, L, 33, 0).handle, B, C) > 0
    cost, w = _grid_np(nlat, "equiangular")
    with pytest.raises(_lib.B200ShtError):
        Plan.create_ex(nlat, nlon, L, 17, 16, _lib.PLAN_VECTOR | _lib.PLAN_FFT_ONLY, cost, w, True, DEV)
    for cls, arg in ((mbd.DistributedRealVectorSHT, x), (mbd.DistributedInverseRealVectorSHT, torch.zeros(B, C, 2, L, 33, dtype=torch.complex64, device=DEV))):
        with pytest.raises(_lib.B200ShtError):
            cls(nlat, nlon, precision="fp32x3")(arg)
    torch.cuda.synchronize()

"""The CUDA per-rank stage of DistributedNeighborhoodAttentionS2 on one GPU, h x w virtual ranks in one process:

* the forward and the query side on every rank's window plan, run with the rank's (b, h) pairs at heads = 1: y, lse, D and dq are
  bit-identical to the corresponding slice of the single-GPU kernels' outputs, at FCN3's processor grid (360 x 720 Legendre-Gauss,
  theta_c = 4 pi / 359), at 721 x 1440 equiangular -> 360 x 720 Legendre-Gauss and at a small equiangular grid whose pole windows are whole
  rings wider than one staged chunk, h in {2, 4}, w in {1, 2} (w splits the pairs);
* dk and dv of the window plans, added into the owners' rows in rank order as the halo's adjoint adds them: bit-identical to the single-GPU
  kernel on the input rows only one rank's output rows reach, within the per-element bound of tests/attention_ref.py (C_ATTN) against fp64
  everywhere, and identical run to run;
* the module's arithmetic on every rank (projections on the local pixels, the pair transposes and the halo as slicing, window attention,
  output projection) against the single-GPU module: output, input and parameter gradients at rtol 1e-5 in fp32, 2e-3 with TF32, bf16 inputs;
* the window path launches the same attn_query_kernel / attn_kv_kernel instantiations as the single-GPU call.
The module itself needs process groups and does not run here; its collectives and autograd are covered on CPU, with the oracle stage, by
tests/test_distributed_attention_cpu.py."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import attention_ref as AR
import makani_b200.distributed as mbd
from makani_b200 import attention as A
from makani_b200.distributed import attention as DA
from makani_b200.distributed import disco as DD
from test_gpu_attention import C_ATTN, _launched_attn, _plan_omega, _run, _untouched, attn_kernels, em_vec
from test_gpu_engine import launched_kernels
from test_gpu_parity import close

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

# in_shape, out_shape, grid_in, grid_out, theta_cutoff, B, heads, E_k, E_v
GEOMS = {
    "processor": ((360, 720), (360, 720), "legendre-gauss", "legendre-gauss", 4 * math.pi / 359, 1, 4, 16, 8),
    "downsample": ((721, 1440), (360, 720), "equiangular", "legendre-gauss", 4 * math.pi / 1440, 1, 2, 16, 16),
    # every row of the 9 x 520 grid is a whole ring of 520 input points within 1.5 spacings of the pole rows: more columns than one chunk
    # of the staged K / V (90 at E 64 + 8) or q / dy
    "rings": ((9, 520), (9, 260), "equiangular", "equiangular", 1.5 * math.pi / 8, 1, 2, 64, 8),
}


def _ops(key, win):
    return DA.CudaAttentionLocalOps(SimpleNamespace(_key=key, window=win))


def _pairs(x, H):
    """(B, P, H E) -> (B H, P, E), each (b, h) pair contiguous"""
    B, P = x.shape[:2]
    return x.view(B, P, H, -1).permute(0, 2, 1, 3).reshape(B * H, P, -1)


def _operands(ish, osh, B, H, ek, ev, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = math.sqrt(3.0) * torch.randn(B, osh[0] * osh[1], H * ek, generator=g, device=DEV)
    k = math.sqrt(3.0) * torch.randn(B, ish[0] * ish[1], H * ek, generator=g, device=DEV)
    v = torch.randn(B, ish[0] * ish[1], H * ev, generator=g, device=DEV)
    dy = torch.randn(B, osh[0] * osh[1], H * ev, generator=g, device=DEV)
    return q, k, v, dy


def _window_runs(key, h, w, q, k, v, dy, ek):
    """every virtual rank's two C-ABI calls on its window plan at heads = 1, over pair operands (B H, P, E):
    yields (window, pair rows r0 .. r0 + n, (y, lse, dq, dk, dv, D)), ranks in (azimuth pairs, polar rank) order"""
    nb = A.get_neighbourhood(*key)
    (hi, wi), (ho, wo) = key[0], key[1]
    wins = DD.disco_windows(nb, mbd.compute_split_shapes(ho, h))
    assert wins[0].lo == 0 and wins[-1].hi == hi
    scale = 1.0 / math.sqrt(ek)
    r0 = 0
    for n in mbd.compute_split_shapes(q.shape[0], w):
        for win in wins:
            o, i = slice(win.t0 * wo, win.t1 * wo), slice(win.lo * wi, win.hi * wi)
            sl = [x[r0 : r0 + n, s].contiguous() for x, s in ((q, o), (k, i), (v, i), (dy, o))]
            outs, bufs = _run(_ops(key, win)._plan(DEV), *sl, 1, scale)
            assert all(_untouched(b, x) for b, x in zip(bufs, outs)), "a kernel wrote outside its output"
            yield win, r0, n, outs
        r0 += n


def _summed(key, h, w, q, k, v, dy, ek):
    """the window runs with dk, dv added into the owners' rows in rank order (the order of halo_adjoint) and y, lse of each window placed"""
    BH, (hi, wi), (ho, wo) = q.shape[0], key[0], key[1]
    dk, dv = torch.zeros_like(k), torch.zeros_like(v)
    y, lse = torch.empty(BH, ho * wo, v.shape[2], device=DEV), torch.empty(BH, 1, ho * wo, device=DEV)
    reach = np.zeros(hi, dtype=int)
    for win, r0, n, (yw, lw, _, dkw, dvw, _) in _window_runs(key, h, w, q, k, v, dy, ek):
        i = slice(win.lo * wi, win.hi * wi)
        dk[r0 : r0 + n, i] += dkw
        dv[r0 : r0 + n, i] += dvw
        y[r0 : r0 + n, win.t0 * wo : win.t1 * wo] = yw
        lse[r0 : r0 + n, :, win.t0 * wo : win.t1 * wo] = lw
        if r0 == 0:
            reach[np.unique(win.psi.col // wi) + win.lo] += 1
    return dk, dv, y, lse, reach


@pytest.mark.parametrize("w", [1, 2])
@pytest.mark.parametrize("h", [2, 4])
@pytest.mark.parametrize("geom", list(GEOMS))
def test_window_kernels_match_single_gpu_slices(geom, h, w):
    ish, osh, gi, go, cutoff, B, H, ek, ev = GEOMS[geom]
    key = (ish, osh, gi, go, cutoff)
    q, k, v, dy = _operands(ish, osh, B, H, ek, ev, seed=7)
    scale = 1.0 / math.sqrt(ek)
    (y, lse, dq, dk, dv, D), _ = _run(A.get_plan(key, DEV), q, k, v, dy, H, scale)
    qp, kp, vp, dyp = (_pairs(x, H) for x in (q, k, v, dy))
    ys, dqs, dks, dvs = (_pairs(x, H) for x in (y, dq, dk, dv))
    lses, Ds = lse.reshape(B * H, 1, -1), D.reshape(B * H, 1, -1)
    wo = osh[1]
    for win, r0, n, (yw, lw, dqw, _, _, Dw) in _window_runs(key, h, w, qp, kp, vp, dyp, ek):
        r, o = slice(r0, r0 + n), slice(win.t0 * wo, win.t1 * wo)
        for what, got, want in (("y", yw, ys[r, o]), ("lse", lw, lses[r, :, o]), ("D", Dw, Ds[r, :, o]), ("dq", dqw, dqs[r, o])):
            assert torch.equal(got, want), (geom, h, w, what, win.t0, win.t1, r0)
    sdk, sdv, _, _, reach = _summed(key, h, w, qp, kp, vp, dyp, ek)
    one = torch.from_numpy(np.repeat(reach == 1, ish[1])).to(DEV)
    assert one.any(), reach
    assert torch.equal(sdk[:, one], dks[:, one]) and torch.equal(sdv[:, one], dvs[:, one]), (geom, h, w)
    print(f"\n[dist attention] {geom} {h}x{w}: {int((reach == 1).sum())} of {ish[0]} input rows reached by one rank, bit-identical")


@pytest.mark.parametrize("h", [2, 3, 4])
@pytest.mark.parametrize("geom", [((33, 64), (33, 64), "equiangular", "equiangular", 3.0, 2, 2, 8, 4),
                                  ((33, 64), (17, 32), "equiangular", "legendre-gauss", 3.0, 1, 4, 16, 12),
                                  ((9, 520), (9, 260), "equiangular", "equiangular", 1.5, 1, 1, 64, 8)])
def test_summed_dk_dv_within_bound_and_deterministic(geom, h):
    ish, osh, gi, go, units, B, H, ek, ev = geom
    key = (ish, osh, gi, go, units * math.pi / (ish[0] - 1))
    nb = A.get_neighbourhood(*key)
    q, k, v, dy = (_pairs(x, H) for x in _operands(ish, osh, B, H, ek, ev, seed=11))
    dk, dv, y, lse, reach = _summed(key, h, 1, q, k, v, dy, ek)
    again = _summed(key, h, 1, q, k, v, dy, ek)
    assert torch.equal(dk, again[0]) and torch.equal(dv, again[1])
    assert (reach > 1).any(), reach
    s32 = torch.tensor(1.0 / math.sqrt(ek), dtype=torch.float32, device=DEV)
    om = _plan_omega(nb, ish[0], ish[1])
    bw = AR.backward((q * s32).double(), k.double(), v.double(), y.double(), lse.double(), dy.double(), nb.row_ptr, nb.col, om, ish[1], osh[1],
                     1, s32.item())
    needs = {"dk": AR.need(dk, *bw["dk"]), "dv": AR.need(dv, *bw["dv"])}
    print(f"\n[dist attention] {ish}->{osh} h={h}: summed over the windows needs C >= " + ", ".join(f"{w} {c:.3g}" for w, c in needs.items()))
    assert all(c <= C_ATTN for c in needs.values()), needs


@pytest.mark.parametrize("geom", ["processor", "rings"])
def test_window_path_launches_the_single_gpu_instantiations(geom):
    ish, osh, gi, go, cutoff, B, H, ek, ev = GEOMS[geom]
    key = (ish, osh, gi, go, cutoff)
    q, k, v, dy = _operands(ish, osh, B, H, ek, ev, seed=3)
    want = attn_kernels(*em_vec(ek, ev, 0))
    single = launched_kernels(lambda: _run(A.get_plan(key, DEV), q, k, v, dy, H, 1.0 / math.sqrt(ek)), lambda n: _launched_attn(n) == want)
    pq, pk, pv, pdy = (_pairs(x, H) for x in (q, k, v, dy))
    windows = launched_kernels(lambda: list(_window_runs(key, 2, 2, pq, pk, pv, pdy, ek)), lambda n: _launched_attn(n) == want)
    assert _launched_attn(single) == _launched_attn(windows) == want, (single, windows)


# ------------------------------------------------------------------------------------------------------------- module arithmetic
def emulated_attention(mod, query, key, value, h, w):
    """the forward of DistributedNeighborhoodAttentionS2 on h x w virtual ranks: projections and output projection on every rank's local
    pixels, the pair all-to-alls and the halo as slicing, the attention on every rank's window plan with its pairs at heads = 1"""
    B, H = query.shape[0], mod.num_heads
    lat_in, lon_in = mbd.compute_split_shapes(mod.nlat_in, h), mbd.compute_split_shapes(mod.nlon_in, w)
    lat_out, lon_out = mbd.compute_split_shapes(mod.nlat_out, h), mbd.compute_split_shapes(mod.nlon_out, w)

    def pairs(x, weight, bias, lats, lons):
        """every rank's projection of its pixels as (B H, rows, lons, E), placed on the whole grid"""
        rows = []
        for xr in torch.split(x, lats, dim=2):
            cols = [A._project_points(xc, weight, bias).view(B, xc.shape[2], xc.shape[3], H, -1).permute(0, 3, 1, 2, 4)
                    for xc in torch.split(xr, lons, dim=3)]
            rows.append(torch.cat(cols, dim=3))
        return torch.cat(rows, dim=2).reshape(B * H, x.shape[2], x.shape[3], -1)

    q = pairs(query, mod.q_weights, mod.q_bias, lat_out, lon_out)
    k = pairs(key, mod.k_weights, mod.k_bias, lat_in, lon_in)
    v = pairs(value, mod.v_weights, mod.v_bias, lat_in, lon_in)
    wins = DD.disco_windows(A.get_neighbourhood(*mod._key), lat_out)
    ys = []
    for win in wins:
        yw, r0 = [], 0
        for n in mbd.compute_split_shapes(B * H, w):
            r = slice(r0, r0 + n)
            yw.append(A._NeighborhoodAttention.apply(q[r, win.t0 : win.t1].reshape(n, -1, q.shape[3]), k[r, win.lo : win.hi].reshape(n, -1, k.shape[3]),
                                                     v[r, win.lo : win.hi].reshape(n, -1, v.shape[3]), _ops(mod._key, win), 1, mod.scale)
                      .view(n, win.t1 - win.t0, mod.nlon_out, -1))
            r0 += n
        ys.append(torch.cat(yw, dim=0))
    y = torch.cat(ys, dim=1)                                                                     # (B H, nlat_out, nlon_out, E_v)
    out = []
    for yr in torch.split(y, lat_out, dim=1):
        cols = []
        for yc in torch.split(yr, lon_out, dim=2):
            P = yc.shape[1] * yc.shape[2]
            yl = yc.reshape(B, H, P, -1).transpose(1, 2).reshape(B, P, -1)
            cols.append(A._project_out(yl, mod.proj_weights, mod.proj_bias).view(B, -1, yc.shape[1], yc.shape[2]))
        out.append(torch.cat(cols, dim=3))
    return torch.cat(out, dim=2)


MODULE_CASES = [
    # in_channels, in_shape, out_shape, grid_in, grid_out, heads, k_channels, out_channels, bias, cutoff units, separate key / value
    (12, (33, 64), (33, 64), "equiangular", "equiangular", 4, None, None, True, 3.0, False),
    (6, (91, 180), (46, 90), "equiangular", "legendre-gauss", 2, 16, 10, True, 3.0, True),
]


def _module(case, seed):
    cin, ish, osh, gi, go, H, ck, cv, bias, units, _ = case
    torch.manual_seed(seed)
    mod = A.NeighborhoodAttentionS2(cin, ish, osh, gi, go, num_heads=H, bias=bias, theta_cutoff=units * math.pi / (ish[0] - 1), k_channels=ck,
                                    out_channels=cv).to(DEV)
    if bias:
        with torch.no_grad():
            for n in ("q_bias", "k_bias", "v_bias", "proj_bias"):
                getattr(mod, n).normal_()
    return mod


def _step(mod, f, xs, gy, tf32):
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = tf32
    try:
        mod.zero_grad()
        ins = [x.clone().requires_grad_(True) for x in xs]
        out = f(*ins)
        out.backward(gy)
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    return out.detach(), [x.grad for x in ins], {n: p.grad.clone() for n, p in mod.named_parameters()}


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("h,w", [(2, 1), (2, 2), (4, 2)])
@pytest.mark.parametrize("case", MODULE_CASES, ids=["same-grid", "downsample"])
def test_virtual_ranks_match_single_gpu_module(case, h, w, tf32):
    cin, ish, osh, separate = case[0], case[1], case[2], case[10]
    mod = _module(case, 21)
    g = torch.Generator(device=DEV).manual_seed(4)
    query = torch.randn(2, cin, *osh, generator=g, device=DEV)
    xs = [query] + ([torch.randn(2, cin, *ish, generator=g, device=DEV) for _ in range(2)] if separate else [])
    gy = torch.randn(2, mod.out_channels, *osh, generator=g, device=DEV)
    ref = _step(mod, mod, xs, gy, tf32)
    got = _step(mod, lambda *t: emulated_attention(mod, *(t if separate else t * 3), h, w), xs, gy, tf32)
    rtol = 2e-3 if tf32 else 1e-5
    close(got[0], ref[0], rtol, f"{h}x{w} out")
    for n, (a, b) in enumerate(zip(got[1], ref[1])):
        close(a, b, rtol, f"{h}x{w} d input {n}")
    for n, b in ref[2].items():
        if n == "k_bias":   # exactly zero: both sides are rounding noise, held to the key weights' gradient scale as in test_gpu_attention
            assert got[2][n].abs().max().item() <= rtol * ref[2]["k_weights"].abs().max().item()
            continue
        close(got[2][n], b, rtol, f"{h}x{w} d {n}")


def test_virtual_ranks_accept_bf16_inputs():
    case = MODULE_CASES[1]
    cin, ish, osh = case[0], case[1], case[2]
    mod = _module(case, 5)
    g = torch.Generator(device=DEV).manual_seed(6)
    xs = [torch.randn(1, cin, *shape, generator=g, device=DEV).to(torch.bfloat16) for shape in (osh, ish, ish)]
    gy = torch.randn(1, mod.out_channels, *osh, generator=g, device=DEV)
    ref = _step(mod, mod, xs, gy, False)
    got = _step(mod, lambda *t: emulated_attention(mod, *t, 4, 2), xs, gy, False)
    assert got[0].dtype == torch.float32 and all(x.dtype == torch.bfloat16 for x in got[1])
    close(got[0], ref[0], 1e-5, "bf16 out")
    for n, (a, b) in enumerate(zip(got[1], ref[1])):
        close(a, b, 1e-2, f"bf16 d input {n}")   # the input gradients are rounded to bf16 on both sides

"""fp64 references of the three neighbourhood-attention kernels of csrc/attention.cu on their exact fp32 operands, each with the magnitude
terms of a first-order rounding bound.  Plain PyTorch over the (p, n) pair gather of `attention_oracle.pairs`: the helpers run on the CPU
(tests/test_attention_ref_cpu.py) or on the device in float64 (tests/test_gpu_attention.py).

Operands.  The kernels multiply q by the fp32 `scale` once, q~ = fl(scale q), and form every logit as an E_k-term fma chain on q~ and k.
The references take q~ itself (`qt`; on the GPU it is `q * scale` in fp32, the same IEEE rounding) and compute l_n = sum_c q~_c k_c in fp64,
so the only error left in a logit is the chain's: |dl_n| <= E_k u L_n with L_n = sum_c |q~_c k_c| and u = 2^-24.  omega is the plan's fp32
quadrature weight.  Every reference returns (ref, mag): a kernel output `got` is within the bound when |got - ref| <= C u mag, C calibrated on
an H100 (DESIGN.md section 5).  Below, N = |N(t, p)| (the same for every p of an output row t), alpha_n = omega_n exp(l_n - lse) (sum 1),
M = max_n l_n, and `ulp` bounds are those of the CUDA math library without fast-math: expf <= 2 ulp (relative <= 4u), logf <= 1 ulp.

Forward (y, lse).  The kernel walks n with a running max m and sum l: when l_n > m it multiplies l and acc by c = expf(fl(m - l_n)) and sets
m = l_n; then e = fl(omega expf(fl(l_n - m))), l += e, acc = fma(e, v_n, acc); finally y = fl(acc fl(1 / l)), lse = fl(m + logf(l)).  The
weight with which term n reaches acc and l carries, relative to omega_n exp(l_n - M):
  * the logit chain, E_k u L_n;
  * the subtraction l_n - m and those of the rescales after n: all differences have one sign and telescope to l_n - M, so u |l_n - M|;
  * expf and the multiply by omega, 4u + u, and expf of each of the at most N - 1 later rescales, 4u each: u (4N + 1) in all.
A relative error eps_n of term n's weight moves y by alpha_n eps_n (v_n - y) and lse by alpha_n eps_n.  The roundings of the sums themselves
are relative to partial sums: acc takes N fma roundings and at most N - 1 rescale roundings, each <= u sum_n alpha_n |v_n| (after the
division by l); l takes N - 1 additions (the first is exact) and N - 1 rescale roundings, and 1 / l and the final multiply add 2, so y moves
by at most 2N u |y| through l.  Hence
    |y^ - y| <= u [ sum_n alpha_n (E_k L_n + |l_n - M| + 4N + 1) |v_n - y|  +  2N (sum_n alpha_n |v_n| + |y|) ]
    |lse^ - lse| <= u [ sum_n alpha_n (E_k L_n + |l_n - M| + 4N + 1)  +  2N  +  2 |lse - M|  +  |lse| ]
(log l = lse - M, so logf's ulp is 2u |lse - M|, and the final add rounds once.)

Backward, on the kernel's own fp32 y and lse (the exact operands of b200sht_attention_backward, so only the backward's roundings count).
  * D = <dy, y>: an E_v-term chain, |D^ - D| <= E_v u G with G = sum_c |dy_c y_c|.
  * alpha_n = fl(omega fl expf(fl(l_n - lse))): relative error eps_n <= u (E_k L_n + |l_n - lse| + 5).
  * g_n = <dy, v_n>: an E_v-term chain, E_v u H_n with H_n = sum_c |dy_c v_nc|; dl_n = fl(alpha_n fl(g_n - D^)) rounds twice more.  So
        |dl^_n - dl_n| <= u Mdl_n,   Mdl_n = alpha_n [ (eps_n / u + 2) |g_n - D| + E_v (H_n + G) ]
    which holds however much g_n - D cancels.
  * dq = fl(scale fl-sum_n dl_n k_n): N fma roundings and one multiply,
        |dq^ - dq| <= u [ |scale| sum_n (Mdl_n + N |dl_n|) |k_n| + |dq| ].
  * dk_n = sum_p dl_pn q~_p and dv_n = sum_p alpha_pn dy_p over the P_n output points that reach n, one fma chain each:
        |dk^ - dk| <= u sum_p (Mdl_pn + P_n |dl_pn|) |q~_p|,   |dv^ - dv| <= u sum_p alpha_pn (eps_pn / u + P_n) |dy_p|.
The key/value kernel recomputes l, alpha and dl with the same fma sequences on the same operands and D^ from the query-side kernel, so its
dl are the query side's bit for bit and the same Mdl bounds them.

Gradual underflow.  The kernels are built without fast-math, so subnormals are kept, and there the roundings above are absolute: an ulp is
2^-149 (`TINY`) however small the value.  A weight whose exponent argument is below about -87 is subnormal (logits of magnitude 100 make
most of them so), and the relative terms alone then bound the dk and dv of points that no output attends to by less than one subnormal ulp
(with the relative terms alone, the logits-100 case of the GPU suite needs C = 3.4e3 there, and nowhere else).  So every rounding that can produce a subnormal also gets
its absolute term: per weight 3 TINY (expf's 2 ulp and the multiply by omega), per product or fma TINY; in the forward each of the at most
N rescales by a subnormal c adds 3 TINY per unit of the rescaled sum (at most N), so a weight carries (3 + 3N) TINY and y and lse move by
that over l.  These terms are below 2^-120 relative to any normal output.
"""
import torch

from attention_oracle import pairs

U32 = 2.0 ** -24
TINY = 2.0 ** -149      # the subnormal ulp of fp32
SUB = TINY / U32         # TINY in the units of `mag`


def _row(row_ptr, col, nlon_in, nlon_out, t, device):
    p, n = pairs(row_ptr, col, nlon_in, nlon_out, t)
    return torch.from_numpy(p).to(device), torch.from_numpy(n).to(device), int(row_ptr[t + 1] - row_ptr[t])


def _logits(qh, kh, t, nlon_out, seg, n):
    """l (B, pairs, H) and L = sum_c |q~_c k_c|, with q~ the scaled query"""
    prod = qh[:, t * nlon_out + seg] * kh[:, n]
    return prod.sum(-1), prod.abs().sum(-1)


def forward(qt, k, v, row_ptr, col, omega, nlon_in, nlon_out, heads):
    """(y, mag_y), (lse, mag_lse) of the forward kernel on the scaled query qt = q~, keys k and values v (module docstring).  Layouts as
    attention_oracle.attention: qt, k (B, points, H E_k), v (B, points, H E_v) -> y (B, P_out, H E_v), lse (B, H, P_out)."""
    B, dev, dt = qt.shape[0], qt.device, qt.dtype
    ek, ev = qt.shape[2] // heads, v.shape[2] // heads
    qh, kh, vh = qt.view(B, -1, heads, ek), k.view(B, -1, heads, ek), v.view(B, -1, heads, ev)
    om = torch.as_tensor(omega, dtype=dt, device=dev)
    ys, mys, ls, mls = [], [], [], []
    for t in range(len(row_ptr) - 1):
        seg, n, N = _row(row_ptr, col, nlon_in, nlon_out, t, dev)
        lg, L = _logits(qh, kh, t, nlon_out, seg, n)
        idx = seg.view(1, -1, 1).expand_as(lg)
        m = torch.full((B, nlon_out, heads), -torch.inf, dtype=dt, device=dev).scatter_reduce(1, idx, lg, "amax")
        e = om[n // nlon_in].view(1, -1, 1) * torch.exp(lg - m[:, seg])
        s = torch.zeros(B, nlon_out, heads, dtype=dt, device=dev).index_add(1, seg, e)
        a = e / s[:, seg]
        vn = vh[:, n]
        y = torch.zeros(B, nlon_out, heads, ev, dtype=dt, device=dev).index_add(1, seg, a[..., None] * vn)
        w = a * (ek * L + (lg - m[:, seg]).abs() + 4 * N + 1)
        spread = torch.zeros_like(y).index_add(1, seg, w[..., None] * (vn - y[:, seg]).abs())
        sv = torch.zeros_like(y).index_add(1, seg, a[..., None] * vn.abs())
        lse = m + torch.log(s)
        sub = (3 + 3 * N) * SUB / s                                             # a weight's subnormal roundings over l
        mlse = torch.zeros_like(lse).index_add(1, seg, w) + 2 * N + 2 * (lse - m).abs() + lse.abs() + N * sub
        svn = torch.zeros_like(y).index_add(1, seg, vn.abs())
        ys.append(y.reshape(B, nlon_out, heads * ev))
        mys.append((spread + 2 * N * (sv + y.abs()) + sub[..., None] * (svn + N * y.abs())).reshape(B, nlon_out, heads * ev))
        ls.append(lse.permute(0, 2, 1))
        mls.append(mlse.permute(0, 2, 1))
    return (torch.cat(ys, 1), torch.cat(mys, 1)), (torch.cat(ls, 2), torch.cat(mls, 2))


def backward(qt, k, v, y, lse, dy, row_ptr, col, omega, nlon_in, nlon_out, heads, scale):
    """{"D", "dq", "dk", "dv": (ref, mag)} of the two backward kernels on the scaled query qt = q~, k, v, the forward's y and lse and the
    output gradient dy (module docstring).  dq is the gradient with respect to the unscaled query (scale sum dl k), dk the one of
    l = <q~, k> (sum dl q~).  D and lse are (B, H, P_out), the gradients have the layouts of q, k and v."""
    B, dev, dt = qt.shape[0], qt.device, qt.dtype
    ek, ev = qt.shape[2] // heads, v.shape[2] // heads
    qh, kh, vh = qt.view(B, -1, heads, ek), k.view(B, -1, heads, ek), v.view(B, -1, heads, ev)
    dyh = dy.view(B, -1, heads, ev)
    om = torch.as_tensor(omega, dtype=dt, device=dev)
    Dprod = dyh * y.view(B, -1, heads, ev)
    D, G = Dprod.sum(-1), Dprod.abs().sum(-1)                                   # (B, P_out, H)
    dq, mdq = torch.zeros_like(qh), torch.zeros_like(qh)
    dk, mdk1, mdk2 = torch.zeros_like(kh), torch.zeros_like(kh), torch.zeros_like(kh)
    dv, mdv1, mdv2 = torch.zeros_like(vh), torch.zeros_like(vh), torch.zeros_like(vh)
    P = torch.zeros(kh.shape[1], dtype=dt, device=dev)                          # pairs reaching each input point
    for t in range(len(row_ptr) - 1):
        seg, n, N = _row(row_ptr, col, nlon_in, nlon_out, t, dev)
        o = t * nlon_out + seg
        lg, L = _logits(qh, kh, t, nlon_out, seg, n)
        ls = lse[:, :, o].permute(0, 2, 1)
        a = om[n // nlon_in].view(1, -1, 1) * torch.exp(lg - ls)
        gprod = dyh[:, o] * vh[:, n]
        gmD = gprod.sum(-1) - D[:, o]
        dl = a * gmD
        eps = ek * L + (lg - ls).abs() + 5
        mdl = a * ((eps + 2) * gmD.abs() + ev * (gprod.abs().sum(-1) + G[:, o])) + (3 * gmD.abs() + 1) * SUB
        kn, qp, dyp = kh[:, n], qh[:, o], dyh[:, o]
        rows = slice(t * nlon_out, (t + 1) * nlon_out)
        dq[:, rows] = torch.zeros(B, nlon_out, heads, ek, dtype=dt, device=dev).index_add(1, seg, dl[..., None] * kn)
        mdq[:, rows] = torch.zeros_like(dq[:, rows]).index_add(1, seg, (mdl + N * dl.abs())[..., None] * kn.abs()) + N * SUB
        dk.index_add_(1, n, dl[..., None] * qp)
        mdk1.index_add_(1, n, mdl[..., None] * qp.abs())
        mdk2.index_add_(1, n, dl.abs()[..., None] * qp.abs())
        dv.index_add_(1, n, a[..., None] * dyp)
        mdv1.index_add_(1, n, (a * eps + 3 * SUB)[..., None] * dyp.abs())
        mdv2.index_add_(1, n, a[..., None] * dyp.abs())
        P.index_add_(0, n, torch.ones(len(n), dtype=dt, device=dev))
    Pn = P.view(1, -1, 1, 1)
    dq = scale * dq
    flat = lambda x: x.reshape(B, x.shape[1], -1)  # noqa: E731
    return {
        "D": (D.permute(0, 2, 1), (ev * G).permute(0, 2, 1)),
        "dq": (flat(dq), flat(abs(scale) * mdq + dq.abs() + SUB)),
        "dk": (flat(dk), flat(mdk1 + Pn * (mdk2 + SUB))),
        "dv": (flat(dv), flat(mdv1 + Pn * (mdv2 + SUB))),
    }


def need(got, ref, mag):
    """the smallest C with |got - ref| <= C u mag for every element (0 / 0 counts as 0); inf where got or ref is not finite"""
    err = (got.double() - ref.double()).abs()
    if not torch.isfinite(err).all():
        return float("inf")
    return (err / (U32 * mag.double() + 1e-300)).max().item()

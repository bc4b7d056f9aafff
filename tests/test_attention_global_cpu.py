"""Global attention on the CPU: the invariants of the fp64 oracle (tests/attention_global_oracle.py) that pin the restated AttentionS2
contract without torch-harmonics, the module's constructor surface and refusals, the shim name, the C ABI symbols, and what the compiler
made of csrc/attention_global.cu (no register spills, wgmma in every instantiation).  Needs neither a GPU nor torch-harmonics."""
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import attention_global_oracle as GO  # noqa: E402
from makani_b200 import attention as A  # noqa: E402
from makani_b200 import _lib  # noqa: E402
from makani_b200._lib import B200ShtError  # noqa: E402
from makani_b200.quadrature import _grid_np  # noqa: E402

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")


def _operands(B, H, nq, nk, dqk, dv, seed=0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, H, nq, dqk, generator=g, dtype=torch.float64)
    k = torch.randn(B, H, nk, dqk, generator=g, dtype=torch.float64)
    v = torch.randn(B, H, dv, nk, generator=g, dtype=torch.float64)
    return q, k, v


@pytest.mark.parametrize("grid", ["equiangular", "legendre-gauss"])
def test_oracle_is_sdpa_with_the_log_weight_mask(grid):
    """the contract is torch's SDPA with attn_mask = log w"""
    q, k, v = _operands(2, 3, 40, 9 * 18, 8, 16)
    bias = GO.key_bias(9, 18, grid)
    o, _ = GO.attention(q, k, v, bias, 0.4)
    ref = F.scaled_dot_product_attention(q, k, v.transpose(-1, -2), attn_mask=bias.view(1, 1, 1, -1), scale=0.4)
    assert torch.allclose(o, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("grid", ["equiangular", "legendre-gauss"])
def test_oracle_zero_queries_give_the_quadrature_mean(grid):
    """q = 0: every key has logit log w_j, so o = sum_j w_j v_j / sum_j w_j"""
    nlat, nlon = 7, 12
    _, k, v = _operands(1, 2, 5, nlat * nlon, 8, 8)
    q = torch.zeros(1, 2, 5, 8, dtype=torch.float64)
    o, lse = GO.attention(q, k, v, GO.key_bias(nlat, nlon, grid), 1.0)
    w = torch.from_numpy(np.repeat(2 * np.pi * _grid_np(nlat, grid)[1] / nlon, nlon))
    mean = (v * w).sum(-1) / w.sum()
    assert torch.allclose(o, mean[:, :, None, :].expand_as(o), rtol=1e-12, atol=1e-12)
    assert torch.allclose(lse, torch.log(w.sum()).expand_as(lse), rtol=1e-12)   # sum_j w_j = 4 pi
    assert abs(float(w.sum()) - 4 * np.pi) < 1e-10


def test_oracle_reproduces_constant_values():
    q, k, _ = _operands(1, 2, 30, 60, 16, 8)
    v = torch.full((1, 2, 8, 60), 2.5, dtype=torch.float64)
    o, _ = GO.attention(q, k, v, GO.key_bias(5, 12, "equiangular"), 0.7)
    assert torch.allclose(o, torch.full_like(o, 2.5), rtol=1e-13)


def test_oracle_longitude_roll_rolls_the_output():
    """with nlon_in == nlon_out, rolling query, key and value by s longitudes rolls the module's output by s"""
    g = torch.Generator().manual_seed(3)
    C, heads, shape_in, shape_out = 8, 2, (6, 10), (4, 10)
    params = {n: torch.randn(s, generator=g, dtype=torch.float64) for n, s in
              [("q_weights", (C, C, 1, 1)), ("k_weights", (C, C, 1, 1)), ("v_weights", (C, C, 1, 1)), ("proj_weights", (C, C, 1, 1)),
               ("q_bias", (C,)), ("k_bias", (C,)), ("v_bias", (C,)), ("proj_bias", (C,))]}
    query = torch.randn(2, C, *shape_out, generator=g, dtype=torch.float64)
    kv = torch.randn(2, C, *shape_in, generator=g, dtype=torch.float64)
    y = GO.module_forward(params, query, kv, kv, "legendre-gauss", heads, 0.5)
    for s in (1, 3):
        yr = GO.module_forward(params, query.roll(s, -1), kv.roll(s, -1), kv.roll(s, -1), "legendre-gauss", heads, 0.5)
        assert torch.allclose(yr, y.roll(s, -1), rtol=1e-12, atol=1e-12)


def test_oracle_ignores_a_zero_weight_key():
    """a key with bias -inf drops out: the same result as without it, whatever its k and v, and no NaN"""
    q, k, v = _operands(1, 2, 12, 20, 8, 8)
    bias = GO.key_bias(4, 5, "legendre-gauss").clone()
    bias[7] = -np.inf
    k[..., 7, :] = 1e3
    v[..., 7] = np.nan
    v2 = v.clone()
    v2[..., 7] = 0.0   # the oracle's matmul would carry the NaN through 0 * NaN: compare on finite values
    o, lse = GO.attention(q, k, v2, bias, 1.0)
    keep = [j for j in range(20) if j != 7]
    o_ref, lse_ref = GO.attention(q, k[..., keep, :], v2[..., keep], bias[keep], 1.0)
    assert torch.isfinite(o).all() and torch.allclose(o, o_ref, rtol=1e-13) and torch.allclose(lse, lse_ref, rtol=1e-13)


def test_oracle_gradcheck():
    q, k, v = _operands(1, 1, 5, 6, 8, 8)
    bias = GO.key_bias(2, 3, "equiangular")
    for t in (q, k, v):
        t.requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b, c: GO.attention(a, b, c, bias, 0.3), (q, k, v))


def test_constructor_contract():
    m = A.AttentionS2(16, 2, (9, 18), (5, 10), grid_in="legendre-gauss", k_channels=32, out_channels=48)
    shapes = {n: tuple(p.shape) for n, p in m.named_parameters()}
    assert shapes == {"q_weights": (32, 16, 1, 1), "k_weights": (32, 16, 1, 1), "v_weights": (48, 16, 1, 1), "proj_weights": (48, 48, 1, 1),
                      "q_bias": (32,), "k_bias": (32,), "v_bias": (48,), "proj_bias": (48,)}
    assert set(m.state_dict()) == set(shapes)
    assert all(float(p.detach().abs().max()) == 0.0 for n, p in m.named_parameters() if n.endswith("_bias"))
    bound = np.sqrt(6.0 / (16 + 32))   # xavier-uniform of (32, 16, 1, 1)
    assert float(m.q_weights.abs().max()) <= bound and float(m.q_weights.std()) > 0.3 * bound
    assert m.scale == pytest.approx(1.0 / 4.0)   # 1 / sqrt(32 / 2)
    assert A.AttentionS2(16, 2, (9, 18), (9, 18), scale=0.25).scale == 0.25
    nb = A.AttentionS2(16, 2, (9, 18), (9, 18), bias=False)
    assert set(nb.state_dict()) == {"q_weights", "k_weights", "v_weights", "proj_weights"}
    w = 2 * np.pi * _grid_np(9, "legendre-gauss")[1] / 18
    assert torch.equal(m.key_bias, torch.from_numpy(np.repeat(np.log(w), 18).astype(np.float32)))


def test_constructor_refusals():
    for heads, ck, cv in [(2, 12, 16), (1, 136, 16), (2, 16, 20), (1, 4, 8)]:   # head dims 6, 136, 10, 4
        with pytest.raises(NotImplementedError, match="multiples of 8 up to 128"):
            A.AttentionS2(8, heads, (5, 10), (5, 10), k_channels=ck, out_channels=cv)
    with pytest.raises(ValueError, match="divisible by num_heads"):
        A.AttentionS2(8, 3, (5, 10), (5, 10), k_channels=32)
    A.AttentionS2(8, 1, (5, 10), (5, 10), k_channels=128, out_channels=8)   # the largest and smallest head dims are served
    with pytest.raises(ValueError):
        A.AttentionS2(8, 1, (5, 10), (5, 10), grid_in="healpix")


def test_forward_refusals_before_any_kernel():
    m = A.AttentionS2(8, 1, (6, 12), (4, 8))
    with pytest.raises(ValueError, match="in_shape == out_shape"):
        m(torch.zeros(1, 8, 4, 8))
    m.eval()
    with pytest.raises(B200ShtError, match="CUDA"):
        m(torch.zeros(1, 8, 4, 8), torch.zeros(1, 8, 6, 12), torch.zeros(1, 8, 6, 12))
    d = A.AttentionS2(8, 1, (4, 8), (4, 8), drop_rate=0.1)
    assert d.drop_rate == 0.1
    with pytest.raises(NotImplementedError, match="dropout"):
        d(torch.zeros(1, 8, 4, 8))
    d.eval()   # in evaluation nothing drops: the module goes on to its device check
    with pytest.raises(B200ShtError, match="CUDA"):
        d(torch.zeros(1, 8, 4, 8))


def test_shim_name_resolves():
    import makani_b200 as mb
    import makani_b200.compat as compat

    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        th = compat.install_torch_harmonics_shim()
        assert th.AttentionS2 is mb.AttentionS2 is A.AttentionS2
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_product_path_does_not_import_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "makani_b200")):
        for f in files:
            if f.endswith(".py"):
                assert "attention_global_oracle" not in open(os.path.join(dirpath, f)).read(), f


def test_c_abi_symbols():
    names = ["b200sht_attention_global_workspace_floats", "b200sht_attention_global_forward", "b200sht_attention_global_backward"]
    header = open(os.path.join(ROOT, "include", "b200sht.h")).read()
    for n in names:
        assert re.search(r"\b" + n + r"\(", header), n
        assert n in _lib._SIGNATURES
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libb200sht.so is not built")
    lib = _lib.load()
    for n in names:
        assert hasattr(lib, n)
    # the workspace query refuses what the kernels do not serve, and needs no device
    assert lib.b200sht_attention_global_workspace_floats(2, 100, 100, 12, 16, _lib.PREC_TF32, 0) == -1
    assert lib.b200sht_attention_global_workspace_floats(2, 100, 100, 16, 136, _lib.PREC_TF32, 0) == -1
    assert lib.b200sht_attention_global_workspace_floats(2, 100, 100, 16, 16, _lib.PREC_FP32, 0) == -1
    fwd = lib.b200sht_attention_global_workspace_floats(2, 100, 100, 16, 16, _lib.PREC_TF32, 0)
    assert fwd >= 3 * 2 * 100 * 16 and lib.b200sht_attention_global_workspace_floats(2, 100, 100, 16, 16, _lib.PREC_FP32X3, 0) >= 2 * fwd - 64 * 6


@pytest.fixture(scope="module")
def compiled():
    """(SASS dump, ptxas report) of attention_global.cu"""
    if not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)):
        pytest.skip("nvcc / cuobjdump are not available")
    csrc = os.path.join(ROOT, "makani_b200", "csrc")
    obj = os.path.join(ROOT, "makani_b200", "build", "attention_global.o")
    sources = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh"))]
    newest = max(os.path.getmtime(s) for s in sources)
    if os.path.exists(obj) and os.path.exists(obj + ".log") and min(os.path.getmtime(obj), os.path.getmtime(obj + ".log")) >= newest:
        report = open(obj + ".log").read()
        sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
        return sass, report
    from makani_b200 import build as _build

    with tempfile.TemporaryDirectory() as tmp:
        o = os.path.join(tmp, "attention_global.o")
        r = subprocess.run([NVCC] + _build.FLAGS + ["-c", os.path.join(csrc, "attention_global.cu"), "-o", o], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        sass = subprocess.run([CUOBJDUMP, "-sass", o], capture_output=True, text=True, check=True).stdout
    return sass, r.stdout + r.stderr


def test_kernels_do_not_spill(compiled):
    _, report = compiled
    pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?Function properties for \1\n\s+(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    kernels = {m.group(1): (int(m.group(3)), int(m.group(4))) for m in pat.finditer(report) if "attention_global" in m.group(1)}
    # 3 kernels x 4 head-dim chunk counts x {TF32, 3 x TF32}, the two prep instantiations and the row dot
    assert sum("attention_global_kernel" in k for k in kernels) == 24 and len(kernels) == 27, kernels
    spilling = {k: v for k, v in kernels.items() if v[0] or v[1]}
    assert not spilling, spilling
    assert "C7510" not in report   # ptxas did not serialize any wgmma


def test_every_instantiation_runs_on_wgmma(compiled):
    sass, _ = compiled
    counts, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if "attention_global_kernel" in m.group(1) else None
            if cur:
                counts[cur] = [0, 0]
        elif cur and "HGMMA." in line:
            counts[cur][0] += 1
        elif cur and "HMMA." in line:
            counts[cur][1] += 1
    assert len(counts) == 24, counts
    for name, (hgmma, hmma) in counts.items():
        kind, dc, split = re.search(r"attention_global_kernelILi(\d)ELi(\d)ELb(\d)E", name).groups()
        kind, dc, split = int(kind), int(dc), int(split)
        # k8 steps per streamed block: forward S (4 dc) + PV (4); dK / dV two S-type (8 dc) + two PV-type (8); dQ 8 dc + 4
        per_block = {0: 4 * dc + 4, 1: 8 * dc + 8, 2: 8 * dc + 4}[kind]
        assert hgmma == per_block * (3 if split else 1) and hmma == 0, (name, hgmma, hmma)

"""Bilinear resampling on the CPU: the product's table builder (makani_b200/resample.py) against the independent oracle
(oracle/makani_resample_oracle.py), and the identities that pin the restated contract without torch-harmonics: coincident nodes, constants,
fields linear in the colatitude, pole rows.  Plus the module's constructor contract and refusals, the shim names and the build log of the two
kernels (no register spills).  Needs neither a GPU nor torch-harmonics."""
import importlib
import os
import re
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from makani_b200 import resample as R  # noqa: E402
from makani_b200._lib import B200ShtError  # noqa: E402
from makani_b200.quadrature import precompute_latitudes, precompute_longitudes  # noqa: E402
from oracle import makani_resample_oracle as O  # noqa: E402

# (nlat_in, nlon_in, nlat_out, nlon_out, grid_in, grid_out): FCN3's decoder scaled (poles expanded), eq -> eq upsampling by 2, downsampling,
# and an odd nlon (rows not 16-byte aligned)
PAIRS = [
    (24, 48, 49, 96, "legendre-gauss", "equiangular"),
    (25, 48, 49, 96, "equiangular", "equiangular"),
    (49, 96, 24, 48, "equiangular", "legendre-gauss"),
    (17, 35, 33, 70, "equiangular", "equiangular"),
]
IDS = ["lg24x48-eq49x96", "eq25x48-eq49x96", "eq49x96-lg24x48", "eq17x35-eq33x70"]


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_tables_match_oracle_exactly(pair):
    t, o = R.precompute_tables(*pair), O.tables(*pair)
    for name in ("lat_idx", "lat_w", "lon_left", "lon_right", "lon_w"):
        a, b = getattr(t, name), o[name].numpy()
        assert a.dtype == b.dtype and np.array_equal(a, b), name
    assert t.expand_poles == o["expand_poles"]


def test_expand_poles_only_where_output_leaves_the_input_band():
    assert [R.precompute_tables(*p).expand_poles for p in PAIRS] == [True, False, False, False]


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_weights_and_indices_in_range(pair):
    t = R.precompute_tables(*pair)
    nexp = pair[0] + 2 * t.expand_poles
    assert t.lat_w.dtype == np.float32 and t.lon_w.dtype == np.float32
    assert (t.lat_w >= 0).all() and (t.lat_w <= 1).all() and (t.lon_w >= 0).all() and (t.lon_w <= 1).all()
    assert (t.lat_idx >= 0).all() and (t.lat_idx + 1 < nexp).all()
    for idx in (t.lon_left, t.lon_right):
        assert (idx >= 0).all() and (idx < pair[1]).all()
    assert (t.lon_right == (t.lon_left + 1) % pair[1]).all()


def _field(pair, seed=0):
    return torch.randn(2, 3, pair[0], pair[1], dtype=torch.float64, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_coincident_nodes_reproduce_the_input(pair):
    nlat_in, nlon_in, nlat_out, nlon_out, gi, go = pair
    th_in, th_out = precompute_latitudes(nlat_in, gi)[0].numpy(), precompute_latitudes(nlat_out, go)[0].numpy()
    ph_in, ph_out = precompute_longitudes(nlon_in).numpy(), precompute_longitudes(nlon_out).numpy()
    rows = [(t, int(np.nonzero(th_in == v)[0][0])) for t, v in enumerate(th_out) if v in th_in]
    cols = [(p, int(np.nonzero(ph_in == v)[0][0])) for p, v in enumerate(ph_out) if v in ph_in]
    x = _field(pair)
    y = O.ResampleS2(*pair)(x)
    if pair[4] == pair[5]:                                             # eq -> eq: every other node coincides
        assert len(rows) >= min(nlat_in, nlat_out) and len(cols) >= min(nlon_in, nlon_out) // 2
    for t, i in rows:
        for p, j in cols:
            assert torch.equal(y[..., t, p], x[..., i, j]), (t, p)


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_constants_are_preserved(pair):
    x = torch.full((2, pair[0], pair[1]), 0.3125, dtype=torch.float64)
    y = O.ResampleS2(*pair)(x)
    assert y.shape == (2, pair[2], pair[3]) and torch.equal(y, torch.full_like(y, 0.3125))


@pytest.mark.parametrize("pair", PAIRS, ids=IDS)
def test_linear_in_colatitude_is_reproduced_at_interior_rows(pair):
    nlat_in, nlon_in, nlat_out, nlon_out, gi, go = pair
    th_in, th_out = precompute_latitudes(nlat_in, gi)[0], precompute_latitudes(nlat_out, go)[0]
    x = (0.7 * th_in - 0.2)[:, None].expand(nlat_in, nlon_in)
    y = O.ResampleS2(*pair)(x)
    t = R.precompute_tables(*pair)
    off = 1 if t.expand_poles else 0
    interior = (t.lat_idx - off >= 0) & (t.lat_idx + 1 - off <= nlat_in - 1)      # both rows are input rows
    assert interior.sum() >= nlat_out - 4
    ref = (0.7 * th_out - 0.2)[:, None].expand(nlat_out, nlon_out)
    # the weights are fp32: the error is at most 0.7 * (row spacing) * 2^-24
    assert torch.allclose(y[interior], ref[interior], rtol=0, atol=0.7 * np.pi / (nlat_in - 1) * 2.0**-23)


def test_pole_rows_are_the_longitude_means():
    pair = PAIRS[0]
    x = _field(pair, 1)
    y = O.ResampleS2(*pair)(x)
    # equiangular output rows 0 and -1 sit on the poles
    assert torch.allclose(y[..., 0, :], x[..., 0, :].mean(-1, keepdim=True).expand_as(y[..., 0, :]), rtol=0, atol=1e-15)
    assert torch.allclose(y[..., -1, :], x[..., -1, :].mean(-1, keepdim=True).expand_as(y[..., -1, :]), rtol=0, atol=1e-15)


def test_constructor_contract_and_refusals():
    res = R.ResampleS2(24, 48, 49, 96, grid_in="legendre-gauss", grid_out="equiangular")
    assert (res.nlat_in, res.nlon_in, res.nlat_out, res.nlon_out) == (24, 48, 49, 96)
    assert (res.grid_in, res.grid_out, res.mode) == ("legendre-gauss", "equiangular", "bilinear")
    assert res.expand_poles and not res.skip_resampling
    assert res.state_dict() == {} and len(list(res.parameters())) == 0
    assert {n for n, _ in res.named_buffers()} == {"lat_idx", "lat_weights", "lon_idx_left", "lon_idx_right", "lon_weights"}
    res.load_state_dict({})
    for mode in ("bilinear-spherical", "nearest"):
        with pytest.raises(NotImplementedError, match=mode):
            R.ResampleS2(24, 48, 49, 96, mode=mode)
    with pytest.raises(B200ShtError):
        res(torch.randn(2, 24, 48))                                     # CPU tensor
    with pytest.raises(B200ShtError):
        res(torch.randn(2, 24, 48, dtype=torch.float64))                # not fp32
    with pytest.raises(B200ShtError):
        res(torch.randn(2, 24, 48, dtype=torch.bfloat16))
    with pytest.raises(ValueError):
        res(torch.randn(2, 24, 47))
    with pytest.raises(ValueError):
        res(torch.randn(48))
    # equal shapes and grids: forward returns its input (no device needed)
    same = R.ResampleS2(24, 48, 24, 48, grid_in="legendre-gauss", grid_out="legendre-gauss")
    x = torch.randn(3, 24, 48)
    assert same.skip_resampling and same(x) is x
    assert not R.ResampleS2(24, 48, 24, 48, grid_in="legendre-gauss", grid_out="equiangular").skip_resampling


def test_shim_names_resolve():
    import makani_b200.compat as compat

    saved = {k: v for k, v in sys.modules.items() if k == "torch_harmonics" or k.startswith("torch_harmonics.")}
    try:
        for k in saved:
            del sys.modules[k]
        th = compat.install_torch_harmonics_shim()
        assert th.ResampleS2 is R.ResampleS2
        thd = importlib.import_module("torch_harmonics.distributed")
        with pytest.raises(NotImplementedError, match="distributed resampling"):
            thd.DistributedResampleS2(24, 48, 49, 96, grid_in="legendre-gauss", grid_out="equiangular", mode="bilinear")
    finally:
        for k in [k for k in sys.modules if k == "torch_harmonics" or k.startswith("torch_harmonics.")]:
            del sys.modules[k]
        sys.modules.update(saved)


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc is not available")
def test_resample_kernels_do_not_spill():
    csrc = os.path.join(ROOT, "makani_b200", "csrc")
    log = os.path.join(ROOT, "makani_b200", "build", "resample.o.log")
    sources = [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cu", ".cuh"))]
    if os.path.exists(log) and os.path.getmtime(log) >= max(os.path.getmtime(s) for s in sources):
        report = open(log).read()
    else:
        from makani_b200 import build as _build

        nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
        with tempfile.TemporaryDirectory() as tmp:
            r = subprocess.run([nvcc] + _build.FLAGS + ["-c", os.path.join(csrc, "resample.cu"), "-o", os.path.join(tmp, "resample.o")],
                               capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-2000:]
        report = r.stdout + r.stderr
    pat = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'\n.*?Function properties for \1\n\s+(\d+) bytes stack frame, "
                     r"(\d+) bytes spill stores, (\d+) bytes spill loads")
    kernels = {m.group(1): (int(m.group(3)), int(m.group(4))) for m in pat.finditer(report) if "resample_" in m.group(1)}
    assert sum("resample_forward_kernel" in k for k in kernels) == 1 and sum("resample_adjoint_kernel" in k for k in kernels) == 1, kernels
    spilling = {k: v for k, v in kernels.items() if v[0] or v[1]}
    assert not spilling, spilling

"""makani_b200.noise against makani's own noise classes (tests/golden/noise_golden.npz, tests/golden/make_noise_golden.py), without a GPU:
buffers and parameters bit for bit, shapes, model-parallel tags, state-dict keys, extra_repr, the errors, build_noise's dispatch, the generator
state round trip, batch resizing and DummyNoiseS2 (which runs no kernel) against the golden draws; update() and forward() of a CPU state raise."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import makani_b200 as mb
from makani_b200 import noise as mn

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, "golden", "noise_golden.npz"))
CASES = sorted({k.split("/")[0] for k in GOLD.files})


def meta(case):
    return json.loads(str(GOLD[f"{case}/meta"]))


def build(case):
    m = meta(case)
    kw = dict(m["kwargs"])
    kw["img_shape"] = tuple(kw["img_shape"])
    if m["how"] == "build_noise":
        return mn.build_noise(**kw)
    return getattr(mn, m["how"])(**kw)


def test_golden_covers_the_cases():
    kinds = {meta(c)["cls"] for c in CASES}
    assert kinds == {"DiffusionNoiseS2", "IsotropicGaussianRandomFieldS2", "DummyNoiseS2"}
    assert any(meta(c)["kwargs"].get("num_time_steps", 1) > 1 and meta(c)["cls"] == "DiffusionNoiseS2" for c in CASES)
    assert any(meta(c)["learnable"] and meta(c)["cls"] == "IsotropicGaussianRandomFieldS2" for c in CASES)


@pytest.mark.parametrize("case", CASES)
def test_structure_matches_makani(case):
    """class, attributes, state-dict keys, parameter tags, extra_repr, is_stateful, and every buffer / parameter bit for bit"""
    ref = meta(case)
    m = build(case)
    assert type(m).__name__ == ref["cls"]
    for a, v in ref["attrs"].items():
        assert getattr(m, a) == v, (case, a, getattr(m, a), v)
    assert getattr(m, "learnable", None) == ref["learnable"]
    assert list(m.state_dict().keys()) == ref["state_dict_keys"]
    tags = {k: [getattr(p, "is_shared_mp", None), getattr(p, "sharded_dims_mp", None)] for k, p in m.named_parameters()}
    assert tags == ref["tags"]
    assert m.extra_repr() == ref["extra_repr"]
    assert m.is_stateful() == ref["is_stateful"]
    assert sorted(k for k, _ in m.named_buffers() if k != "state") == ref["buffers"]
    assert sorted(k for k, _ in m.named_parameters()) == ref["parameters"]
    for k, v in list(m.named_buffers()) + list(m.named_parameters()):
        if k == "state":
            continue
        want = torch.from_numpy(GOLD[f"{case}/t/{k}"])
        assert v.dtype == want.dtype and v.shape == want.shape and torch.equal(v.detach(), want), (case, k)
    assert m.state.device.type == "cpu" and m.state.dtype == torch.float32
    assert tuple(m.state.shape) == GOLD[f"{case}/state0"].shape


@pytest.mark.parametrize("case", [c for c in CASES if meta(c)["cls"] != "DummyNoiseS2"])
def test_cpu_update_and_forward_raise(case):
    m = build(case)
    m.set_tensor_state(torch.from_numpy(GOLD[f"{case}/state0"]))
    rng = m.rng_cpu.get_state()
    for call in (lambda: m.update(), lambda: m.update(replace_state=True), lambda: m()):
        with pytest.raises(mb.B200ShtError, match="no CPU fallback"):
            call()
    assert torch.equal(m.rng_cpu.get_state(), rng), "a refused update must not consume draws"
    assert torch.equal(m.state, torch.from_numpy(GOLD[f"{case}/state0"]))


@pytest.mark.parametrize("case", ["dummy_zero", "dummy_random"])
def test_dummy_matches_makani(case):
    """DummyNoiseS2 on the CPU: forward returns the live state; constant_random draws makani's values from rng_cpu"""
    m = build(case)
    s0 = torch.from_numpy(GOLD[f"{case}/state0"])
    m.set_tensor_state(s0)
    y = m()
    assert y is m.state and torch.equal(y, torch.from_numpy(GOLD[f"{case}/y"]))
    m.update()
    if case == "dummy_random":
        assert torch.equal(m.state, torch.from_numpy(GOLD[f"{case}/upd/random/after"]))
    else:
        assert bool((m.state == 0).all())
    assert not m.is_stateful()


def test_errors():
    kw = dict(img_shape=(17, 32), batch_size=1, num_channels=2)
    with pytest.raises(ValueError, match="kT as a list needs one number per channel"):
        mn.DiffusionNoiseS2(**kw, kT=[1e-3, 1e-3, 1e-3])
    with pytest.raises(ValueError, match="kT as a list needs one number per channel"):
        mn.DiffusionNoiseS2(**kw, kT=[[1e-3], [1e-3]])
    with pytest.raises(ValueError, match="lambd as a list needs one number per channel"):
        mn.DiffusionNoiseS2(**kw, lambd=[1.0])
    with pytest.raises(ValueError, match="lambd as a list needs one number per channel"):
        mn.DiffusionNoiseS2(**kw, lambd=[[1.0], [1.0]])
    with pytest.raises(NotImplementedError, match="learnable"):
        mn.DiffusionNoiseS2(**kw, num_time_steps=2, learnable=True)
    with pytest.raises(ValueError, match="mode must be one of"):
        mn.DummyNoiseS2(**kw, mode="invalid_mode")
    with pytest.raises(NotImplementedError):
        mn.BaseNoiseS2(**kw, num_time_steps=1).is_stateful()
    n = mn.DiffusionNoiseS2(**kw)
    bad = torch.zeros(1, 1, 3, n.lmax_local, n.mmax_local, 2)
    with pytest.raises(ValueError, match="holds states of shape"):
        n.set_tensor_state(bad)
    assert tuple(n.state.shape) == (1, 1, 2, 17, 17, 2)
    b = dict(img_shape=(17, 32), batch_size=1, num_channels=1, num_time_steps=1, grid_type="equiangular", seed=1, reflect=False)
    with pytest.raises(ValueError, match="has no 'type'"):
        mn.build_noise({}, **b)
    with pytest.raises(NotImplementedError, match="not supported"):
        mn.build_noise({"type": "pink"}, **b)


@pytest.mark.parametrize("cast", ["double", "half", "bfloat16"])
@pytest.mark.parametrize("case", [c for c in CASES if meta(c)["cls"] != "DummyNoiseS2"])
def test_non_fp32_modules_raise_before_drawing(case, cast):
    """the kernels read and write the state, sigma_l, phi and discount as fp32: after a dtype cast of the module, update() and forward()
    raise B200ShtError (naming the dtype) before anything is drawn or written, on any device"""
    m = getattr(build(case), cast)()
    assert m.state.dtype != torch.float32
    rng, state = m.rng_cpu.get_state(), m.get_tensor_state()
    for call in (lambda: m.update(), lambda: m.update(replace_state=True), lambda: m()):
        with pytest.raises(mb.B200ShtError, match="float32 only"):
            call()
    assert torch.equal(m.rng_cpu.get_state(), rng) and torch.equal(m.state, state)


def test_non_fp32_parameters_raise():
    """a float32 state with a cast sigma_l / phi is refused as well"""
    n = mn.DiffusionNoiseS2((17, 32), 1, 2)
    n.phi = n.phi.double()
    with pytest.raises(mb.B200ShtError, match="phi is torch.float64"):
        n.update()
    g = mn.IsotropicGaussianRandomFieldS2((17, 32), 1, 2)
    g.sigma_l = g.sigma_l.half()
    with pytest.raises(mb.B200ShtError, match="sigma_l is torch.float16"):
        g()


def test_build_noise_dispatch_and_defaults():
    b = dict(img_shape=(17, 32), batch_size=1, num_channels=2, num_time_steps=1, grid_type="equiangular", seed=5, reflect=True)
    d = mn.build_noise({"type": "diffusion"}, **b, default_lambd=0.25)
    assert isinstance(d, mn.DiffusionNoiseS2) and d.kT == 0.5 * (100 / 6370) ** 2 and d.lambd == 0.25 and d.reflect and not d.learnable
    assert mn.DiffusionNoiseS2((17, 32), 1, 2).kT == 0.5 * (500.0 / 6370.0) ** 2   # the class's default differs from the factory's
    w = mn.build_noise({"type": "white", "alpha": 2.0, "learnable": True, "lmax": 8}, **b)
    assert isinstance(w, mn.IsotropicGaussianRandomFieldS2) and w.alpha == 2.0 and w.learnable and w.lmax == 8 and w.mmax == 8
    assert isinstance(w.sigma_l, torch.nn.Parameter)
    z = mn.build_noise({"type": "dummy", "mode": "constant_random"}, **b)
    assert isinstance(z, mn.DummyNoiseS2) and z.mode == "constant_zero"   # makani's factory passes no mode


def test_rng_state_round_trip_and_batch_resizing():
    m = mn.DummyNoiseS2((17, 32), 2, 3, mode="constant_random", seed=7)
    cpu, gpu = m.get_rng_state()
    assert gpu is None or isinstance(gpu, torch.Tensor)
    m.update()
    first = m.get_tensor_state()
    m.set_rng_state(cpu, None)
    m.update()
    assert torch.equal(m.state, first)
    m.update(batch_size=5)
    assert m.state.shape[0] == 5 and "state" in dict(m.named_buffers())
    m.set_tensor_state(torch.ones(1, 1, 3, 17, 32))
    assert m.state.shape[0] == 1 and bool((m.state == 1).all())
    m.reset(batch_size=4)
    assert m.state.shape[0] == 4 and bool((m.state == 0).all())
    ptr = m.state.data_ptr()
    m._ensure_state(4)
    assert m.state.data_ptr() == ptr
    n = mn.IsotropicGaussianRandomFieldS2((17, 32), 2, 3)
    n.reset(batch_size=3)
    assert tuple(n.state.shape) == (3, 1, 3, 17, 17, 2) and "state" not in n.state_dict()


def test_import_needs_neither_makani_nor_torch_harmonics():
    code = ("import sys, makani_b200.noise as n; m = n.DiffusionNoiseS2((721, 1440), 1, 8, kT=[1e-3] * 8, lambd=1.0, seed=333);"
            "assert tuple(m.state.shape) == (1, 1, 8, 721, 721, 2);"
            "bad = [k for k in sys.modules if k.split('.')[0] in ('makani', 'torch_harmonics')]; assert not bad, bad")
    r = subprocess.run([sys.executable, "-c", code], cwd=os.path.dirname(HERE), capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

#!/usr/bin/env python
"""Golden vectors for the spherical noise restatement (makani_b200/noise.py), produced by the REFERENCE's own classes:
makani/models/noise.py (IsotropicGaussianRandomFieldS2, DiffusionNoiseS2, DummyNoiseS2, build_noise; unmodified) on the CPU, with the oracle's
InverseRealSHT (oracle/makani_oracle.py) posed as torch_harmonics, in the environment of make_fcn3_golden.py.  Geometries 17 x 32 equiangular and
16 x 32 Legendre-Gauss, at the default and a truncated lmax.

Stored per case:
    <case>/meta          JSON: class, constructor arguments, attributes, state-dict keys, parameter tags, extra_repr, is_stateful
    <case>/t/<name>      every buffer and parameter but the state and the transform's own
    <case>/state0        a seeded state, set with set_tensor_state
    <case>/y             forward() of that state (the fields, or for DummyNoiseS2 the state it returns)
    <case>/g, <case>/dsigma   learnable isotropic field: a fixed cotangent of y and the gradient of sigma_l it gives
    <case>/upd/<mode>/xi, <case>/upd/<mode>/after   for each update mode, from state0: the standard normals replayed from rng_cpu and the state after
        (mode "ar": update(); "stationary": update(replace_state=True); "base": the memoryless update of the isotropic field)

    python tests/golden/make_noise_golden.py        # needs a makani checkout -> tests/golden/noise_golden.npz
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "reference_suites"))

# config/fourcastnet3.yaml input_noise: 8 diffusion channels of these spatial correlation lengths
SHIPPED_KT = [3.0806e-5, 1.2322e-4, 4.9289e-4, 1.9716e-3, 7.8862e-3, 3.1545e-2, 1.2618e-1, 5.0472e-1]
EA = dict(img_shape=(17, 32), grid_type="equiangular")
LG = dict(img_shape=(16, 32), grid_type="legendre-gauss")

# name -> (class or "build_noise", constructor arguments)
NOISE_GOLDEN_CASES = {
    "diffusion_shipped": ("DiffusionNoiseS2", dict(EA, batch_size=2, num_channels=8, num_time_steps=1, sigma=1.0, kT=SHIPPED_KT, lambd=1.0, seed=333)),
    "diffusion_shipped_lg_lmax10": ("DiffusionNoiseS2", dict(LG, batch_size=1, num_channels=8, num_time_steps=1, sigma=1.0, kT=SHIPPED_KT, lambd=1.0,
                                                             lmax=10, seed=334)),
    "diffusion_t3": ("DiffusionNoiseS2", dict(EA, batch_size=2, num_channels=2, num_time_steps=3, sigma=0.8, kT=0.01, lambd=0.5, lmax=12, seed=335)),
    "diffusion_reflect_lambd": ("DiffusionNoiseS2", dict(LG, batch_size=1, num_channels=3, num_time_steps=1, kT=[1e-3, 1e-2, 1e-1],
                                                         lambd=[0.25, 1.0, 2.0], reflect=True, seed=336)),
    "diffusion_t2_lambd_lmax9": ("DiffusionNoiseS2", dict(EA, batch_size=1, num_channels=3, num_time_steps=2, kT=[1e-3, 1e-2, 1e-1],
                                                          lambd=[0.25, 1.0, 2.0], lmax=9, reflect=True, seed=337)),
    "diffusion_learnable": ("DiffusionNoiseS2", dict(EA, batch_size=1, num_channels=2, num_time_steps=1, kT=0.02, lambd=0.7, learnable=True,
                                                     seed=338)),
    "diffusion_build": ("build_noise", dict(noise_params={"type": "diffusion", "lmax": 10}, img_shape=(17, 32), batch_size=1, num_channels=2,
                                            num_time_steps=1, grid_type="equiangular", seed=339, reflect=False, default_lambd=0.5)),
    "grf_alpha0": ("IsotropicGaussianRandomFieldS2", dict(EA, batch_size=2, num_channels=3, num_time_steps=1, sigma=1.0, alpha=0.0, seed=340)),
    "grf_alpha2_lmax12": ("IsotropicGaussianRandomFieldS2", dict(EA, batch_size=1, num_channels=2, num_time_steps=1, sigma=1.5, alpha=2.0, lmax=12,
                                                                 seed=341)),
    "grf_alpha2_learnable_lg": ("IsotropicGaussianRandomFieldS2", dict(LG, batch_size=2, num_channels=2, num_time_steps=2, sigma=0.7, alpha=2,
                                                                       lmax=10, reflect=True, learnable=True, seed=342)),
    "grf_build": ("build_noise", dict(noise_params={"type": "white", "alpha": 1.0, "sigma": 2.0}, img_shape=(16, 32), batch_size=1, num_channels=1,
                                      num_time_steps=1, grid_type="legendre-gauss", seed=343, reflect=True)),
    "dummy_zero": ("DummyNoiseS2", dict(img_shape=(17, 32), batch_size=2, num_channels=3, num_time_steps=1, seed=344)),
    "dummy_random": ("DummyNoiseS2", dict(img_shape=(17, 32), batch_size=1, num_channels=2, num_time_steps=2, mode="constant_random", seed=345)),
}
ATTRS = ["nlat", "nlon", "lmax", "mmax", "lmax_local", "mmax_local", "nlat_local", "nlon_local", "num_channels", "num_time_steps", "reflect"]


def reference_module():
    """makani's noise module on the oracle's InverseRealSHT posed as torch_harmonics"""
    import importlib

    import run_reference_tests as base

    base.install_environment()
    comm = sys.modules["makani.utils.comm"]
    if not hasattr(comm, "get_local_rank"):
        comm.get_local_rank = lambda: 0
    return importlib.import_module("makani.models.noise")


def update_modes(kind):
    if kind.startswith("diffusion"):
        return {"ar": False, "stationary": True}
    if kind.startswith("grf"):
        return {"base": False}
    return {"random": False} if kind == "dummy_random" else {}


def main():
    N = reference_module()
    out = {}
    for name, (cls, kw) in NOISE_GOLDEN_CASES.items():
        m = N.build_noise(**kw) if cls == "build_noise" else getattr(N, cls)(**kw)
        tags = {k: [getattr(p, "is_shared_mp", None), getattr(p, "sharded_dims_mp", None)] for k, p in m.named_parameters()}
        meta = dict(cls=type(m).__name__, how=cls, kwargs=kw, attrs={a: getattr(m, a) for a in ATTRS}, learnable=getattr(m, "learnable", None),
                    state_dict_keys=list(m.state_dict().keys()), tags=tags, extra_repr=m.extra_repr(), is_stateful=m.is_stateful(),
                    buffers=sorted(k for k, _ in m.named_buffers() if k != "state" and not k.startswith("isht.")),
                    parameters=sorted(k for k, _ in m.named_parameters()))
        out[f"{name}/meta"] = np.array(json.dumps(meta, sort_keys=True))
        for k, v in list(m.named_buffers()) + list(m.named_parameters()):
            if k != "state" and not k.startswith("isht."):
                out[f"{name}/t/{k}"] = v.detach().numpy()
        gen = torch.Generator().manual_seed(1000 + len(out))
        state0 = torch.randn(m.state.shape, generator=gen)
        m.set_tensor_state(state0)
        y = m()
        out[f"{name}/state0"], out[f"{name}/y"] = state0.numpy(), y.detach().numpy().copy()
        if getattr(m, "learnable", False) and cls != "DiffusionNoiseS2" and name.startswith("grf"):
            g = torch.randn(y.shape, generator=gen)
            (y * g).sum().backward()
            out[f"{name}/g"], out[f"{name}/dsigma"] = g.numpy(), m.sigma_l.grad.numpy()
        for mode, replace in update_modes(name).items():
            m.set_tensor_state(state0)
            rng = m.rng_cpu.get_state()
            m.update(replace_state=replace)
            replay = torch.Generator()
            replay.set_state(rng)
            shape = state0.shape if (replace or not name.startswith("diffusion")) else (state0.shape[0], 1, *state0.shape[2:])
            out[f"{name}/upd/{mode}/xi"] = torch.empty(shape).normal_(mean=0.0, std=1.0, generator=replay).numpy()
            out[f"{name}/upd/{mode}/after"] = m.get_tensor_state().numpy()
        print(name, meta["cls"], "state", tuple(state0.shape), "y", tuple(y.shape), "updates", list(update_modes(name)))
    path = os.path.join(HERE, "noise_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

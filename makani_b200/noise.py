"""Random fields on the sphere on the CUDA kernels of this package: makani's spherical noise without a makani checkout.

The module family of makani/models/noise.py (BaseNoiseS2, IsotropicGaussianRandomFieldS2, DiffusionNoiseS2, DummyNoiseS2, build_noise) with
the same constructor arguments and defaults, attributes, buffers and parameters (which of them are persistent, their values, the model-parallel tags),
methods and error types.  FourCastNet 3's shipped input noise (`input_noise: {type: diffusion, n_channels: 8, ...}`) is a DiffusionNoiseS2.

The state keeps makani's layout, fp32 (B, T, C, L_loc, M_loc, 2), allocated on the CPU at construction, so get_tensor_state /
set_tensor_state and checkpoints carry it unchanged.  The standard normal draws are `normal_(generator=self.rng_gpu)` with makani's shapes and
in makani's order, so a seed (or a makani checkpoint's get_rng_state()) gives makani's noise; everything after the draw runs in csrc/noise.cu:

    update   b200sht_noise_update: the AR step, the stationary redraw (replace_state=True) or the memoryless update, in place
    forward  b200sht_noise_spectrum -> InverseRealSHT.forward_packed (one pass from the state to the packed synthesis input), fp32 out
    learnable isotropic sigma: its gradient is b200sht_noise_sigma_grad of the packed gradient the synthesis backward returns

The kernels take fp32 CUDA tensors only: update() and forward() raise B200ShtError, before anything is drawn, when the state or the sigma_l /
phi / discount they pass is on the CPU or not float32 (after `.double()` or `.half()` of the module, say; makani_b200 has no CPU or
other-precision fallback).  DummyNoiseS2 runs no kernel and works on any device and dtype.  A learnable diffusion sigma / phi gets no
gradient, as in makani, which only reads them under no_grad.

h x w: when makani_b200.distributed is initialised with more than one rank in the polar x azimuth grid, the synthesis is a
DistributedInverseRealSHT and sigma is split as makani splits it (isotropic field: l over h, m over w; diffusion: l over h).
"""
import math

import numpy as np
import torch
import torch.nn as nn
from torch import amp

from . import _lib
from ._lib import B200ShtError, launch_stream as _stream, ptr as _ptr
from .sht import InverseRealSHT


def _grid():
    """(h, w, rank_h, rank_w) of makani_b200.distributed, or None when it is not initialised or has a single rank"""
    from . import distributed as mbd

    if not mbd.is_initialized():
        return None
    h, w = mbd.polar_group_size(), mbd.azimuth_group_size()
    if h * w == 1:
        return None
    return h, w, mbd.polar_group_rank(), mbd.azimuth_group_rank()


def _check_operands(what, **tensors):
    """B200ShtError unless every given tensor is a float32 CUDA tensor: the kernels read and write them as float / float2 device memory"""
    given = [(name, t) for name, t in tensors.items() if t is not None]
    for name, t in given:
        if t.dtype != torch.float32:
            raise B200ShtError(f"{what}: {name} is {t.dtype}; the noise kernels take float32 only (no fallback for other dtypes)")
    for name, t in given:
        if not t.is_cuda:
            raise B200ShtError(f"{what} runs on CUDA devices only ({name} on {t.device}); makani_b200 has no CPU fallback")


class _NoiseSpectrum(torch.autograd.Function):
    """state -> what the synthesis reads (b200sht_noise_spectrum): the packed spec (packed) or complex (B, TC, L, M) coefficients.
    sigma: the isotropic field's (1, 1, 1, L, M) sigma_l, or None (the state as it is).  Backward: the gradient of sigma."""

    @staticmethod
    def forward(ctx, state, sigma, packed):
        B, T, C, L, M, _ = state.shape
        TC = T * C
        if packed:
            out = torch.empty(int(_lib.load().b200sht_spec_elems_lm(L, M, B, TC)), dtype=torch.float32, device=state.device)
        else:
            out = torch.empty((B, TC, L, M), dtype=torch.complex64, device=state.device)
        sig = sigma.detach().contiguous() if sigma is not None else None
        _lib.call("b200sht_noise_spectrum", _ptr(state), _ptr(sig), _ptr(out), B, TC, L, M, int(packed), _stream(state.device))
        ctx.packed, ctx.dims = packed, (B, TC, L, M)
        if ctx.needs_input_grad[1]:
            ctx.save_for_backward(state.clone())   # the state is updated in place after forward(update_internal_state=True)
        return out

    @staticmethod
    def backward(ctx, g):
        if not ctx.needs_input_grad[1]:
            return None, None, None
        (state,) = ctx.saved_tensors
        B, TC, L, M = ctx.dims
        g = g.contiguous()
        gf = g if ctx.packed else torch.view_as_real(g)
        dsigma = torch.empty((1, 1, 1, L, M), dtype=torch.float32, device=state.device)
        _lib.call("b200sht_noise_sigma_grad", _ptr(state), _ptr(gf), _ptr(dsigma), B, TC, L, M, int(ctx.packed), _stream(state.device))
        return None, dsigma, None


class BaseNoiseS2(nn.Module):
    r"""Common part of the noise modules: the inverse SHT (distributed under h x w), a CPU and a CUDA generator seeded with `seed`, and the
    non-persistent spectral state buffer.  Its own update() is memoryless (the isotropic field's).  Arguments as makani's BaseNoiseS2."""

    def __init__(self, img_shape, batch_size, num_channels, num_time_steps, grid_type="equiangular", lmax=None, seed=333, reflect=False, **kwargs):
        super().__init__()
        self.nlat, self.nlon = img_shape
        self.num_channels = num_channels
        self.num_time_steps = num_time_steps
        self.reflect = reflect

        grid = _grid()
        self._distributed = grid is not None
        if self._distributed:
            from .distributed import DistributedInverseRealSHT

            rank_h, rank_w = grid[2], grid[3]
            self.isht = DistributedInverseRealSHT(self.nlat, self.nlon, lmax=lmax, mmax=lmax, grid=grid_type)
            self.lmax_local, self.nlat_local = self.isht.l_shapes[rank_h], self.isht.lat_shapes[rank_h]
            self.mmax_local, self.nlon_local = self.isht.m_shapes[rank_w], self.isht.lon_shapes[rank_w]
        else:
            self.isht = InverseRealSHT(self.nlat, self.nlon, lmax=lmax, mmax=lmax, grid=grid_type)
            self.lmax_local, self.nlat_local = self.isht.lmax, self.nlat
            self.mmax_local, self.nlon_local = self.isht.mmax, self.nlon
        self.lmax, self.mmax = self.isht.lmax, self.isht.mmax

        self.set_rng(seed=seed)
        self._ensure_state(batch_size, device=torch.device("cpu"), dtype=torch.float32)

    @property
    def _state_shape_suffix(self):
        return (self.num_time_steps, self.num_channels, self.lmax_local, self.mmax_local, 2)

    def _ensure_state(self, batch_size, device=None, dtype=None):
        """give the state buffer `batch_size` rows: registered anew (zeros, on the state's device and dtype unless given) only when its shape
        changes, so `.to()` keeps moving it and an unchanged size keeps the same storage"""
        shape = (batch_size, *self._state_shape_suffix)
        current = self._buffers.get("state")
        if current is not None and tuple(current.shape) == shape:
            return
        if device is None:
            device = torch.device("cpu") if current is None else current.device
        if dtype is None:
            dtype = torch.float32 if current is None else current.dtype
        self.register_buffer("state", torch.zeros(shape, dtype=dtype, device=device), persistent=False)

    def is_stateful(self):
        raise NotImplementedError(f"{type(self).__name__} does not say whether it carries state across calls")

    def extra_repr(self):
        # makani's text, so printed models read the same
        return (f"img_shape=({self.nlat}, {self.nlon}), num_channels={self.num_channels}, num_time_steps={self.num_time_steps}, "
                f"lmax={self.lmax}, reflect={self.reflect}")

    def set_rng(self, seed=333):
        """new private generators seeded with `seed`: a CPU one, and a CUDA one on the current device when CUDA is available"""
        self.rng_cpu = torch.Generator(device=torch.device("cpu"))
        self.rng_cpu.manual_seed(seed)
        if torch.cuda.is_available():
            self.rng_gpu = torch.Generator(device=torch.device("cuda", torch.cuda.current_device()))
            self.rng_gpu.manual_seed(seed)

    def reset(self, batch_size=None):
        """zero the state, first resizing it to `batch_size` when that is given"""
        if batch_size is not None:
            self._ensure_state(batch_size)
        with torch.no_grad():
            self.state.zero_()

    def _draw(self, shape):
        """standard normals of `shape` from the CUDA generator: makani's draw"""
        xi = torch.empty(shape, dtype=self.state.dtype, device=self.state.device)
        return xi.normal_(mean=0.0, std=1.0, generator=self.rng_gpu)

    def _advance(self, xi, mode, sigma=None, phi=None, discount=None):
        B, T, C, L, M, _ = self.state.shape
        _lib.call("b200sht_noise_update", _ptr(self.state), _ptr(xi), _ptr(sigma), _ptr(phi), _ptr(discount), B, T, C, L, M, mode,
                  1 if self.reflect else 0, _stream(self.state.device))

    def update(self, replace_state=False, batch_size=None):
        """memoryless: the state becomes fresh standard normal coefficients (negated when `reflect`); replace_state is ignored"""
        if batch_size is not None:
            self._ensure_state(batch_size)
        _check_operands(f"{type(self).__name__}.update", state=self.state)
        with torch.no_grad():
            self._advance(self._draw(self.state.shape), _lib.NOISE_BASE)

    def set_rng_state(self, cpu_state, gpu_state):
        """restore generator states from get_rng_state(); None leaves that generator as it is (the CUDA one also without CUDA)"""
        if cpu_state is not None:
            self.rng_cpu.set_state(cpu_state)
        if gpu_state is not None and torch.cuda.is_available():
            self.rng_gpu.set_state(gpu_state)

    def get_rng_state(self):
        """(CPU generator state, CUDA generator state or None without CUDA)"""
        return self.rng_cpu.get_state(), (self.rng_gpu.get_state() if torch.cuda.is_available() else None)

    def get_tensor_state(self):
        return self.state.detach().clone()

    def set_tensor_state(self, newstate):
        """copy `newstate` into the state; its batch size may differ (the buffer is resized), any other dimension raises ValueError before the
        state is touched"""
        want = tuple(self._state_shape_suffix)
        got = tuple(newstate.shape[1:])
        if newstate.dim() == 0 or got != want:
            raise ValueError(f"set_tensor_state: {type(self).__name__} holds states of shape (batch, {', '.join(map(str, want))}); "
                             f"got {tuple(newstate.shape)}")
        self._ensure_state(newstate.shape[0])
        with torch.no_grad():
            self.state.copy_(newstate)

    def _synthesize(self, sigma):
        """state (scaled by sigma when given) -> fp32 fields (B, T, C, nlat_local, nlon_local)"""
        _check_operands(f"{type(self).__name__}.forward", state=self.state, sigma_l=sigma)
        B = self.state.shape[0]
        TC = self.num_time_steps * self.num_channels
        with amp.autocast(device_type="cuda", enabled=False):
            if self._distributed:
                eta = self.isht(_NoiseSpectrum.apply(self.state, sigma, False))
            else:
                eta = self.isht.forward_packed(_NoiseSpectrum.apply(self.state, sigma, True), B, TC, torch.float32)
        return eta.reshape(B, self.num_time_steps, self.num_channels, self.nlat_local, self.nlon_local)


def _shard(t, dims_and_sizes):
    """this rank's slice of `t`: for each (dim, number of ranks, rank) the chunk of makani_b200.distributed's split"""
    from .distributed import split_tensor_along_dim

    for dim, n, rank in dims_and_sizes:
        if n > 1:
            t = split_tensor_along_dim(t, dim=dim, num_chunks=n)[rank]
    return t


class IsotropicGaussianRandomFieldS2(BaseNoiseS2):
    r"""Isotropic Gaussian random field on the sphere, redrawn independently by every update (not stateful).

    Degree l has standard deviation sigma_l = sigma sqrt((2l+1)^-alpha / Z) with Z = sum_l (2l+1)^(1-alpha) / (4 pi), so the field's
    pointwise variance is sigma^2 whatever alpha and the truncation; sigma_l is 0 for m > l.  forward() synthesises (state / sqrt 2) sigma_l.
    `learnable` makes sigma_l a parameter.  Arguments as makani's class."""

    def __init__(self, img_shape, batch_size, num_channels, num_time_steps=1, sigma=1.0, alpha=0.0, grid_type="equiangular", lmax=None, seed=333,
                 reflect=False, learnable=False, **kwargs):
        super().__init__(img_shape=img_shape, batch_size=batch_size, num_channels=num_channels, num_time_steps=num_time_steps, grid_type=grid_type,
                         lmax=lmax, seed=seed, reflect=reflect)
        self.sigma, self.alpha, self.learnable = sigma, alpha, learnable

        degree = torch.arange(self.lmax).reshape(-1, 1)
        order = torch.arange(self.mmax)
        spectrum = torch.pow(2 * degree + 1, -float(alpha))
        z = torch.sum((2 * degree + 1) * spectrum / 4.0 / math.pi)
        sigma_l = torch.where(order <= degree, sigma * torch.sqrt(spectrum / z), 0.0)
        sigma_l = sigma_l.reshape(1, 1, 1, self.lmax, self.mmax).to(dtype=torch.float32)

        grid = _grid()
        if grid is not None:
            h, w, rank_h, rank_w = grid
            sigma_l = _shard(sigma_l, [(-2, h, rank_h), (-1, w, rank_w)])
        sigma_l = sigma_l.contiguous()
        if learnable:
            self.sigma_l = nn.Parameter(sigma_l)
            self.sigma_l.sharded_dims_mp = [None, None, None, "h", "w"]
        else:
            self.register_buffer("sigma_l", sigma_l, persistent=False)

    def is_stateful(self):
        return False

    def extra_repr(self):
        return super().extra_repr() + f", sigma={self.sigma}, alpha={self.alpha}, learnable={self.learnable}"

    @torch.compiler.disable
    def forward(self, update_internal_state=False):
        """(state / sqrt 2) sigma_l through the inverse SHT: fp32 (B, T, C, nlat_local, nlon_local); then update() if requested"""
        eta = self._synthesize(self.sigma_l)
        if update_internal_state:
            self.update()
        return eta


def _per_channel(value, name, num_channels):
    """a scalar repeated, or a list with one entry per channel, as a (num_channels, 1) tensor"""
    if not isinstance(value, list):
        return torch.as_tensor([value]).repeat(num_channels).reshape(num_channels, 1)
    t = torch.as_tensor(value)
    if t.dim() != 1 or t.shape[0] != num_channels:
        raise ValueError(f"{name} as a list needs one number per channel ({num_channels}), got shape {tuple(t.shape)}")
    return t.reshape(num_channels, 1)


def _discount(phi, T):
    """[C][T][T] fp32: discount[c][t][q] = phi_c^(t - q) for q <= t, 0 above the diagonal (powers in fp64, from each fp32 phi)"""
    k = np.arange(T)
    lag = k[:, None] - k[None, :]
    out = []
    for p in phi.reshape(-1).tolist():
        phivec = np.power(p, k)
        out.append(torch.as_tensor(np.where(lag >= 0, phivec[np.clip(lag, 0, None)], 0.0)).to(dtype=torch.float32))
    return torch.stack(out, dim=0)


class DiffusionNoiseS2(BaseNoiseS2):
    r"""Temporally correlated random field from a diffusion process on the sphere (stateful).

    Every spectral coefficient follows an AR(1) process eta_{t+1} = phi eta_t + sigma_l xi_t, phi = exp(-lambd) per channel, with
    sigma_l = sqrt(4 pi) F0 exp(-kT l (l+1) / 2) and F0 = sigma sqrt((1 - phi^2) / (2 sum_{l >= 1} (2l+1) exp(-kT l (l+1)))): kT sets the
    spatial correlation length, lambd the temporal one; either may be a list with one value per channel.  Arguments as makani's class."""

    def __init__(self, img_shape, batch_size, num_channels, num_time_steps=1, sigma=1.0, kT=0.5 * (500.0 / 6370.0) ** 2, lambd=1.0,
                 grid_type="equiangular", lmax=None, seed=333, reflect=False, learnable=False, **kwargs):
        super().__init__(img_shape=img_shape, batch_size=batch_size, num_channels=num_channels, num_time_steps=num_time_steps, grid_type=grid_type,
                         lmax=lmax, seed=seed, reflect=reflect)
        self.sigma, self.kT, self.lambd, self.learnable = sigma, kT, lambd, learnable
        if learnable and num_time_steps > 1:
            raise NotImplementedError("DiffusionNoiseS2: a learnable process is supported for num_time_steps = 1 only")

        k = _per_channel(kT, "kT", num_channels)
        lam = _per_channel(lambd, "lambd", num_channels)
        # the same sequence of fp32 operations as the reference, so the buffers agree bit for bit
        degree = torch.arange(self.lmax)
        damping = torch.exp(-k * degree * (degree + 1))
        total = torch.sum((2 * degree[1:] + 1) * damping[..., 1:], dim=-1, keepdim=True)
        phi = torch.exp(-lam)
        f0 = sigma * torch.sqrt(0.5 * (1 - phi**2) / total)
        sigma_l = math.sqrt(4 * math.pi) * (f0 * torch.exp(-0.5 * k * degree * (degree + 1)))

        phi = phi.reshape(num_channels, 1, 1, 1).to(dtype=torch.float32)
        sigma_l = sigma_l.reshape(1, 1, num_channels, self.lmax, 1).to(dtype=torch.float32)
        grid = _grid()
        if grid is not None:
            sigma_l = _shard(sigma_l, [(-2, grid[0], grid[2])])
        sigma_l = sigma_l.unsqueeze(-1).contiguous()

        if learnable:
            self.phi = nn.Parameter(phi)
            self.phi.is_shared_mp = ["matmul", "h", "w"]
            self.phi.sharded_dims_mp = [None, None, None]
            self.sigma_l = nn.Parameter(sigma_l)
            self.sigma_l.is_shared_mp = ["matmul", "w"]
            self.sigma_l.sharded_dims_mp = [None, None, None, "h", None, None]
        else:
            self.register_buffer("phi", phi, persistent=False)
            self.register_buffer("sigma_l", sigma_l, persistent=False)
        if num_time_steps > 1:
            self.register_buffer("discount", _discount(self.phi, num_time_steps), persistent=False)

    def is_stateful(self):
        return True

    def extra_repr(self):
        return super().extra_repr() + f", sigma={self.sigma}, kT={self.kT}, lambd={self.lambd}, learnable={self.learnable}"

    def update(self, replace_state=False, batch_size=None):
        """replace_state=False: one AR step (the oldest of T steps dropped); True: a fresh history from the stationary distribution (step 0
        scaled by 1 / sqrt(1 - phi^2), the T steps correlated by the discount)"""
        if batch_size is not None:
            self._ensure_state(batch_size)
        discount = self.discount if (replace_state and self.num_time_steps > 1) else None
        sigma_l, phi = self.sigma_l.detach(), self.phi.detach()
        _check_operands("DiffusionNoiseS2.update", state=self.state, sigma_l=sigma_l, phi=phi, discount=discount)
        with torch.no_grad():
            if replace_state:
                xi = self._draw(self.state.shape)
            else:
                xi = self._draw((self.state.shape[0], 1, self.num_channels, self.lmax_local, self.mmax_local, 2))
            self._advance(xi, _lib.NOISE_STATIONARY if replace_state else _lib.NOISE_AR, sigma=sigma_l.contiguous(), phi=phi.contiguous(),
                          discount=None if discount is None else discount.contiguous())

    @torch.compiler.disable
    def forward(self, update_internal_state=False):
        """the state through the inverse SHT: fp32 (B, T, C, nlat_local, nlon_local); then update() if requested"""
        eta = self._synthesize(None)
        if update_internal_state:
            self.update()
        return eta


class DummyNoiseS2(BaseNoiseS2):
    """Noise of the right shape without a transform (spatial state (B, T, C, nlat_local, nlon_local)): mode 'constant_zero' or
    'constant_random' (a Gaussian draw held until the next update).  Runs on any device."""

    MODES = ("constant_zero", "constant_random")

    def __init__(self, img_shape, batch_size, num_channels, num_time_steps=1, mode="constant_zero", seed=333, **kwargs):
        if mode not in self.MODES:
            raise ValueError(f"DummyNoiseS2: mode must be one of {self.MODES}, got {mode!r}")
        self.mode = mode
        super().__init__(img_shape=img_shape, batch_size=batch_size, num_channels=num_channels, num_time_steps=num_time_steps, seed=seed)

    @property
    def _state_shape_suffix(self):
        return (self.num_time_steps, self.num_channels, self.nlat_local, self.nlon_local)

    def is_stateful(self):
        return False

    def extra_repr(self):
        return super().extra_repr() + f", mode={self.mode}"

    def update(self, replace_state=False, batch_size=None):
        """constant_zero: zeros; constant_random: standard normals from the generator of the state's device (replace_state is ignored)"""
        if batch_size is not None:
            self._ensure_state(batch_size)
        with torch.no_grad():
            if self.mode == "constant_random":
                self.state.normal_(mean=0.0, std=1.0, generator=self.rng_gpu if self.state.is_cuda else self.rng_cpu)
            else:
                self.state.zero_()

    def forward(self, update_internal_state=False):
        """the live state buffer (not a copy); then update() if requested"""
        state = self.state
        if update_internal_state:
            self.update()
        return state


_BUILDERS = {"diffusion": DiffusionNoiseS2, "white": IsotropicGaussianRandomFieldS2, "dummy": DummyNoiseS2}


def build_noise(noise_params, *, img_shape, batch_size, num_channels, num_time_steps, grid_type, seed, reflect, default_lambd=1.0):
    """the noise module a config asks for: noise_params["type"] "diffusion" / "white" / "dummy" -> DiffusionNoiseS2 /
    IsotropicGaussianRandomFieldS2 / DummyNoiseS2, with makani's factory defaults (kT 0.5 (100 / 6370)^2 here, not the class's; lambd
    `default_lambd`; a dummy is always constant_zero)"""
    kind = noise_params.get("type")
    if kind is None:
        raise ValueError("build_noise: noise_params has no 'type' (one of 'diffusion', 'white', 'dummy')")
    if kind not in _BUILDERS:
        raise NotImplementedError(f"build_noise: noise type {kind!r} is not supported (one of 'diffusion', 'white', 'dummy')")
    shape = dict(img_shape=img_shape, batch_size=batch_size, num_channels=num_channels, num_time_steps=num_time_steps)
    if kind == "dummy":
        return DummyNoiseS2(**shape)
    spectral = dict(shape, sigma=noise_params.get("sigma", 1.0), grid_type=grid_type, lmax=noise_params.get("lmax"), seed=seed, reflect=reflect,
                    learnable=noise_params.get("learnable", False))
    if kind == "white":
        return IsotropicGaussianRandomFieldS2(alpha=noise_params.get("alpha", 0.0), **spectral)
    return DiffusionNoiseS2(kT=noise_params.get("kT", 0.5 * (100 / 6370) ** 2), lambd=noise_params.get("lambd", default_lambd), **spectral)

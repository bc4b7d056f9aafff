"""Checkpoints, parameter synchronisation and gradient reduction of a model under h x w spatial model parallelism, driven only by the
`is_shared_mp` / `sharded_dims_mp` tags makani sets on parameters (any tagged model, not only FCN3).

    scatter_state_dict(model, global_sd)   makani/utils/checkpoint_helpers.py:scatter_model_state_dict: this rank's slice of every dimension
                                           tagged "h" or "w", by compute_split_shapes of its global size
    gather_state_dict(model)               gather_model_state_dict: those dimensions reassembled, every tensor on the CPU
    sync_shared_params(model)              makani/mpu/helpers.py:sync_params (mode "broadcast"): each parameter broadcast from the first rank of
                                           every group in its is_shared_mp
    reduce_shared_gradients(model)         the comm hook of makani/mpu/mappings.py:init_gradient_reduction_hooks without the data-parallel
                                           mean: each gradient summed over every group in its is_shared_mp

Group names: "h" is makani_b200.distributed.polar_group(), "w" azimuth_group(); "spatial" and "model" are both (h x w; "model" equals "spatial"
while makani's matmul parallelism is 1, and it is never built here); "matmul" is a group of one.  A parameter without is_shared_mp counts as
["model"], as makani treats it.  Groups are reduced azimuth first, then polar, in a fixed order, so every rank of the grid sums the same values in
the same order.
"""
from collections import OrderedDict

import torch
import torch.distributed as dist
from torch._utils import _flatten_dense_tensors, _unflatten_dense_tensors

from .primitives import compute_split_shapes

_SHARDED = ("h", "w")


def _group_of(name):
    """the process group of a sharded-dimension tag"""
    from . import azimuth_group, polar_group
    return {"h": polar_group, "w": azimuth_group}[name]()


def _shared_groups(param):
    """the process groups a parameter's gradient is summed over / its value is broadcast over, in the fixed order (azimuth, polar)"""
    from . import azimuth_group, polar_group
    names = set()
    for tag in getattr(param, "is_shared_mp", ["model"]):
        if tag in ("spatial", "model"):
            names |= {"h", "w"}
        elif tag in _SHARDED:
            names.add(tag)
        elif tag != "matmul":
            raise ValueError(f"unknown model-parallel group {tag!r} in is_shared_mp (known: h, w, spatial, model, matmul)")
    return [g for n, g in (("w", azimuth_group()), ("h", polar_group())) if n in names and _size(g) > 1]


def _size(g):
    from . import _size as size
    return size(g)


def _sharded_dims(param):
    """[(dim, group name)] of the dimensions of `param` split over a group of more than one rank"""
    out = []
    for d, tag in enumerate(getattr(param, "sharded_dims_mp", None) or []):
        if tag is None or tag == "matmul":
            continue
        if tag not in _SHARDED:
            raise ValueError(f"unknown model-parallel group {tag!r} in sharded_dims_mp (known: h, w, matmul)")
        if _size(_group_of(tag)) > 1:
            out.append((d, tag))
    return out


def scatter_state_dict(model, global_sd):
    """the state dict of this rank from the global (flexible-format) one: every parameter dimension tagged "h" / "w" sliced to this rank's
    compute_split_shapes part, every other entry as given.  Load the result with model.load_state_dict(local_sd, strict=True)."""
    from . import _rank
    params = dict(model.named_parameters())
    out = OrderedDict()
    for k, v in global_sd.items():
        p = params.get(k)
        if p is not None:
            for d, tag in _sharded_dims(p):
                g = _group_of(tag)
                v = torch.split(v, compute_split_shapes(v.shape[d], _size(g)), dim=d)[_rank(g)]
            v = v.contiguous()
        out[k] = v
    return out


def _gather_uneven(t, dim, group):
    """the shards of every rank of `group` concatenated along `dim` in rank order; shards may differ in size along `dim` (padded for the
    all-gather, which needs equal sizes)"""
    n = _size(group)
    size = torch.tensor([t.shape[dim]], dtype=torch.int64, device=t.device)
    sizes = [torch.empty_like(size) for _ in range(n)]
    dist.all_gather(sizes, size, group=group)
    sizes = [int(s.item()) for s in sizes]
    pad = list(t.shape)
    pad[dim] = max(sizes)
    buf = t.new_zeros(pad)
    buf.narrow(dim, 0, t.shape[dim]).copy_(t)
    parts = [torch.empty_like(buf) for _ in range(n)]
    dist.all_gather(parts, buf, group=group)
    return torch.cat([p.narrow(dim, 0, s) for p, s in zip(parts, sizes)], dim=dim)


def gather_state_dict(model):
    """the global state dict (on the CPU) of a model whose parameters are this rank's shards: every dimension tagged "h" / "w" gathered over its
    group in rank order; every rank issues the same collectives and receives the whole state dict"""
    params = dict(model.named_parameters())
    out = OrderedDict()
    for k, v in model.state_dict().items():
        p = params.get(k)
        if p is not None:
            for d, tag in _sharded_dims(p):
                v = _gather_uneven(v, d, _group_of(tag))
        out[k] = v.detach().cpu()
    return out


@torch.no_grad()
def sync_shared_params(model):
    """each parameter broadcast from the first rank of every group in its is_shared_mp (azimuth, then polar: a parameter shared over the whole
    grid takes the value of the grid's first rank), so that replicated parameters start out identical"""
    for p in model.parameters():
        for g in _shared_groups(p):
            t = torch.view_as_real(p) if p.is_complex() else p
            buf = t.detach().contiguous()
            dist.broadcast(buf, src=dist.get_global_rank(g, 0), group=g)
            if buf.data_ptr() != t.data_ptr():
                t.copy_(buf)


@torch.no_grad()
def reduce_shared_gradients(model):
    """after backward: each gradient summed over every group in its parameter's is_shared_mp, one coalesced all-reduce per group and dtype.  A
    parameter replicated on every spatial rank then holds the gradient of the whole grid, and a sharded one the gradient of its slice.  Call it
    between backward() and the optimizer step; the data-parallel reduction, if any, is the caller's."""
    from . import azimuth_group, polar_group
    for g in (azimuth_group(), polar_group()):
        if _size(g) == 1:
            continue
        by_dtype = {}
        for p in model.parameters():
            if p.grad is not None and any(h is g for h in _shared_groups(p)):
                grad = torch.view_as_real(p.grad) if p.grad.is_complex() else p.grad
                by_dtype.setdefault((grad.dtype, grad.device), []).append(grad)
        for grads in by_dtype.values():
            flat = _flatten_dense_tensors(grads)
            dist.all_reduce(flat, group=g)
            for grad, red in zip(grads, _unflatten_dense_tensors(flat, grads)):
                grad.copy_(red)

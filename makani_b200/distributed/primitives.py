"""Collective primitives of the h x w spatial model-parallel path -- mirror of `torch_harmonics.distributed.primitives`
as makani uses it (/root/reference/makani/mpu/mappings.py:19-25,45,65,91,104,127,141,162,175).

`_transpose` is the all-to-all that moves the shard from one tensor dimension to another.  On NCCL it is one grouped
`dist.all_to_all` over NVLink; backends without all-to-all (gloo, used by the CPU tests) fall back to batched isend/irecv.
"""
from typing import List

import torch
import torch.distributed as dist


def compute_split_shapes(size: int, num_chunks: int) -> List[int]:
    """chunk = ceil(size / n) for the first n-1 ranks, remainder last (floor split if the last would be empty)."""
    if num_chunks == 1:
        return [size]
    chunk = (size + num_chunks - 1) // num_chunks
    last = max(0, size - chunk * (num_chunks - 1))
    if last == 0:
        chunk = size // num_chunks
        last = size - chunk * (num_chunks - 1)
    return [chunk for _ in range(num_chunks - 1)] + [last]


def split_tensor_along_dim(tensor, dim, num_chunks):
    if dim >= tensor.dim() or dim < -tensor.dim():
        raise ValueError(f"cannot split tensor of dimension {tensor.dim()} along dimension {dim}")
    if tensor.shape[dim] < num_chunks:
        raise ValueError(f"cannot split dimension {dim} of size {tensor.shape[dim]} into {num_chunks} chunks")
    return torch.split(tensor, compute_split_shapes(tensor.shape[dim], num_chunks), dim=dim)


def _group_size(group):
    return dist.get_world_size(group=group) if (dist.is_available() and dist.is_initialized()) else 1


def _all_to_all(recv, send, group):
    backend = dist.get_backend(group)
    if backend == "nccl" or backend == "mpi":
        return dist.all_to_all(recv, send, group=group)
    # gloo: pairwise exchange; empty chunks (the variable-size halo of the distributed DISCO convolution) are not sent
    rank = dist.get_rank(group=group)
    ranks = dist.get_process_group_ranks(group) if group is not None else list(range(dist.get_world_size()))
    recv[rank].copy_(send[rank])
    ops = []
    for j, peer in enumerate(ranks):
        if j == rank:
            continue
        if send[j].numel():
            ops.append(dist.P2POp(dist.isend, send[j], peer, group))
        if recv[j].numel():
            ops.append(dist.P2POp(dist.irecv, recv[j], peer, group))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return None


def _transpose(tensor, dim0, dim1, dim1_split_sizes, group=None, async_op=False):
    """Shard along dim0, gather along dim1.  Returns (list of received chunks, dim0 split sizes, request)."""
    comm_size = dist.get_world_size(group=group)
    comm_rank = dist.get_rank(group=group)
    x_send = [t.contiguous() for t in split_tensor_along_dim(tensor, dim0, comm_size)]
    x_send_shapes = [t.shape for t in x_send]
    x_recv = []
    x_shape = list(x_send_shapes[comm_rank])
    for dim1_len in dim1_split_sizes:
        x_shape[dim1] = dim1_len
        x_recv.append(torch.empty(x_shape, dtype=tensor.dtype, device=tensor.device))
    req = _all_to_all(x_recv, x_send, group)
    dim0_split_sizes = [s[dim0] for s in x_send_shapes]
    return x_recv, dim0_split_sizes, req


def _reduce(input_, use_fp32=True, group=None):
    if _group_size(group) == 1:
        return input_
    if use_fp32 and input_.dtype.itemsize < 4 and input_.dtype.is_floating_point:
        dtype = input_.dtype
        inputf = input_.float()
        dist.all_reduce(inputf, group=group)
        return inputf.to(dtype)
    inp = input_.contiguous()
    dist.all_reduce(inp, group=group)
    return inp


def _split(input_, dim_, group=None):
    comm_size = _group_size(group)
    if comm_size == 1:
        return input_
    return split_tensor_along_dim(input_, dim_, comm_size)[dist.get_rank(group=group)].contiguous()


def _gather(input_, dim_, shapes_, group=None):
    comm_size = _group_size(group)
    if comm_size == 1:
        return input_
    if len(shapes_) != comm_size or dim_ >= input_.dim():
        raise ValueError("_gather: shapes / dim mismatch")
    comm_rank = dist.get_rank(group=group)
    input_ = input_.contiguous()
    shape = list(input_.shape)
    chunks = []
    for s in shapes_:
        shape[dim_] = s
        chunks.append(torch.empty(shape, dtype=input_.dtype, device=input_.device))
    chunks[comm_rank] = input_
    dist.all_gather(chunks, input_, group=group)
    return torch.cat(chunks, dim=dim_).contiguous()


class _DistributedTranspose(torch.autograd.Function):
    """forward: shard dims[0], gather dims[1]; backward: the inverse transpose (as /root/reference/makani/mpu/mappings.py:38-67)."""

    @staticmethod
    def forward(ctx, x, dims, dim1_split_sizes, group):
        xlist, dim0_split_sizes, _ = _transpose(x.contiguous(), dims[0], dims[1], dim1_split_sizes, group=group)
        ctx.dims, ctx.dim0_split_sizes, ctx.group = dims, dim0_split_sizes, group
        return torch.cat(xlist, dim=dims[1]).contiguous()

    @staticmethod
    def backward(ctx, go):
        gilist, _, _ = _transpose(go.contiguous(), ctx.dims[1], ctx.dims[0], ctx.dim0_split_sizes, group=ctx.group)
        return torch.cat(gilist, dim=ctx.dims[0]).contiguous(), None, None, None

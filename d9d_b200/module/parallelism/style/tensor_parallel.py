"""Tensor parallelism for linear layers — net-new (the reference only reserves the ``tp`` mesh dim and raises).

``ColwiseLinearParallel``  shards the *output* features: ``W [out, in] -> Shard(0)``; the input is replicated
(identity forward / all-reduce backward) or, with ``sequence_parallel=True``, all-gathered along the sequence dim
(all-gather forward / reduce-scatter backward).

``RowwiseLinearParallel``  shards the *input* features: ``W -> Shard(1)``; partial outputs are all-reduced
(all-reduce forward / identity backward) or reduce-scattered along the sequence dim when ``sequence_parallel``.

With ``sequence_parallel=True`` on CUDA the collective is fused into the wgmma GEMM over NVLink peer memory
(``d9d_b200.kernel.tp``): all-gather→GEMM loads every A tile from the owning peer through TMA, GEMM→reduce-scatter
TMA reduce-adds every output tile into the owner's shard; backward uses the mirrored kernels.  Otherwise (CPU/gloo,
unsupported shapes, plain all-reduce TP) the collectives are autograd functions over the ``tp`` process group around
the local GEMM.
"""

from __future__ import annotations

from typing import Any

import torch
import torch.distributed as dist
from torch import nn
from torch.distributed import DeviceMesh
from torch.distributed.tensor import DTensor, Replicate, Shard, distribute_tensor
from torch.distributed.tensor.parallel import ParallelStyle

from d9d_b200.kernel._native import MAIN_PARAM_ATTR


class _CopyToGroup(torch.autograd.Function):
    """Identity forward, all-reduce(SUM) backward."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, group: dist.ProcessGroup) -> torch.Tensor:
        ctx.group = group
        return x

    @staticmethod
    def backward(ctx: Any, grad: torch.Tensor):  # type: ignore[override]
        grad = grad.contiguous()
        dist.all_reduce(grad, group=ctx.group)
        return grad, None


class _ReduceFromGroup(torch.autograd.Function):
    """all-reduce(SUM) forward, identity backward."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, group: dist.ProcessGroup) -> torch.Tensor:
        x = x.contiguous()
        dist.all_reduce(x, group=group)
        return x

    @staticmethod
    def backward(ctx: Any, grad: torch.Tensor):  # type: ignore[override]
        return grad, None


class _GatherSequence(torch.autograd.Function):
    """all-gather along ``dim`` forward, reduce-scatter backward (sequence parallel entry)."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, group: dist.ProcessGroup, dim: int) -> torch.Tensor:
        ctx.group, ctx.dim = group, dim
        parts = [torch.empty_like(x) for _ in range(group.size())]
        dist.all_gather(parts, x.contiguous(), group=group)
        return torch.cat(parts, dim=dim)

    @staticmethod
    def backward(ctx: Any, grad: torch.Tensor):  # type: ignore[override]
        chunks = [c.contiguous() for c in grad.chunk(ctx.group.size(), dim=ctx.dim)]
        out = torch.empty_like(chunks[0])
        dist.reduce_scatter(out, chunks, group=ctx.group)
        return out, None, None


class _ScatterSequence(torch.autograd.Function):
    """reduce-scatter along ``dim`` forward, all-gather backward (sequence parallel exit)."""

    @staticmethod
    def forward(ctx: Any, x: torch.Tensor, group: dist.ProcessGroup, dim: int) -> torch.Tensor:
        ctx.group, ctx.dim = group, dim
        chunks = [c.contiguous() for c in x.chunk(group.size(), dim=dim)]
        out = torch.empty_like(chunks[0])
        dist.reduce_scatter(out, chunks, group=group)
        return out

    @staticmethod
    def backward(ctx: Any, grad: torch.Tensor):  # type: ignore[override]
        parts = [torch.empty_like(grad) for _ in range(ctx.group.size())]
        dist.all_gather(parts, grad.contiguous(), group=ctx.group)
        return torch.cat(parts, dim=ctx.dim), None, None


class _TensorParallelLinear(ParallelStyle):
    shard_dim: int

    def __init__(self, tp_dim_name: str = "tp", sequence_parallel: bool = False, sequence_dim: int = 1):
        self._tp = tp_dim_name
        self._sp = sequence_parallel
        self._seq_dim = sequence_dim

    def _distribute(self, module: nn.Module, device_mesh: DeviceMesh) -> dist.ProcessGroup:
        if not isinstance(module, nn.Linear):
            raise TypeError("tensor-parallel styles apply to nn.Linear modules")
        names = device_mesh.mesh_dim_names
        if names is None or self._tp not in names:
            raise ValueError(f"mesh must have a '{self._tp}' dimension")
        placements = [Shard(self.shard_dim) if n == self._tp else Replicate() for n in names]
        weight = module.weight
        if isinstance(weight.data, DTensor):
            raise ValueError("weight is already distributed")
        module.weight = nn.Parameter(distribute_tensor(weight.data, device_mesh, placements, src_data_rank=None),
                                     requires_grad=weight.requires_grad)
        if module.bias is not None:
            bias_pl = [Shard(0) if (n == self._tp and self.shard_dim == 0) else Replicate() for n in names]
            module.bias = nn.Parameter(distribute_tensor(module.bias.data, device_mesh, bias_pl, src_data_rank=None),
                                       requires_grad=module.bias.requires_grad)
        return device_mesh.get_group(self._tp)


def _local(t: torch.Tensor | None) -> torch.Tensor | None:
    if isinstance(t, DTensor):
        local = t.to_local()
        setattr(local, MAIN_PARAM_ATTR, t)  # wgrad kernels may accumulate straight into the sharded parameter's .grad
        return local
    return t


class ColwiseLinearParallel(_TensorParallelLinear):
    shard_dim = 0

    def _apply(self, module: nn.Module, device_mesh: DeviceMesh) -> nn.Module:
        from d9d_b200.kernel.gemm import linear

        group = self._distribute(module, device_mesh)
        sp, seq_dim = self._sp, self._seq_dim

        def forward(x: torch.Tensor) -> torch.Tensor:
            if sp and seq_dim == x.dim() - 2:
                from d9d_b200.kernel.tp.fused import all_gather_linear, fused_tp_supported

                weight = _local(module.weight)
                if fused_tp_supported(x, weight, group, x.shape[-2] * group.size()):
                    out = all_gather_linear(x, weight, group)  # all-gather fused into the GEMM's TMA loads
                    bias = _local(module.bias)
                    return out if bias is None else out + bias
            x = _GatherSequence.apply(x, group, seq_dim) if sp else _CopyToGroup.apply(x, group)
            return linear(x, _local(module.weight), _local(module.bias))

        module.forward = forward  # type: ignore[method-assign]
        return module


class RowwiseLinearParallel(_TensorParallelLinear):
    shard_dim = 1

    def _apply(self, module: nn.Module, device_mesh: DeviceMesh) -> nn.Module:
        from d9d_b200.kernel.gemm import linear

        group = self._distribute(module, device_mesh)
        sp, seq_dim = self._sp, self._seq_dim

        def forward(x: torch.Tensor) -> torch.Tensor:
            if sp and seq_dim == x.dim() - 2:
                from d9d_b200.kernel.tp.fused import fused_tp_supported, linear_reduce_scatter

                weight = _local(module.weight)
                if fused_tp_supported(x, weight, group, x.shape[-2]):
                    out = linear_reduce_scatter(x, weight, group)  # reduce-scatter fused into the GEMM epilogue
                    bias = _local(module.bias)
                    return out if bias is None else out + bias
            partial = linear(x, _local(module.weight), None)
            out = _ScatterSequence.apply(partial, group, seq_dim) if sp else _ReduceFromGroup.apply(partial, group)
            bias = _local(module.bias)
            return out if bias is None else out + bias

        module.forward = forward  # type: ignore[method-assign]
        return module

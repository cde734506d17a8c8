"""Auxiliary-loss-free load balancing (DeepSeek-V3, §2.1.2): after each optimizer step every expert's selection bias moves
by a fixed rate toward balance, ``b_e += rate * sign(mean(c) - c_e)`` with ``c_e`` the number of times expert ``e`` was
selected during the step."""

from __future__ import annotations

from collections.abc import Iterable

import torch
import torch.distributed as dist
from torch import nn
from torch.distributed import ProcessGroup

from .layer import MoELayer


def expert_bias_layers(modules: Iterable[nn.Module]) -> list[MoELayer]:
    """The MoE layers under ``modules`` whose router carries an expert bias, each once, in module order."""
    found: dict[int, MoELayer] = {}
    for module in modules:
        for m in module.modules():
            if isinstance(m, MoELayer) and m.router.expert_bias is not None:
                found.setdefault(id(m), m)
    return list(found.values())


def expert_bias_master(layer: MoELayer) -> torch.Tensor:
    """The fp32 master copy of ``layer``'s expert bias.

    The bias buffer is usually bf16 (models are cast whole), where a step of ~1e-3 is lost once ``|b| >= 0.5``; the
    update is therefore applied to this master and the buffer receives its rounded value.  The master is (re)taken from
    the buffer whenever the buffer no longer holds the master's rounded value, e.g. after weights were loaded."""
    bias = layer.router.expert_bias
    master = getattr(layer.router, "expert_bias_master", None)
    if master is None or master.device != bias.device or not torch.equal(master.to(bias.dtype), bias):
        master = bias.detach().float().clone()
        layer.router.expert_bias_master = master
    return master


@torch.no_grad()
def update_expert_bias(modules: Iterable[nn.Module], update_rate: float, group: ProcessGroup | None = None) -> None:
    """Apply one balancing step to every MoE layer under ``modules`` whose router has an expert bias.

    The layers' ``tokens_per_expert`` counters are summed over ``group`` (one all-reduce for all layers; pass every rank
    that holds the same layers), ``b_e += update_rate * sign(mean(c) - c_e)`` is applied to the fp32 master of each bias,
    and the counters are reset.  Only the sign of the imbalance matters, so counting every token a uniform number of times
    (activation recomputation, tensor-parallel ranks that all route the same tokens) changes nothing.  Layers without a
    bias are left alone.
    """
    layers = expert_bias_layers(modules)
    if not layers:
        return
    counts = torch.cat([layer.tokens_per_expert for layer in layers])
    if dist.is_available() and dist.is_initialized():
        dist.all_reduce(counts, op=dist.ReduceOp.SUM, group=group)
    offset = 0
    for layer in layers:
        n = layer.tokens_per_expert.numel()
        c = counts[offset:offset + n].double()
        offset += n
        master = expert_bias_master(layer)
        master.add_(torch.sign(c.mean() - c).float(), alpha=update_rate)
        layer.router.expert_bias.copy_(master)
        layer.reset_stats()


__all__ = ["expert_bias_layers", "expert_bias_master", "update_expert_bias"]

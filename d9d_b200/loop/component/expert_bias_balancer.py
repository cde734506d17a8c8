from __future__ import annotations

from typing import Any

import torch
from torch.distributed import ProcessGroup

from d9d_b200.core.dist_context import BATCH_DOMAIN, DistributedContext
from d9d_b200.loop.config import ExpertBiasBalancingConfig
from d9d_b200.module.block.moe import MoELayer
from d9d_b200.module.block.moe.balancing import expert_bias_master, update_expert_bias

from .model_stage_factory import TrackedModules


class ExpertBiasBalancer:
    """Auxiliary-loss-free load balancing of the local pipeline stages' MoE routers (``update_expert_bias``).

    Selection counts are summed over every rank that holds the same stage (data, context, tensor and expert ranks); each
    stage balances its own layers.  The fp32 master copies of the biases are part of the job checkpoint, so a resumed run
    continues the exact trajectory even when the bias buffers are bf16."""

    def __init__(self, dist_context: DistributedContext, tracked_modules: TrackedModules, config: ExpertBiasBalancingConfig):
        self._modules = tracked_modules.modules
        self._config = config
        self._group: ProcessGroup | None = None
        if dist_context.mesh_params.is_distributed:
            stage_ranks = dist_context.mesh_for(BATCH_DOMAIN)["dp", "cp", "tp"]
            self._group = stage_ranks._flatten().get_group()  # noqa: SLF001
        self._layers = {f"{stage}.{name}": layer for stage, module in enumerate(self._modules)
                        for name, layer in module.named_modules()
                        if isinstance(layer, MoELayer) and layer.router.expert_bias is not None}

    def reset_counters(self) -> None:
        """Start counting a new step's selections (call before its first forward)."""
        for layer in self._layers.values():
            layer.reset_stats()

    def update(self) -> None:
        """One balancing step from the selections counted since ``reset_counters`` (call after the optimizer step)."""
        update_expert_bias(self._modules, self._config.update_rate, self._group)

    def state_dict(self) -> dict[str, Any]:
        return {"masters": {name: expert_bias_master(layer) for name, layer in self._layers.items()}}

    def load_state_dict(self, state_dict: dict[str, Any]) -> None:
        for name, layer in self._layers.items():
            master = expert_bias_master(layer)
            master.copy_(state_dict["masters"][name])
            with torch.no_grad():
                layer.router.expert_bias.copy_(master)

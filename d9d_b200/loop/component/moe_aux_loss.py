from __future__ import annotations

import torch
import torch.distributed as dist

from d9d_b200.core.dist_context import DistributedContext
from d9d_b200.loop.config import MoEAuxLossConfig
from d9d_b200.loop.control import LOSS_WEIGHT_PER_TOKEN
from d9d_b200.module.block.moe import MoELayer
from d9d_b200.tracker import BaseTrackerRun

from .model_stage_factory import TrackedModules


class MoEAuxLoss:
    """Trains the local pipeline stages' softmax MoE routers with the load-balancing and router z auxiliary losses
    (``TopKRouter.set_aux_loss``) and logs them.

    The gradients are added inside each router's backward, so pipelining, split backward, activation recomputation and
    expert parallelism need nothing more.  The logged values are the token-weighted means over the step's MoE layers,
    microbatches and ranks: ``moe_load_balancing_loss = sum w T A / sum w T`` and ``moe_router_z_loss = sum w T Z /
    sum w T``, from one all-reduce of three floats over every rank (pipeline stages included) on the steps the job
    logger is due.  Nothing is checkpointed: the sums restart every step."""

    def __init__(self, dist_context: DistributedContext, tracked_modules: TrackedModules, config: MoEAuxLossConfig):
        self._device = dist_context.current_device
        self._distributed = dist_context.mesh_params.is_distributed
        self._layers = [layer for module in tracked_modules.modules for layer in module.modules() if isinstance(layer, MoELayer)]
        for layer in self._layers:
            layer.router.set_aux_loss(config.load_balancing_coef, config.z_loss_coef, LOSS_WEIGHT_PER_TOKEN)

    def reset(self) -> None:
        """Start a new step's sums (call before its first forward)."""
        for layer in self._layers:
            layer.router.reset_aux_loss_sums()

    def log(self, run: BaseTrackerRun) -> None:
        """Log the step's values (call after the step's last backward, on every rank, when the job logger is due)."""
        sums = torch.zeros(3, dtype=torch.float32, device=self._device)
        for layer in self._layers:
            sums += layer.router.aux_loss_sums.to(self._device)
        if self._distributed and dist.is_initialized():
            dist.all_reduce(sums)
        lb, z, weight = sums.tolist()
        if weight > 0:
            run.scalar("moe_load_balancing_loss", lb / weight)
            run.scalar("moe_router_z_loss", z / weight)

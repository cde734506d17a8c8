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
    (``TopKRouter.set_aux_loss``), and softmax or sigmoid routers with the sequence-wise balance loss
    (``TopKRouter.set_sequence_balance_loss``), and logs them.

    The gradients are added inside each router's backward, so pipelining, split backward, activation recomputation and
    expert parallelism need nothing more.  The logged values are the token-weighted means over the step's MoE layers,
    microbatches and ranks: ``moe_load_balancing_loss = sum w T A / sum w T`` and ``moe_router_z_loss = sum w T Z /
    sum w T`` and ``moe_sequence_balance_loss = sum w S sum_b A_b / sum w T``, from one all-reduce of five floats over
    every rank (pipeline stages included) on the steps the job logger is due.  Nothing is checkpointed: the sums restart
    every step.

    The sequence-wise loss needs each MoE layer's input to hold whole sequences, so context-parallel and tensor-parallel
    (sequence-parallel) meshes are refused; expert and pipeline parallelism route whole local sequences before dispatch."""

    def __init__(self, dist_context: DistributedContext, tracked_modules: TrackedModules, config: MoEAuxLossConfig):
        mesh = dist_context.mesh_params
        if config.sequence_balance_coef > 0 and (mesh.context_parallel_replicate > 1 or mesh.context_parallel_shard > 1
                                                 or mesh.tensor_parallel > 1):
            raise ValueError("the sequence-wise balance loss needs whole sequences on every rank: it does not support "
                             "context_parallel_replicate, context_parallel_shard or tensor_parallel > 1")
        self._device = dist_context.current_device
        self._distributed = mesh.is_distributed
        self._layers = [layer for module in tracked_modules.modules for layer in module.modules() if isinstance(layer, MoELayer)]
        for layer in self._layers:
            layer.router.set_aux_loss(config.load_balancing_coef, config.z_loss_coef, LOSS_WEIGHT_PER_TOKEN)
            layer.router.set_sequence_balance_loss(config.sequence_balance_coef, LOSS_WEIGHT_PER_TOKEN)

    def reset(self) -> None:
        """Start a new step's sums (call before its first forward)."""
        for layer in self._layers:
            layer.router.reset_aux_loss_sums()

    def log(self, run: BaseTrackerRun) -> None:
        """Log the step's values (call after the step's last backward, on every rank, when the job logger is due)."""
        sums = torch.zeros(5, dtype=torch.float32, device=self._device)
        for layer in self._layers:
            sums[:3] += layer.router.aux_loss_sums.to(self._device)
            sums[3:] += layer.router.sequence_balance_sums.to(self._device)
        if self._distributed and dist.is_initialized():
            dist.all_reduce(sums)
        lb, z, weight, seq, seq_weight = sums.tolist()
        if weight > 0:
            run.scalar("moe_load_balancing_loss", lb / weight)
            run.scalar("moe_router_z_loss", z / weight)
        if seq_weight > 0:
            run.scalar("moe_sequence_balance_loss", seq / seq_weight)

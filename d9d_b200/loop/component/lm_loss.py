from __future__ import annotations

import torch
import torch.distributed as dist

from d9d_b200.core.dist_context import DistributedContext
from d9d_b200.loop.config import LMLossConfig
from d9d_b200.module.block.head import SplitLanguageModellingHead
from d9d_b200.tracker import BaseTrackerRun

from .model_stage_factory import TrackedModules


class LMLoss:
    """Trains the local pipeline stages' LM heads with label smoothing and the z-loss
    (``SplitLanguageModellingHead.set_loss_regularisation``), and logs the plain NLL and ``lse^2``.

    The regularised loss and its gradient come from the fused linear cross-entropy, so the task's loss, pipelining and
    recomputation need nothing more.  The logged values are token means over the step's microbatches and ranks:
    ``lm_nll = sum nll / n`` (the unsmoothed NLL) and ``lm_z_loss = sum lse^2 / n`` (unscaled by ``z_loss_coef``), from
    one all-reduce of three floats over every rank (pipeline stages included) on the steps the job logger is due.
    Nothing is checkpointed: the sums restart every step."""

    def __init__(self, dist_context: DistributedContext, tracked_modules: TrackedModules, config: LMLossConfig):
        self._device = dist_context.current_device
        self._distributed = dist_context.mesh_params.is_distributed
        self._heads: list[SplitLanguageModellingHead] = []
        for module in tracked_modules.modules:
            heads = [m for m in module.modules() if isinstance(m, SplitLanguageModellingHead)]
            stage = getattr(module, "_stage", None)
            if stage is not None and stage.is_current_stage_last and not heads:
                raise ValueError(f"lm_loss is set, but the last pipeline stage ({type(module).__name__}) has no LM head")
            self._heads += heads
        for head in self._heads:
            head.set_loss_regularisation(config.label_smoothing, config.z_loss_coef)

    def reset(self) -> None:
        """Start a new step's sums (call before its first forward)."""
        for head in self._heads:
            head.reset_loss_sums()

    def log(self, run: BaseTrackerRun) -> None:
        """Log the step's values (call after the step's last backward, on every rank, when the job logger is due)."""
        sums = torch.zeros(3, dtype=torch.float32, device=self._device)
        for head in self._heads:
            sums += head.lm_loss_sums.to(self._device)
        if self._distributed and dist.is_initialized():
            dist.all_reduce(sums)
        nll, lse2, count = sums.tolist()
        if count > 0:
            run.scalar("lm_nll", nll / count)
            run.scalar("lm_z_loss", lse2 / count)

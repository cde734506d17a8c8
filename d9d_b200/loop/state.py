"""Aggregated job state (everything the loops need + what gets checkpointed).

Checkpoint key tree (reference ``d9d/loop/state.py:64-118``): ``stepper``, ``tracked_modules``, ``data_loader`` and,
for training, ``logger``, ``task``, ``metrics``, ``optimizer``, ``lr_scheduler`` (+ ``expert_bias_balancer`` when expert-bias
balancing is on).
"""

from __future__ import annotations

import dataclasses
from typing import Any

from torch.distributed.checkpoint.stateful import Stateful
from torchdata.stateful_dataloader import StatefulDataLoader

from d9d_b200.core.dist_context import DistributedContext
from d9d_b200.core.protocol import LRSchedulerProtocol, OptimizerProtocol
from d9d_b200.loop.component import (
    BatchMaths,
    ExpertBiasBalancer,
    MoEAuxLoss,
    LMLoss,
    GradientClipper,
    GradientManager,
    InferenceTaskOperator,
    JobLogger,
    JobProfiler,
    ManualGarbageCollector,
    ModelStageExporter,
    StateCheckpointer,
    Stepper,
    TimeoutManager,
    TrackedModules,
    TrainTaskOperator,
)
from d9d_b200.loop.control import InferenceTask, TrainTask
from d9d_b200.loop.event import EventBus
from d9d_b200.metric.impl.container import ComposeMetric


class _CheckpointedFields(Stateful):
    """``state_dict`` / ``load_state_dict`` derived from ``CHECKPOINTED``: the names of the fields that are Stateful and
    belong in a job checkpoint (subclasses extend the tuple).  Optional fields that are ``None`` are left out."""

    CHECKPOINTED: tuple[str, ...] = ()

    def state_dict(self) -> dict[str, Any]:
        return {name: getattr(self, name).state_dict() for name in self.CHECKPOINTED if getattr(self, name) is not None}

    def load_state_dict(self, state_dict: dict[str, Any]) -> None:
        for name in self.CHECKPOINTED:
            if getattr(self, name) is not None:
                getattr(self, name).load_state_dict(state_dict[name])


@dataclasses.dataclass(kw_only=True)
class JobState(_CheckpointedFields):
    """What training and inference jobs share."""

    CHECKPOINTED = ("stepper", "tracked_modules", "data_loader")

    dist_context: DistributedContext
    event_bus: EventBus
    stepper: Stepper
    tracked_modules: TrackedModules
    data_loader: StatefulDataLoader
    batch_maths: BatchMaths
    checkpointer: StateCheckpointer
    garbage_collector: ManualGarbageCollector
    profiler: JobProfiler
    timeout_manager: TimeoutManager


@dataclasses.dataclass(kw_only=True)
class TrainJobState(JobState):
    CHECKPOINTED = (*JobState.CHECKPOINTED, "logger", "task", "metrics", "optimizer", "lr_scheduler", "expert_bias_balancer")

    task: TrainTask
    task_operator: TrainTaskOperator
    metrics: ComposeMetric
    logger: JobLogger
    optimizer: OptimizerProtocol
    lr_scheduler: LRSchedulerProtocol
    gradient_manager: GradientManager
    gradient_clipper: GradientClipper
    exporter: ModelStageExporter
    expert_bias_balancer: ExpertBiasBalancer | None = None
    moe_aux_loss: MoEAuxLoss | None = None  # not checkpointed: its sums restart every step
    lm_loss: LMLoss | None = None  # not checkpointed: its sums restart every step


@dataclasses.dataclass(kw_only=True)
class InferenceJobState(JobState):
    CHECKPOINTED = (*JobState.CHECKPOINTED, "task")

    task: InferenceTask
    task_operator: InferenceTaskOperator

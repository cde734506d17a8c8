from __future__ import annotations

import abc
import dataclasses
from collections.abc import Mapping
from typing import TYPE_CHECKING, Any, Generic, Protocol, TypeVar, runtime_checkable

import torch
from torch.distributed.checkpoint.stateful import Stateful

from d9d_b200.core.dist_context import DistributedContext
from d9d_b200.core.types import ScalarTree
from d9d_b200.loop.event import EventBus
from d9d_b200.pipelining.api import PipelineShardingSpec

if TYPE_CHECKING:
    from d9d_b200.internals.pipeline_state import PipelineState
    from d9d_b200.loop.component import Stepper
    from d9d_b200.metric import Metric

TBatch = TypeVar("TBatch")


@dataclasses.dataclass(kw_only=True)
class BuildForwardInputsContext(Generic[TBatch]):
    batch: TBatch
    state: "PipelineState"  # scratch shared with compute_loss / update_metrics of the same step


@dataclasses.dataclass(kw_only=True)
class BuildForwardInputsResult:
    inputs: dict[str, torch.Tensor]  # first pipeline stage only
    kwargs: dict[str, Any]  # every pipeline stage
    pipeline_sharding_spec: PipelineShardingSpec | None = None


@dataclasses.dataclass(kw_only=True)
class RegisterTaskEventsContext:
    dist_context: DistributedContext
    event_bus: EventBus


@dataclasses.dataclass(kw_only=True)
class FinalizeContext:
    pass


class BaseTask(abc.ABC, Stateful, Generic[TBatch]):
    @abc.abstractmethod
    def build_forward_inputs(self, ctx: BuildForwardInputsContext[TBatch]) -> BuildForwardInputsResult: ...

    def state_dict(self) -> dict[str, Any]:
        return {}

    def load_state_dict(self, state_dict: dict[str, Any]) -> None:  # noqa: B027
        """Stateless by default."""

    def register_events(self, context: RegisterTaskEventsContext) -> None:  # noqa: B027
        """Optional: subscribe to loop events."""

    def finalize(self, ctx: FinalizeContext) -> None:  # noqa: B027
        """Called once after the loop finished."""


@dataclasses.dataclass(kw_only=True)
class ComputeLossContext:
    pipeline_results: Mapping[str, torch.Tensor]
    state: "PipelineState"
    stepper: "Stepper"


# Loss weight of one token: ``CausalLMTask`` weighs a microbatch of ``n`` target tokens ``n * LOSS_WEIGHT_PER_TOKEN``, and
# the MoE routers' auxiliary losses weigh a forward of ``T`` tokens ``T * LOSS_WEIGHT_PER_TOKEN``, so both are
# token-weighted means in the same units.
LOSS_WEIGHT_PER_TOKEN = 1 / 1000


@dataclasses.dataclass(kw_only=True)
class ComputeLossResult:
    loss: torch.Tensor
    loss_weight: torch.Tensor | None  # None == 1.0; gradients are normalised by the global sum of weights


@dataclasses.dataclass(kw_only=True)
class CreateMetricsContext:
    pass


@dataclasses.dataclass(kw_only=True)
class CreateMetricsResult:
    metrics: dict[str, "Metric"]


@dataclasses.dataclass(kw_only=True)
class UpdateMetricsContext:
    state: "PipelineState"
    metrics: Mapping[str, "Metric"]


class TrainTask(BaseTask, abc.ABC, Generic[TBatch]):
    @abc.abstractmethod
    def compute_loss(self, ctx: ComputeLossContext) -> ComputeLossResult: ...

    def create_metrics(self, ctx: CreateMetricsContext) -> CreateMetricsResult:
        return CreateMetricsResult(metrics={})

    def update_metrics(self, ctx: UpdateMetricsContext) -> None:  # noqa: B027
        """Optional."""

    def dump_hparams(self) -> ScalarTree:
        return {}


@dataclasses.dataclass(kw_only=True)
class TrainTaskProviderContext:
    dist_context: DistributedContext


@runtime_checkable
class TrainTaskProvider(Protocol):
    def __call__(self, ctx: TrainTaskProviderContext) -> TrainTask: ...


@dataclasses.dataclass(kw_only=True)
class ProcessOutputsContext:
    pipeline_results: dict[str, torch.Tensor]
    state: "PipelineState"


class InferenceTask(BaseTask, abc.ABC, Generic[TBatch]):
    @abc.abstractmethod
    def process_outputs(self, ctx: ProcessOutputsContext) -> None: ...


@dataclasses.dataclass(kw_only=True)
class InferenceTaskProviderContext:
    dist_context: DistributedContext


@runtime_checkable
class InferenceTaskProvider(Protocol):
    def __call__(self, ctx: InferenceTaskProviderContext) -> InferenceTask: ...

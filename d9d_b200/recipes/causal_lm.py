"""Causal-LM pre-training / evaluation building blocks.

The same roles as the user code of the reference's ``example/qwen3_moe/pretrain.py`` (dataset provider, model
provider, SFT task), packaged so that the example script, the benchmark and the tests share one implementation.
"""

from __future__ import annotations

from typing import Literal

import torch
from pydantic import BaseModel

from d9d_b200.core.dist_context import DistributedContext
from d9d_b200.core.types import ScalarTree
from d9d_b200.dataset import SyntheticTokenDataset, shard_batch_along_sequence, shard_dataset_data_parallel
from d9d_b200.loop.control import (
    LOSS_WEIGHT_PER_TOKEN,
    BuildForwardInputsContext,
    BuildForwardInputsResult,
    ComputeLossContext,
    ComputeLossResult,
    CreateMetricsContext,
    CreateMetricsResult,
    DatasetProvider,
    InferenceTask,
    InitializeDatasetContext,
    InitializeDatasetResult,
    InitializeModelStageContext,
    InitializeModelStageResult,
    ModelProvider,
    ParallelizeModelStageContext,
    PrepareExportModelStageContext,
    PrepareExportModelStageResult,
    ProcessOutputsContext,
    TrainTask,
    UpdateMetricsContext,
)
from d9d_b200.metric.impl.aggregation import SumMetric
from d9d_b200.model_state.mapper.adapters import identity_mapper_from_module, restrict_mapper_to_module
from d9d_b200.module.block.head import LM_IGNORE_INDEX
from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode
from d9d_b200.module.model.qwen3_moe import (
    Qwen3MoEExpertsFormat,
    Qwen3MoEForCausalLM,
    Qwen3MoEForCausalLMParameters,
    mapper_from_huggingface_qwen3_moe_for_causal_lm,
    mapper_to_huggingface_qwen3_moe_for_causal_lm,
)
from d9d_b200.module.parallelism.model.qwen3_moe import parallelize_qwen3_moe_for_causal_lm


class SyntheticDataConfig(BaseModel):
    num_samples: int
    seq_len: int
    vocab_size: int
    seed: int = 0
    learnable: bool = False


class SyntheticDataProvider(DatasetProvider):
    """Fixed-length random token samples (``input_ids`` / next-token ``labels`` / ``position_ids``), sharded over the
    data-parallel ranks.  There is no network in CI, so this stands in for a tokenised corpus."""

    def __init__(self, config: SyntheticDataConfig):
        self._config = config

    def __call__(self, context: InitializeDatasetContext) -> InitializeDatasetResult:
        c = self._config
        data = SyntheticTokenDataset(c.num_samples, c.seq_len, c.vocab_size, seed=c.seed, learnable=c.learnable)
        return InitializeDatasetResult(dataset=shard_dataset_data_parallel(data, context.dist_context),
                                       collator=SyntheticTokenDataset.collate)


class Qwen3MoEModelProviderConfig(BaseModel):
    model: Qwen3MoEForCausalLMParameters
    checkpointing: bool = False
    dtype: str = "bfloat16"
    # layout of ``model_stage_factory.source_checkpoint`` and of ``Trainer.export``: this framework's own parameter names
    # or HuggingFace ``Qwen3MoeForCausalLM`` (``experts_format``: fused 3-D expert tensors of transformers 5, or one
    # ``nn.Linear`` per expert of transformers 4)
    checkpoint_format: Literal["native", "huggingface"] = "native"
    experts_format: Qwen3MoEExpertsFormat = Qwen3MoEExpertsFormat.FUSED


class Qwen3MoEModelProvider(ModelProvider):
    def __init__(self, config: Qwen3MoEModelProviderConfig):
        self._config = config

    def initialize_model_stage(self, context: InitializeModelStageContext) -> InitializeModelStageResult:
        model = Qwen3MoEForCausalLM(self._config.model, context.stage, HiddenStatesAggregationMode.no,
                                    self._config.checkpointing).to(getattr(torch, self._config.dtype))
        if self._config.checkpoint_format == "huggingface":
            # the whole-model mapper, cut down to the parameters this pipeline stage holds
            whole = mapper_from_huggingface_qwen3_moe_for_causal_lm(self._config.model, self._config.experts_format)
            return InitializeModelStageResult(model=model, state_mapper=restrict_mapper_to_module(whole, model, module_keys_are="outputs"))
        return InitializeModelStageResult(model=model, state_mapper=identity_mapper_from_module(model))

    def parallelize_model_stage(self, context: ParallelizeModelStageContext) -> None:
        parallelize_qwen3_moe_for_causal_lm(context.dist_context, context.model, context.stage)

    def prepare_export_model_stage(self, context: PrepareExportModelStageContext) -> PrepareExportModelStageResult:
        if self._config.checkpoint_format == "huggingface":
            whole = mapper_to_huggingface_qwen3_moe_for_causal_lm(self._config.model, self._config.experts_format)
            return PrepareExportModelStageResult(state_mapper=restrict_mapper_to_module(whole, context.model,
                                                                                        module_keys_are="inputs"))
        return PrepareExportModelStageResult(state_mapper=identity_mapper_from_module(context.model))

    def dump_hparams(self) -> ScalarTree:
        return self._config.model_dump(mode="json")


class CausalLMTask(TrainTask):
    """Token-mean next-token loss; the loss weight is the number of target tokens (so gradient accumulation and
    data parallelism produce the exact global token mean).  Given the distributed context, batches are cut along the
    sequence for context-parallel meshes (every ``cp`` rank keeps ``S / cp`` tokens of each sample)."""

    def __init__(self, dist_context: DistributedContext | None = None) -> None:
        self._ctx = dist_context

    def build_forward_inputs(self, ctx: BuildForwardInputsContext) -> BuildForwardInputsResult:
        batch = ctx.batch if self._ctx is None else shard_batch_along_sequence(ctx.batch, self._ctx)
        ctx.state["labels"] = batch["labels"]
        return BuildForwardInputsResult(
            inputs={"input_ids": batch["input_ids"]},
            kwargs={"labels": batch["labels"], "position_ids": batch["position_ids"]},
        )

    def create_metrics(self, ctx: CreateMetricsContext) -> CreateMetricsResult:
        return CreateMetricsResult(metrics={"num_tokens": SumMetric()})

    def update_metrics(self, ctx: UpdateMetricsContext) -> None:
        ctx.metrics["num_tokens"].update(ctx.state["num_tokens"])

    def compute_loss(self, ctx: ComputeLossContext) -> ComputeLossResult:
        num_tokens = (ctx.state["labels"] != LM_IGNORE_INDEX).sum()
        ctx.state["num_tokens"] = num_tokens
        # a context-parallel rank may hold no target token of a microbatch: its loss is 0 with weight 0.  The count is
        # divided by 1 / LOSS_WEIGHT_PER_TOKEN (exactly 1000.0): each weight is the correctly rounded fp32 n / 1000
        return ComputeLossResult(loss=ctx.pipeline_results["logps"].sum() / num_tokens.clamp_min(1),
                                 loss_weight=num_tokens / (1 / LOSS_WEIGHT_PER_TOKEN))


class CausalLMPerplexityTask(InferenceTask):
    """Accumulates summed negative log-likelihood and token counts; ``perplexity()`` after the run.

    The running sums are part of the job checkpoint (keyed by rank: every rank holding a last pipeline stage accumulates
    its own share), so an interrupted evaluation resumes without losing what was already scored."""

    def __init__(self, dist_context: DistributedContext | None = None) -> None:
        self._ctx = dist_context
        self.nll_sum = 0.0
        self.num_tokens = 0

    def build_forward_inputs(self, ctx: BuildForwardInputsContext) -> BuildForwardInputsResult:
        batch = ctx.batch if self._ctx is None else shard_batch_along_sequence(ctx.batch, self._ctx)
        ctx.state["labels"] = batch["labels"]
        return BuildForwardInputsResult(
            inputs={"input_ids": batch["input_ids"]},
            kwargs={"labels": batch["labels"], "position_ids": batch["position_ids"]},
        )

    def process_outputs(self, ctx: ProcessOutputsContext) -> None:
        self.nll_sum += float(ctx.pipeline_results["logps"].sum())
        self.num_tokens += int((ctx.state["labels"] != LM_IGNORE_INDEX).sum())

    def _key(self) -> str:
        return f"rank_{self._ctx.global_rank if self._ctx is not None else 0}"

    def state_dict(self) -> dict[str, torch.Tensor]:
        return {self._key(): torch.tensor([self.nll_sum, float(self.num_tokens)], dtype=torch.float64)}

    def load_state_dict(self, state_dict: dict[str, torch.Tensor]) -> None:
        sums = state_dict[self._key()]
        self.nll_sum, self.num_tokens = float(sums[0]), int(sums[1])

    def perplexity(self) -> float:
        return float(torch.tensor(self.nll_sum / max(self.num_tokens, 1)).exp())

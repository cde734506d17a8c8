from __future__ import annotations

import itertools
from collections.abc import Callable
from typing import Any

import torch
from torch import nn
from torch.distributed.checkpoint.stateful import Stateful

from d9d_b200.core.dist_context import REGULAR_DOMAIN, DistributedContext
from d9d_b200.loop.config import ModelStageFactoryConfig, PipeliningConfig
from d9d_b200.loop.control import InitializeModelStageContext, ModelProvider, ParallelizeModelStageContext
from d9d_b200.model_state.io import load_model_state
from d9d_b200.module.base import ModuleLateInit
from d9d_b200.pipelining.api import PipelineStageInfo
from d9d_b200.pipelining.factory import PipelineScheduleInfo, build_schedule

from .batch_maths import BatchMaths
from .pipeline_result_processing import PipelineOutputsProcessor

StatefulPredicate = Callable[[str, torch.Tensor], bool]


class TrackedModules(Stateful):
    """The model stages owned by this rank as one checkpointable object: keys ``pp_{pp_rank}_stage_{i}.<fqn>``,
    restricted to tensors accepted by the predicate (all, or only ``requires_grad`` ones for PEFT)."""

    def __init__(self, dist_context: DistributedContext, modules: list[nn.Module], stateful_predicate: StatefulPredicate):
        self._pp_rank = dist_context.mesh_for(REGULAR_DOMAIN)["pp"].get_local_rank() if dist_context.mesh_params.is_distributed else 0
        self._modules = modules
        self._predicate = stateful_predicate

    @property
    def modules(self) -> list[nn.Module]:
        return self._modules

    def _allowed(self, module: nn.Module) -> set[str]:
        return {n for n, t in itertools.chain(module.named_parameters(), module.named_buffers()) if self._predicate(n, t)}

    def state_dict(self) -> dict[str, Any]:
        out = {}
        for i, module in enumerate(self._modules):
            allowed = self._allowed(module)
            out[f"pp_{self._pp_rank}_stage_{i}"] = {k: v for k, v in module.state_dict().items() if k in allowed}
        return out

    def load_state_dict(self, state_dict: dict[str, Any]) -> None:
        for i, module in enumerate(self._modules):
            allowed = self._allowed(module)
            result = module.load_state_dict(state_dict[f"pp_{self._pp_rank}_stage_{i}"], strict=False)
            missing = allowed & set(result.missing_keys)
            if missing:
                raise ValueError(f"Missing keys: {missing}")
            if result.unexpected_keys:
                raise ValueError(f"Extra keys: {set(result.unexpected_keys)}")


class ModelStageFactory:
    """meta-init -> parallelise -> materialise on the device -> ``reset_parameters`` -> optional checkpoint load,
    for every stage the schedule places on this rank (reference ``model_stage_factory.py:150-214``)."""

    def __init__(self, model_provider: ModelProvider, dist_context: DistributedContext, batch_maths: BatchMaths,
                 config_model: ModelStageFactoryConfig, config_pipelining: PipeliningConfig,
                 pipeline_callback: PipelineOutputsProcessor):
        self._provider = model_provider
        self._ctx = dist_context
        self._maths = batch_maths
        self._config_model = config_model
        self._config_pipelining = config_pipelining
        self._callback = pipeline_callback

    def _build_model_stage(self, stage: PipelineStageInfo) -> nn.Module:
        with torch.device("meta"):
            built = self._provider.initialize_model_stage(InitializeModelStageContext(dist_context=self._ctx, stage=stage))
        model = built.model
        if not isinstance(model, nn.Module) or not isinstance(model, ModuleLateInit):
            raise ValueError("Model stage is required to be nn.Module instance implementing ModuleLateInit protocol")
        self._apply_fp8(model)
        self._apply_fp8_experts(model)
        if self._ctx.mesh_params.is_distributed:
            self._provider.parallelize_model_stage(ParallelizeModelStageContext(model=model, stage=stage, dist_context=self._ctx))
        model.to_empty(device=self._ctx.current_device)
        with torch.no_grad():
            model.reset_parameters()
        if self._config_model.source_checkpoint:
            load_model_state(src_dir=self._config_model.source_checkpoint, mapper=built.state_mapper,
                             device=str(self._ctx.current_device), model=model, position=self._ctx.local_rank)
        model.train()
        return model

    def _apply_fp8(self, model: nn.Module) -> None:
        cfg = self._config_model.fp8_linear
        if cfg is None:
            return
        if self._ctx.mesh_params.tensor_parallel > 1:
            raise NotImplementedError("model_stage_factory.fp8_linear is not combined with tensor parallelism (the fused TP GEMMs are bf16)")
        import re

        from d9d_b200.kernel.fp8 import convert_linears_to_fp8

        include, exclude = re.compile(cfg.include), re.compile(cfg.exclude) if cfg.exclude else None
        n = convert_linears_to_fp8(model, lambda name, _m: bool(include.search(name)) and not (exclude and exclude.search(name)),
                                   recipe=cfg.recipe)
        self._ctx.logger.info(f"fp8: {n} linear layers of this stage run in e4m3")

    def _apply_fp8_experts(self, model: nn.Module) -> None:
        if not self._config_model.fp8_experts:
            return
        if self._ctx.mesh_params.tensor_parallel > 1:
            raise NotImplementedError("model_stage_factory.fp8_experts is not combined with tensor parallelism")
        from d9d_b200.module.block.moe import GroupedSwiGLU

        recipe = self._config_model.fp8_experts_recipe
        blocks = [m for m in model.modules() if isinstance(m, GroupedSwiGLU)]
        for block in blocks:
            block.enable_fp8(recipe)  # refuses LoRA-wrapped projections and sizes that are not multiples of 16
        self._ctx.logger.info(f"fp8: {len(blocks)} expert blocks of this stage run in e4m3 ({recipe})")

    def build_pipeline_and_modules(self) -> tuple[PipelineScheduleInfo, TrackedModules]:
        if self._config_model.checkpoint_only_trainable_parameters:
            predicate: StatefulPredicate = lambda _name, t: t.requires_grad  # noqa: E731
        else:
            predicate = lambda _name, _t: True  # noqa: E731
        schedule, modules = build_schedule(dist_context=self._ctx, n_microbatches=self._maths.num_microbatches_pipelining,
                                           schedule_config=self._config_pipelining.schedule,
                                           model_provider=self._build_model_stage, callback=self._callback)
        return schedule, TrackedModules(self._ctx, modules, predicate)

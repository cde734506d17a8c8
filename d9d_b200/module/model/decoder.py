"""Family-independent decoder-only backbone and task heads.

The reference duplicates ~550 lines per family (``d9d/module/model/qwen3_dense/model.py`` and
``qwen3_moe/model.py`` differ only in the layer class).  Here a family is *(params, layer factory)* plugged into
shared classes; the forward/pipelining contracts are the reference's:

* inputs by keyword; stage 0 gets ``input_ids [B,S]``, later stages ``hidden_states [B,S,H]`` (+ snapshot);
  every stage gets ``position_ids`` (+ ``labels`` / ``pooling_mask`` / ``hidden_states_agg_mask``);
* output is a dict; layers are stored in a ``ModuleDict`` keyed by *global* layer index so state-dict names are
  independent of the pipeline split; optional per-layer activation checkpointing.
"""

from __future__ import annotations

import inspect
from collections.abc import Callable
from typing import Any, Protocol

import torch
from torch import nn
from torch.utils.checkpoint import checkpoint

from d9d_b200.module.base import ModuleLateInit
from d9d_b200.module.block.embedding import SplitTokenEmbeddings
from d9d_b200.module.block.head import ClassificationHead, EmbeddingHead, SplitLanguageModellingHead
from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode, create_hidden_states_aggregator
from d9d_b200.module.block.normalization import RMSNorm
from d9d_b200.module.block.positional import RopeScaling, RotaryEmbeddingProvider, RotaryEmbeddingStyle
from d9d_b200.pipelining.api import ModuleSupportsPipelining, PipelineStageInfo, distribute_layers_for_pipeline_stage


class _LayerParams(Protocol):
    hidden_size: int
    rms_norm_eps: float
    head_dim: int


class _BackboneParams(Protocol):
    layer: Any
    num_hidden_layers: int
    rope_base: int
    max_position_ids: int
    split_vocab_size: dict[str, int]
    split_vocab_order: list[str]
    pipeline_num_virtual_layers_pre: int
    pipeline_num_virtual_layers_post: int


class DecoderBackbone(nn.Module, ModuleLateInit, ModuleSupportsPipelining):
    """Embeddings (first stage) -> this stage's decoder layers -> final RMSNorm (last stage)."""

    def __init__(
        self,
        params: _BackboneParams,
        stage: PipelineStageInfo,
        hidden_states_snapshot_mode: HiddenStatesAggregationMode,
        enable_checkpointing: bool,
        layer_factory: Callable[..., nn.Module],
        rope_style: RotaryEmbeddingStyle = RotaryEmbeddingStyle.HALF,
        rope_scaling: RopeScaling | None = None,
        zero_centered_norm: bool = False,
    ):
        super().__init__()
        hidden = params.layer.hidden_size
        if stage.is_current_stage_first:
            self.embed_tokens = SplitTokenEmbeddings(
                split_vocab_size=params.split_vocab_size, split_order=params.split_vocab_order, hidden_size=hidden
            )
        first, last = distribute_layers_for_pipeline_stage(
            num_layers=params.num_hidden_layers,
            num_virtual_layers_pre=params.pipeline_num_virtual_layers_pre,
            num_virtual_layers_post=params.pipeline_num_virtual_layers_post,
            stage=stage,
        )
        self._num_layers_before = first
        self._layer_keys = [str(i) for i in range(first, last)]
        # heterogeneous stacks (e.g. dense first layers, MoE afterwards) take the global layer index as second argument
        indexed = len(inspect.signature(layer_factory).parameters) >= 2
        self.layers = nn.ModuleDict({key: (layer_factory(params.layer, int(key)) if indexed else layer_factory(params.layer))
                                     for key in self._layer_keys})
        self.rope_provider = RotaryEmbeddingProvider(
            # families with partial rotary embeddings expose the rotated width as ``layer.rope_dim``
            rope_base=params.rope_base, head_dim=getattr(params.layer, "rope_dim", params.layer.head_dim),
            max_position_ids=params.max_position_ids,
            style=rope_style, rope_scaling=rope_scaling,
        )
        if stage.is_current_stage_last:
            self.norm = RMSNorm(hidden, eps=params.layer.rms_norm_eps, zero_centered=zero_centered_norm)
        self._stage = stage
        self._snapshot_mode = hidden_states_snapshot_mode
        self._hidden_size = hidden
        self._enable_checkpointing = enable_checkpointing

    def output_dtype(self) -> torch.dtype:
        return self.layers[self._layer_keys[0]].input_layernorm.weight.dtype

    def forward(
        self,
        input_ids: torch.Tensor | None = None,
        hidden_states: torch.Tensor | None = None,
        position_ids: torch.Tensor | None = None,
        hidden_states_snapshot: torch.Tensor | None = None,
        hidden_states_agg_mask: torch.Tensor | None = None,
    ) -> dict[str, torch.Tensor | None]:
        aggregator = create_hidden_states_aggregator(self._snapshot_mode, hidden_states_agg_mask)
        if input_ids is not None:
            x = self.embed_tokens(input_ids)
            aggregator.add_hidden_states(x)
        else:
            x = hidden_states
        rope = self.rope_provider(position_ids)
        for key in self._layer_keys:
            layer = self.layers[key]
            if self._enable_checkpointing:
                x = checkpoint(layer, x, rope, use_reentrant=False)
            else:
                x = layer(x, rope)
            aggregator.add_hidden_states(x)
        if self._stage.is_current_stage_last:
            x = self.norm(x)
        return {"hidden_states": x, "hidden_states_snapshot": aggregator.pack_with_snapshot(hidden_states_snapshot)}

    def reset_parameters(self) -> None:
        if self._stage.is_current_stage_first:
            self.embed_tokens.reset_parameters()
        self.rope_provider.reset_parameters()
        for key in self._layer_keys:
            self.layers[key].reset_parameters()
        if self._stage.is_current_stage_last:
            self.norm.reset_parameters()

    # ------------------------------------------------------------------ pipeline shape inference
    def _microbatch_hidden(self, input_ids: torch.Tensor, n_microbatches: int) -> torch.Tensor:
        return torch.empty((input_ids.shape[0] // n_microbatches, input_ids.shape[1], self._hidden_size),
                           dtype=self.output_dtype(), device=input_ids.device)

    def _snapshot(self, input_ids: torch.Tensor, n_microbatches: int, num_entries: int) -> torch.Tensor:
        return torch.empty((num_entries, input_ids.shape[0] // n_microbatches, self._hidden_size),
                           dtype=self.output_dtype(), device=input_ids.device)

    def infer_stage_inputs_from_pipeline_inputs(self, inputs: dict[str, torch.Tensor], n_microbatches: int) -> dict[str, torch.Tensor]:
        ids = inputs["input_ids"]
        if self._stage.is_current_stage_first:
            return {"input_ids": torch.empty((ids.shape[0] // n_microbatches, ids.shape[1]), dtype=torch.long, device=ids.device)}
        out = {"hidden_states": self._microbatch_hidden(ids, n_microbatches)}
        if self._snapshot_mode != HiddenStatesAggregationMode.no:
            out["hidden_states_snapshot"] = self._snapshot(ids, n_microbatches, self._num_layers_before + 1)
        return out

    def infer_stage_outputs_from_pipeline_inputs(self, inputs: dict[str, torch.Tensor], n_microbatches: int) -> dict[str, torch.Tensor]:
        ids = inputs["input_ids"]
        out = {"hidden_states": self._microbatch_hidden(ids, n_microbatches)}
        if self._snapshot_mode != HiddenStatesAggregationMode.no:
            out["hidden_states_snapshot"] = self._snapshot(ids, n_microbatches, self._num_layers_before + 1 + len(self.layers))
        return out


class _HeadedDecoder(nn.Module, ModuleLateInit, ModuleSupportsPipelining):
    """Backbone under ``self.model`` + a task head on the last stage."""

    model: DecoderBackbone

    def __init__(self, stage: PipelineStageInfo, hidden_size: int):
        super().__init__()
        self._stage = stage
        self._hidden_size = hidden_size

    def _head_modules(self) -> list[nn.Module]:
        return []

    def reset_parameters(self) -> None:
        self.model.reset_parameters()
        if self._stage.is_current_stage_last:
            for head in self._head_modules():
                head.reset_parameters()

    def infer_stage_inputs_from_pipeline_inputs(self, inputs: dict[str, torch.Tensor], n_microbatches: int) -> dict[str, torch.Tensor]:
        return self.model.infer_stage_inputs_from_pipeline_inputs(inputs, n_microbatches)

    def infer_stage_outputs_from_pipeline_inputs(self, inputs: dict[str, torch.Tensor], n_microbatches: int) -> dict[str, torch.Tensor]:
        return self.model.infer_stage_outputs_from_pipeline_inputs(inputs, n_microbatches)


class DecoderForCausalLM(_HeadedDecoder):
    """Adds ``lm_head``; the last stage outputs ``logps [B,S]`` = fp32 per-token training objective (0 at ignored labels):
    the NLL, unless ``lm_head.set_loss_regularisation`` added label smoothing or a z-loss."""

    def __init__(self, backbone: DecoderBackbone, params: _BackboneParams, stage: PipelineStageInfo):
        super().__init__(stage, params.layer.hidden_size)
        self.model = backbone
        if stage.is_current_stage_last:
            self.lm_head = SplitLanguageModellingHead(split_vocab_size=params.split_vocab_size,
                                                      split_order=params.split_vocab_order,
                                                      hidden_size=params.layer.hidden_size)

    def _head_modules(self) -> list[nn.Module]:
        return [self.lm_head]

    def forward(self, input_ids=None, hidden_states=None, position_ids=None, hidden_states_snapshot=None,
                hidden_states_agg_mask=None, labels=None) -> dict[str, torch.Tensor | None]:
        out = self.model(input_ids=input_ids, hidden_states=hidden_states, position_ids=position_ids,
                         hidden_states_snapshot=hidden_states_snapshot, hidden_states_agg_mask=hidden_states_agg_mask)
        if self._stage.is_current_stage_last:
            out["logps"] = self.lm_head(hidden_states=out["hidden_states"], labels=labels)
        return out

    def infer_stage_outputs_from_pipeline_inputs(self, inputs, n_microbatches):
        out = super().infer_stage_outputs_from_pipeline_inputs(inputs, n_microbatches)
        if self._stage.is_current_stage_last:
            ids = inputs["input_ids"]
            out["logps"] = torch.empty((ids.shape[0] // n_microbatches, ids.shape[1]), dtype=torch.float32, device=ids.device)
        return out


class DecoderForClassification(_HeadedDecoder):
    """Adds ``cls_head``; the last stage outputs ``scores [n_pooled, num_labels]`` (fp32)."""

    def __init__(self, backbone: DecoderBackbone, params: _BackboneParams, stage: PipelineStageInfo, num_labels: int,
                 classifier_dropout: float):
        super().__init__(stage, params.layer.hidden_size)
        self.model = backbone
        self._num_labels = num_labels
        if stage.is_current_stage_last:
            self.cls_head = ClassificationHead(hidden_size=params.layer.hidden_size, num_labels=num_labels,
                                               dropout=classifier_dropout)

    def _head_modules(self) -> list[nn.Module]:
        return [self.cls_head]

    def forward(self, input_ids=None, hidden_states=None, position_ids=None, hidden_states_snapshot=None,
                hidden_states_agg_mask=None, pooling_mask=None) -> dict[str, torch.Tensor | None]:
        out = self.model(input_ids=input_ids, hidden_states=hidden_states, position_ids=position_ids,
                         hidden_states_snapshot=hidden_states_snapshot, hidden_states_agg_mask=hidden_states_agg_mask)
        if self._stage.is_current_stage_last:
            out["scores"] = self.cls_head(hidden_states=out["hidden_states"], pooling_mask=pooling_mask)
        return out

    def infer_stage_outputs_from_pipeline_inputs(self, inputs, n_microbatches):
        out = super().infer_stage_outputs_from_pipeline_inputs(inputs, n_microbatches)
        if self._stage.is_current_stage_last:
            ids = inputs["input_ids"]
            out["scores"] = torch.empty((ids.shape[0] // n_microbatches, self._num_labels), dtype=torch.float32, device=ids.device)
        return out


class DecoderForEmbedding(_HeadedDecoder):
    """Adds ``embedding_head``; the last stage outputs ``embeddings [n_pooled, dim]`` (fp32)."""

    def __init__(self, backbone: DecoderBackbone, params: _BackboneParams, stage: PipelineStageInfo,
                 embedding_dim: int | None, normalize: bool):
        super().__init__(stage, params.layer.hidden_size)
        self.model = backbone
        self._embedding_dim = embedding_dim if embedding_dim is not None else params.layer.hidden_size
        if stage.is_current_stage_last:
            self.embedding_head = EmbeddingHead(hidden_size=params.layer.hidden_size, embedding_dim=embedding_dim,
                                                normalize=normalize)

    def _head_modules(self) -> list[nn.Module]:
        return [self.embedding_head]

    def forward(self, input_ids=None, hidden_states=None, position_ids=None, hidden_states_snapshot=None,
                hidden_states_agg_mask=None, pooling_mask=None) -> dict[str, torch.Tensor | None]:
        out = self.model(input_ids=input_ids, hidden_states=hidden_states, position_ids=position_ids,
                         hidden_states_snapshot=hidden_states_snapshot, hidden_states_agg_mask=hidden_states_agg_mask)
        if self._stage.is_current_stage_last:
            out["embeddings"] = self.embedding_head(hidden_states=out["hidden_states"], pooling_mask=pooling_mask)
        return out

    def infer_stage_outputs_from_pipeline_inputs(self, inputs, n_microbatches):
        out = super().infer_stage_outputs_from_pipeline_inputs(inputs, n_microbatches)
        if self._stage.is_current_stage_last:
            ids = inputs["input_ids"]
            out["embeddings"] = torch.empty((ids.shape[0] // n_microbatches, self._embedding_dim), dtype=torch.float32, device=ids.device)
        return out


class PreNormDecoderLayer(nn.Module, ModuleLateInit):
    """``x + attn(norm(x))`` then ``x + mlp(norm(x))`` — the layer shape shared by Qwen3 / Llama-3 / Mixtral."""

    def __init__(self, self_attn: nn.Module, mlp: nn.Module, hidden_size: int, rms_norm_eps: float,
                 zero_centered_norm: bool = False):
        super().__init__()
        self.self_attn = self_attn  # any token mixer taking (hidden_states, position_embeddings, attention_mask)
        self.mlp = mlp
        self.input_layernorm = RMSNorm(hidden_size, eps=rms_norm_eps, zero_centered=zero_centered_norm)
        self.post_attention_layernorm = RMSNorm(hidden_size, eps=rms_norm_eps, zero_centered=zero_centered_norm)

    def forward(self, hidden_states: torch.Tensor, position_embeddings: tuple[torch.Tensor, torch.Tensor]) -> torch.Tensor:
        attn = self.self_attn(hidden_states=self.input_layernorm(hidden_states), position_embeddings=position_embeddings,
                              attention_mask=None)
        hidden_states = hidden_states + attn
        return hidden_states + self.mlp(self.post_attention_layernorm(hidden_states))

    def reset_parameters(self) -> None:
        self.self_attn.reset_parameters()
        self.mlp.reset_parameters()
        self.input_layernorm.reset_parameters()
        self.post_attention_layernorm.reset_parameters()

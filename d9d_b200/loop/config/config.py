from pathlib import Path
from typing import Literal

from pydantic import BaseModel, Field, NonNegativeFloat

from d9d_b200.pipelining.factory import AnyPipelineScheduleConfig
from d9d_b200.tracker import AnyTrackerConfig, RunConfig

from .types import StepActionPeriod


class BatchingConfig(BaseModel):
    global_batch_size: int  # over all replicas and accumulation steps
    microbatch_size: int  # one forward on one device


class DeterminismConfig(BaseModel):
    base_seed: int


class PipeliningConfig(BaseModel):
    schedule: AnyPipelineScheduleConfig


class GarbageCollectionConfig(BaseModel):
    period_steps: StepActionPeriod


class DataLoadingConfig(BaseModel):
    num_workers: int
    pin_memory: bool
    persistent_workers: bool


class CheckpointingConfig(BaseModel):
    save_dir: Path
    period_steps: StepActionPeriod
    num_to_keep: int | None
    # stage the state in host memory and write it from a background thread while training continues (the next save,
    # a load and the end of the job wait for the write in flight)
    async_save: bool = False


class Fp8LinearConfig(BaseModel):
    """Run the selected dense linear layers in fp8 (e4m3, dynamic row / column scaling for forward, input-gradient and
    weight-gradient GEMMs - ``d9d_b200.kernel.fp8.Fp8Linear``).  Net-new: the reference has no fp8 path.

    ``include`` / ``exclude`` are regular expressions searched in the module names of a model stage; only plain linear
    layers whose feature sizes are multiples of 16 are converted (LoRA wrappers, grouped expert weights, norms are not;
    ``ModelStageFactoryConfig.fp8_experts`` runs the expert blocks in fp8)."""

    include: str = r".*"
    exclude: str | None = r"lm_head|cls_head|embedding_head|router|\.gate$"
    # "mx": MXFP8 block scaling (feature sizes and token count multiples of 128); "blockwise": DeepSeek-V3's 1x128 activation
    # / 128x128 weight scaling with promoted accumulation (feature sizes multiples of 16)
    recipe: Literal["rowwise", "mx", "blockwise"] = "rowwise"


class ModelStageFactoryConfig(BaseModel):
    source_checkpoint: Path | None
    checkpoint_only_trainable_parameters: bool
    fp8_linear: Fp8LinearConfig | None = None
    # run every MoE expert block (GroupedSwiGLU) of the stage in fp8: e4m3 grouped GEMMs for the forward, input gradient
    # and weight gradient; the weights stay bf16 masters
    fp8_experts: bool = False
    # the fp8 experts' scaling: "rowwise" (per-expert row / column scales) or "blockwise" (DeepSeek-V3's 1x128 activation /
    # 128x128 weight scales, promoted per 128-deep k-block); read only when fp8_experts is on
    fp8_experts_recipe: Literal["rowwise", "blockwise"] = "rowwise"


class GradientClippingConfig(BaseModel):
    max_norm: float | None
    log_total_steps: StepActionPeriod


class ProfilingConfig(BaseModel):
    enabled: bool
    traces_dir: Path
    period_steps: int
    warmup_steps: int
    active_steps: int


class JobLoggerConfig(BaseModel):
    period_steps: StepActionPeriod
    tracker: AnyTrackerConfig


class GradientManagerConfig(BaseModel):
    grad_dtype: str | None  # None => parameter dtype
    bucket_size_mb: int
    # fold the 1/sum(weights) scaling and the clip coefficient into the optimizer's gradient-scale input instead of
    # rewriting every gradient twice (only when every optimizer accepts a device ``grad_scale``, e.g. StochasticAdamW)
    fold_scaling_into_optimizer: bool = True


class ExpertBiasBalancingConfig(BaseModel):
    """Auxiliary-loss-free load balancing (DeepSeek-V3): after every optimizer step each expert bias of the model's MoE
    routers moves by ``update_rate`` toward balance, ``b_e += update_rate * sign(mean(c) - c_e)``, ``c_e`` counting the
    step's selections of expert ``e`` over every rank of the pipeline stage."""

    update_rate: float


class MoEAuxLossConfig(BaseModel):
    """Train softmax MoE routers with the Switch Transformer load-balancing loss and the ST-MoE router z-loss, per MoE layer
    and forward: ``load_balancing_coef * A + z_loss_coef * Z`` with ``A = E sum_e f_e P_e`` (``f_e``: share of the ``T k``
    selections that went to expert ``e``, ``P_e``: mean softmax score of expert ``e``) and ``Z = mean_t logsumexp(x_t)^2``,
    weighted like the LM loss (``T * LOSS_WEIGHT_PER_TOKEN``) and summed over the MoE layers.  ``A`` is ``k`` times
    smaller than Hugging Face's ``load_balancing_loss_func``, which also averages over layers: HF's
    ``router_aux_loss_coef`` ``c`` corresponds to ``load_balancing_coef = c * k / num_moe_layers``.  Sigmoid routers are
    refused for these two terms (they balance with ``expert_bias_balancing``).

    ``sequence_balance_coef`` adds the sequence-wise balance loss of softmax and sigmoid routers (DeepSeek-V3 eqs. 17-20,
    ``alpha``; DeepSeek-V2's ``seq_aux``): ``sequence_balance_coef * mean_b A_b`` per MoE layer and forward of ``B``
    sequences, ``A_b = E / (k S^2) sum_e c[b, e] sum_{t in b} s[t, e]`` over the sequence's ``S`` tokens, weighted like the
    other terms.  It needs whole sequences on every rank: context and tensor (sequence) parallel meshes are refused."""

    load_balancing_coef: NonNegativeFloat = 0.0
    z_loss_coef: NonNegativeFloat = 0.0
    sequence_balance_coef: NonNegativeFloat = 0.0


class LMLossConfig(BaseModel):
    """Regularise the LM loss per target token: ``cross_entropy(z, y, label_smoothing) + z_loss_coef * lse(z)^2`` in the
    fused linear cross-entropy (PaLM's z-loss: ``z_loss_coef`` around 1e-4)."""

    label_smoothing: float = Field(default=0.0, ge=0.0, le=1.0)
    z_loss_coef: NonNegativeFloat = 0.0


class TimeoutConfig(BaseModel):
    init_timeout: int = 10000
    step_timeout: int = 100


class TrainerConfig(BaseModel):
    run: RunConfig
    batching: BatchingConfig
    data_loading: DataLoadingConfig
    logging: JobLoggerConfig
    pipelining: PipeliningConfig
    model_stage_factory: ModelStageFactoryConfig
    determinism: DeterminismConfig
    gc: GarbageCollectionConfig
    checkpointing: CheckpointingConfig
    gradient_clipping: GradientClippingConfig
    profiling: ProfilingConfig | None
    gradient_manager: GradientManagerConfig
    timeout: TimeoutConfig = TimeoutConfig()
    expert_bias_balancing: ExpertBiasBalancingConfig | None = None  # None: expert biases stay as loaded
    moe_aux_loss: MoEAuxLossConfig | None = None  # None: routers train without auxiliary losses
    lm_loss: LMLossConfig | None = None  # None: the LM head trains on the plain NLL and logs nothing more


class InferenceConfig(BaseModel):
    batching: BatchingConfig
    data_loading: DataLoadingConfig
    model_stage_factory: ModelStageFactoryConfig
    determinism: DeterminismConfig
    gc: GarbageCollectionConfig
    checkpointing: CheckpointingConfig
    profiling: ProfilingConfig | None
    timeout: TimeoutConfig = TimeoutConfig()

"""Pydantic job configuration (reference ``d9d/loop/config``)."""

from .config import (
    BatchingConfig,
    CheckpointingConfig,
    DataLoadingConfig,
    DeterminismConfig,
    ExpertBiasBalancingConfig,
    GarbageCollectionConfig,
    GradientClippingConfig,
    GradientManagerConfig,
    InferenceConfig,
    JobLoggerConfig,
    Fp8LinearConfig,
    ModelStageFactoryConfig,
    MoEAuxLossConfig,
    PipeliningConfig,
    ProfilingConfig,
    TimeoutConfig,
    TrainerConfig,
)
from .types import StepActionPeriod, StepActionSpecial

__all__ = [
    "BatchingConfig",
    "CheckpointingConfig",
    "DataLoadingConfig",
    "DeterminismConfig",
    "ExpertBiasBalancingConfig",
    "MoEAuxLossConfig",
    "GarbageCollectionConfig",
    "GradientClippingConfig",
    "GradientManagerConfig",
    "InferenceConfig",
    "JobLoggerConfig",
    "Fp8LinearConfig",
    "ModelStageFactoryConfig",
    "PipeliningConfig",
    "ProfilingConfig",
    "StepActionPeriod",
    "StepActionSpecial",
    "TimeoutConfig",
    "TrainerConfig",
]

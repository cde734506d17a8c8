"""Building blocks of the training / inference loops (reference ``d9d/loop/component``)."""

from .batch_maths import BatchMaths
from .checkpointer import StateCheckpointer
from .data_loader_factory import DataLoaderFactory, IteratorBatchGroup, StatefulDataLoaderDataParallelAware
from .expert_bias_balancer import ExpertBiasBalancer
from .moe_aux_loss import MoEAuxLoss
from .lm_loss import LMLoss
from .garbage_collector import ManualGarbageCollector
from .gradient_clipper import GradientClipper
from .gradient_manager import GradientManager
from .job_logger import JobLogger
from .job_profiler import JobProfiler
from .model_stage_exporter import ModelStageExporter
from .model_stage_factory import ModelStageFactory, TrackedModules
from .optimizer_factory import OptimizerFactory
from .pipeline_result_processing import STATE_LOSS, STATE_LOSS_WEIGHT, InferenceProcessor, LossComputer, PipelineOutputsProcessor
from .stepper import Stepper
from .task_operator import ForwardResult, InferenceTaskOperator, TrainTaskOperator
from .timeout_manager import TimeoutManager

__all__ = [
    "STATE_LOSS",
    "STATE_LOSS_WEIGHT",
    "BatchMaths",
    "DataLoaderFactory",
    "ExpertBiasBalancer",
    "ForwardResult",
    "MoEAuxLoss",
    "LMLoss",
    "GradientClipper",
    "GradientManager",
    "InferenceProcessor",
    "InferenceTaskOperator",
    "IteratorBatchGroup",
    "JobLogger",
    "JobProfiler",
    "LossComputer",
    "ManualGarbageCollector",
    "ModelStageExporter",
    "ModelStageFactory",
    "OptimizerFactory",
    "PipelineOutputsProcessor",
    "StateCheckpointer",
    "StatefulDataLoaderDataParallelAware",
    "Stepper",
    "TimeoutManager",
    "TrackedModules",
    "TrainTaskOperator",
]

"""Mixture-of-Experts building blocks."""

from .balancing import update_expert_bias
from .grouped_experts import GroupedSwiGLU
from .grouped_linear import GroupedLinear
from .layer import MoELayer
from .router import RouterParameters, RoutingResult, TopKRouter
from .shared_expert import SharedExpertParameters, SharedSwiGLU

__all__ = [
    "GroupedLinear",
    "GroupedSwiGLU",
    "MoELayer",
    "RouterParameters",
    "RoutingResult",
    "SharedExpertParameters",
    "SharedSwiGLU",
    "TopKRouter",
    "update_expert_bias",
]

"""Stochastic-rounding kernels (reference ``d9d/kernel/stochastic``).

SR primitive: add 16 counter-based random bits (Philox-4x32-10 keyed by ``(seed, element offset)``) below the kept
bf16 mantissa, truncate.  Unbiased, reproducible, independent of launch geometry.
Difference from the reference: AdamW is a *multi-tensor* launch (one kernel for a whole parameter group) with an optional
device-side gradient scale (fuses ``grad / sum(loss_weight)`` and clipping into the update).
"""

from .adamw_step import adamw_stochastic_bf16_, adamw_stochastic_bf16_multi_
from .copy import copy_fp32_to_bf16_stochastic_

__all__ = ["adamw_stochastic_bf16_", "adamw_stochastic_bf16_multi_", "copy_fp32_to_bf16_stochastic_"]

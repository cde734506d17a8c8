"""MoE token routing kernels.

Native path (``layout.py``): a stable counting sort builds a 128-row aligned, expert-sorted layout *on the
device* (no ``bincount().cpu()``, no host-side ``batch_sizes``), tokens are scattered/gathered by fused kernels and
the grouped wgmma GEMM walks a device-side tile->expert table.

Compatibility surface (``compat.py``): ``fused_indices_to_multihot``, ``moe_permute_with_probs``,
``moe_unpermute_mask`` with the reference's signatures (``d9d/kernel/moe/*.py``).
"""

from .compat import fused_indices_to_multihot, moe_permute_with_probs, moe_unpermute_mask
from .experts import fp8_grouped_linear_reference, grouped_swiglu, grouped_swiglu_fp8_reference
from .layout import MoELayout, build_moe_layout, grouped_linear, moe_permute, moe_unpermute

__all__ = [
    "MoELayout",
    "build_moe_layout",
    "fp8_grouped_linear_reference",
    "fused_indices_to_multihot",
    "grouped_linear",
    "grouped_swiglu",
    "grouped_swiglu_fp8_reference",
    "moe_permute",
    "moe_permute_with_probs",
    "moe_unpermute",
    "moe_unpermute_mask",
]

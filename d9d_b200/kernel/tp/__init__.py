"""Sequence-parallel tensor-parallel linears whose collective is fused into the wgmma GEMM over NVLink peer memory.

* ``all_gather_linear``      ``y = all_gather_seq(x) @ W_col^T``     A tiles are TMA-loaded from the owning peer
* ``linear_reduce_scatter``  ``y = reduce_scatter_seq(x @ W_row^T)``  output tiles are TMA reduce-added into the owner
  (backward passes use the mirrored kernels plus the token-sharded wgrad).
"""

from .fused import TensorParallelWorkspace, all_gather_linear, linear_reduce_scatter

__all__ = ["TensorParallelWorkspace", "all_gather_linear", "linear_reduce_scatter"]

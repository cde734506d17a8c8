"""Kernel layer: the public op surface of ``d9d.kernel`` re-implemented on hand-written sm_90a CUDA kernels.

Every op has two implementations:

* the **native** one (``d9d_b200.ops``: wgmma GEMMs fed by TMA, fused bandwidth-bound kernels) which is
  *mandatory* for CUDA tensors — there is no silent PyTorch fallback on a GPU box;
* a plain PyTorch fp32 **oracle** used on CPU (plumbing tests, gloo runs) and as the numerics reference in tests.
"""

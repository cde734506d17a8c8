from __future__ import annotations

import torch

# kernels launched per native op call (used for the bench's ``gpu_launches`` accounting)
_KERNELS_PER_OP = {
    "rms_norm_bwd": 2,
    "moe_build_layout": 3,
    "moe_permute": 2,
    "ce_forward": 3,  # zero-fill of the target-logit buffer + GEMM + finalize
    "ce_forward_ex": 3,
    "ce_forward_reg": 3,
    "flash_attn_bwd": 3,  # delta pre-pass + dK/dV kernel + dQ kernel
    "quantize_colwise_t_batched": 2,  # column amax + transposing quantiser
    "quantize_segments_t": 2,
}


class _CountingOps:
    """Thin proxy over ``torch.ops.d9d_b200`` that counts kernel launches of the native extension."""

    def __init__(self, ns):
        self._ns = ns
        self.launches = 0
        self._cache: dict[str, object] = {}

    def __getattr__(self, name: str):
        fn = self._cache.get(name)
        if fn is None:
            op = getattr(self._ns, name)
            n = _KERNELS_PER_OP.get(name, 1)

            def call(*args, __op=op, __n=n, **kwargs):
                self.launches += __n
                return __op(*args, **kwargs)

            fn = call
            self._cache[name] = fn
        return fn


_proxy: _CountingOps | None = None


def native_ops() -> _CountingOps:
    """The native op namespace (loads / builds the extension on first use)."""
    global _proxy
    if _proxy is None:
        from d9d_b200 import ops

        _proxy = _CountingOps(ops.load())
    return _proxy


def native_launch_count() -> int:
    return _proxy.launches if _proxy is not None else 0


def contiguous_aligned(t: torch.Tensor) -> torch.Tensor:
    """``t.contiguous()``, copied into a fresh buffer when its first element is not 16-byte aligned.  The native kernels
    load and store 16 bytes at a time and refuse such operands; ``.contiguous()`` alone returns a contiguous view at an
    element offset (``flat[3:3 + n]``) unchanged."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def on_gpu(*tensors: torch.Tensor) -> bool:
    """True if the op must run on the native CUDA path."""
    return any(t is not None and t.is_cuda for t in tensors)


def grad_dtype_of(t: torch.Tensor) -> torch.dtype:
    """Dtype autograd expects for the gradient of ``t`` (``grad_dtype`` is only defined on leaves)."""
    try:
        gd = t.grad_dtype if t.is_leaf else None
    except (RuntimeError, AttributeError):
        gd = None
    if gd not in (torch.bfloat16, torch.float32):
        return t.dtype
    return gd


# ------------------------------------------------------------------------------------------------------------------
# Weight-gradient accumulation fused into the wgrad GEMM epilogue
# ------------------------------------------------------------------------------------------------------------------
MAIN_PARAM_ATTR = "_d9d_main_param"  # set on local views handed to modules: the (D)Tensor parameter that owns .grad
FUSED_WGRAD_ATTR = "_d9d_fused_wgrad"  # set by the gradient infrastructure on parameters whose .grad is pre-allocated
# set on parameters whose gradient reduction, scaling, clipping and zeroing belong to an optimizer that reduces over
# NVLink itself (value: that optimizer); GradientSynchronizer / GradientManager / GradientClipper leave them alone
EXTERNAL_GRAD_OWNER_ATTR = "_d9d_external_grad_owner"


def fused_wgrad_owner(weight: torch.Tensor) -> torch.Tensor | None:
    """The leaf parameter whose pre-allocated ``.grad`` the wgrad GEMM of ``weight`` may accumulate into, or None.

    Writing ``dW`` straight into the flat gradient arena (``beta = 1`` in the GEMM epilogue, a TMA reduce-add)
    removes the temporary ``dW`` tensor and autograd's ``grad += dW`` pass.  Protocol used by the autograd functions:

    * forward receives the *detached* weight plus the owner as an extra (unused) input, so the owner stays a leaf of
      the graph;
    * backward accumulates into ``fused_wgrad_buffer(owner)`` and returns ``None`` for the owner – the autograd engine
      still runs the owner's ``AccumulateGrad`` node with an undefined gradient, which fires its post-accumulate-grad
      hooks exactly once (this is what drives the bucketed gradient all-reduce).

    Only parameters the gradient infrastructure opted in (``GradientSynchronizer.bind`` / the bench runner) qualify.
    """
    if not torch.is_grad_enabled() or not weight.requires_grad:
        return None
    owner = getattr(weight, MAIN_PARAM_ATTR, weight)
    if not getattr(owner, FUSED_WGRAD_ATTR, False) or not owner.is_leaf or owner.grad is None:
        return None
    local = getattr(owner.grad, "_local_tensor", owner.grad)
    if local.shape != weight.shape or not local.is_contiguous() or local.dtype not in (torch.float32, torch.bfloat16):
        return None
    return owner


def fused_wgrad_buffer(owner: torch.Tensor) -> torch.Tensor:
    grad = owner.grad
    if grad is None:
        raise RuntimeError("d9d_b200: the gradient buffer of a fused-wgrad parameter disappeared between forward and backward")
    return getattr(grad, "_local_tensor", grad)  # DTensor -> local shard

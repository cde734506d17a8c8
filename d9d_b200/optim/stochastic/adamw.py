"""AdamW for bf16 parameters with fp32 math and stochastic rounding.

Parity: reference ``d9d/optim/stochastic/adamw.py:45-163`` (state layout ``step / exp_avg / exp_avg_sq``, DTensor
aware state allocation, own CPU generator checkpointed under ``_d9d_generator_state``).

Difference from the reference: the reference issues one Triton launch *and* one CPU ``randint().item()`` per parameter per step;
here every parameter group is updated by ONE multi-tensor kernel launch with ONE seed draw, the pointer tables live
on the device and are cached across steps, and an optional device-side ``grad_scale`` scalar lets the caller fold
``1/sum(loss_weight)`` and the clipping coefficient into the update (no extra pass over the gradients).
"""

from __future__ import annotations

from typing import cast

import torch
from torch.distributed.tensor import DTensor
from torch.optim import Optimizer
from torch.optim.optimizer import ParamsT, StateDict

from d9d_b200.kernel.stochastic.adamw_step import AdamWLaunchPlan, adamw_stochastic_bf16_multi_

_GENERATOR_STATE_KEY = "_d9d_generator_state"


def _local(t: torch.Tensor) -> torch.Tensor:
    return t.to_local() if isinstance(t, DTensor) else t


def _new_state(p: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    local = torch.zeros_like(_local(p), dtype=dtype, memory_format=torch.contiguous_format)
    if isinstance(p, DTensor):
        return DTensor.from_local(local, device_mesh=p.device_mesh, placements=p.placements, run_check=False,
                                  shape=p.shape, stride=p.stride())
    return local


class StochasticAdamW(Optimizer):
    def __init__(
        self,
        params: ParamsT,
        lr: float,
        betas: tuple[float, float] = (0.9, 0.999),
        eps: float = 1e-8,
        weight_decay: float = 1e-2,
        generator: torch.Generator | None = None,
        state_dtype: torch.dtype = torch.float32,
    ):
        if lr <= 0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps <= 0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if weight_decay < 0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if generator is None:
            generator = torch.Generator(device="cpu")
            generator.manual_seed(cast(int, torch.randint(0, 2**32, (1,)).item()))
        self._generator = generator
        self._plans: dict[tuple, AdamWLaunchPlan | None] = {}
        self.grad_scale: torch.Tensor | None = None  # optional device fp32 scalar applied to every gradient
        super().__init__(params, {"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay,
                                  "state_dtype": state_dtype})

    def state_dict(self) -> StateDict:
        sd = super().state_dict()
        sd[_GENERATOR_STATE_KEY] = self._generator.get_state()
        return sd

    def load_state_dict(self, state_dict: StateDict) -> None:
        """Restore moments, step counters, hyper-parameters and the rounding stream.

        ``torch.optim.Optimizer.load_state_dict`` casts every floating-point state tensor to the *parameter* dtype, which
        would silently truncate fp32 moments of bf16 parameters on resume, so the state is re-attached here as saved
        (matched to the parameters by position, like the base class does).
        """
        state_dict = dict(state_dict)
        if _GENERATOR_STATE_KEY in state_dict:
            self._generator.set_state(state_dict.pop(_GENERATOR_STATE_KEY))
        saved_groups, saved_state = state_dict["param_groups"], state_dict["state"]
        if len(saved_groups) != len(self.param_groups):
            raise ValueError("loaded state dict has a different number of parameter groups")
        by_id: dict[int, torch.Tensor] = {}
        for saved, group in zip(saved_groups, self.param_groups, strict=True):
            if len(saved["params"]) != len(group["params"]):
                raise ValueError("loaded state dict contains a parameter group that doesn't match the size of optimizer's group")
            by_id.update(zip(saved["params"], group["params"], strict=True))
            group.update({k: v for k, v in saved.items() if k != "params"})
        self.state.clear()
        for pid, entries in saved_state.items():
            if isinstance(pid, str) and pid.isdigit():
                # torch.distributed.checkpoint loads tensors in place (under the original integer ids) and hands the
                # non-tensor leaves - the step counters - back under stringified ids: merge both views
                pid = int(pid)
            param = by_id[pid]
            device = _local(param).device
            self.state[param].update({k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in entries.items()})
        self._plans.clear()

    @torch.no_grad()
    def step(self, closure: None = None) -> None:  # type: ignore[override]
        """One fused launch per (step count, gradient dtype) bucket of each parameter group.  Parameters without a
        gradient are skipped and keep their state.  Each launch draws one seed from the generator: groups in order, and
        within a group the buckets in the order of their first parameter."""
        if closure is not None:
            raise ValueError("Closure is not supported")
        for gi, group in enumerate(self.param_groups):
            beta1, beta2 = group["betas"]
            # bucket by (step, grad dtype): one fused launch per bucket (normally exactly one per group)
            buckets: dict[tuple[int, torch.dtype], list[tuple[torch.Tensor, ...]]] = {}
            first: dict[tuple[int, torch.dtype], int] = {}
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("StochasticAdamW does not support sparse gradients")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = _new_state(p, group["state_dtype"])
                    state["exp_avg_sq"] = _new_state(p, group["state_dtype"])
                state["step"] += 1
                key = (int(state["step"]), _local(p.grad).dtype)
                first.setdefault(key, id(p))
                buckets.setdefault(key, []).append(
                    (_local(p), _local(p.grad), _local(state["exp_avg"]), _local(state["exp_avg_sq"]))
                )
            for (step, grad_dtype), items in buckets.items():
                ps, gs, ms, vs = (list(col) for col in zip(*items, strict=True))
                # a bucket's plan is found again by its first parameter, not its step count: a parameter that got its
                # first gradient later lags by a step for good, and its bucket must not evict the group's plan
                plan_key = (gi, grad_dtype, first[(step, grad_dtype)], len(ps))
                self._plans[plan_key] = adamw_stochastic_bf16_multi_(
                    ps, gs, ms, vs, lr=group["lr"], beta1=beta1, beta2=beta2, eps=group["eps"],
                    weight_decay=group["weight_decay"], step=step, generator=self._generator,
                    grad_scale=self.grad_scale, plan=self._plans.get(plan_key),
                )

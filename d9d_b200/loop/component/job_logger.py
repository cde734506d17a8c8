from __future__ import annotations

from collections.abc import Generator, Iterator
from contextlib import contextmanager
from typing import Any

import torch
import torch.utils._pytree as pytree
from torch.distributed.checkpoint.stateful import Stateful

from d9d_b200.core.dist_context import DistributedContext
from d9d_b200.core.types import ScalarTree
from d9d_b200.internals.metric_collector import AsyncMetricCollector
from d9d_b200.internals.state import load_state_dict_main_process, state_dict_main_process
from d9d_b200.loop.config import JobLoggerConfig
from d9d_b200.metric.impl.container import ComposeMetric
from d9d_b200.tracker import BaseTracker, BaseTrackerRun, RunConfig, tracker_from_config
from d9d_b200.tracker.provider.null import NullTrackerConfig

from .stepper import Stepper


def flatten_metric_tree(tree: Any) -> dict[str, Any]:
    """Nested results -> ``{"a/b/c": value}``."""
    flat = {}
    for path, value in pytree.tree_leaves_with_path(tree):
        parts = []
        for key in path:
            if isinstance(key, pytree.MappingKey):
                parts.append(str(key.key))
            elif isinstance(key, pytree.SequenceKey):
                parts.append(str(key.idx))
            elif isinstance(key, pytree.GetAttrKey):
                parts.append(key.name)
            else:
                parts.append(str(key))
        flat["/".join(parts)] = value
    return flat


class _DeferredScalar:
    """Device scalar -> host without stalling the step: the value is copied into pinned memory on the current stream
    and read one step later (after its event completed).  The reference calls ``loss.item()`` every step, i.e. a
    full device sync per step."""

    def __init__(self, device: torch.device):
        self._cuda = device.type == "cuda"
        self._pending: list[tuple[int, torch.Tensor, Any]] = []

    def push(self, step: int, value: torch.Tensor) -> None:
        if self._cuda:
            host = torch.empty((), dtype=torch.float32, pin_memory=True)
            host.copy_(value.detach().float(), non_blocking=True)
            event = torch.cuda.Event()
            event.record()
            self._pending.append((step, host, event))
        else:
            self._pending.append((step, value.detach().float().cpu(), None))

    def pop_ready(self, force: bool = False) -> list[tuple[int, float]]:
        out = []
        while self._pending:
            step, host, event = self._pending[0]
            if event is not None and not force and not event.query():
                break
            if event is not None and force:
                event.synchronize()
            out.append((step, float(host)))
            self._pending.pop(0)
        return out


class JobLogger(Stateful):
    """Logs ``loss`` every step and the task metrics every ``period_steps`` (synchronised on a side stream)."""

    def __init__(self, dist_context: DistributedContext, config: JobLoggerConfig, metrics: ComposeMetric, stepper: Stepper,
                 run_config: RunConfig, additional_hparams: ScalarTree):
        self._ctx, self._config, self._stepper = dist_context, config, stepper
        self._run_config = run_config.model_copy(deep=True, update={"hparams": {"run": run_config.hparams, "params": additional_hparams}})
        self._tracker: BaseTracker = tracker_from_config(config.tracker if dist_context.is_main_process else NullTrackerConfig())
        self._collector = AsyncMetricCollector(metrics)
        self._loss_reader = _DeferredScalar(dist_context.current_device)
        self.last_loss: float | None = None

    @contextmanager
    def new_run(self) -> Generator[BaseTrackerRun, None, None]:
        with self._tracker.open(self._run_config) as run:
            yield run

    @contextmanager
    def install(self) -> Iterator[None]:
        self._collector.bind(self._ctx.current_device)
        try:
            yield
        finally:
            self._collector.unbind()

    def _due(self) -> bool:
        return self._stepper.should_do_action(self._config.period_steps, enable_on_last_step_if_periodic=True)

    def is_due(self) -> bool:
        """Whether this step logs the metrics (the same answer on every rank)."""
        return self._due()

    def trigger_sync(self) -> None:
        if self._due():
            self._collector.schedule_collection(self._ctx)

    def _emit_losses(self, run: BaseTrackerRun, force: bool) -> None:
        current = self._stepper.current_step
        for step, value in self._loss_reader.pop_ready(force=force):
            run.set_step(step)
            run.scalar("loss", value)
            self.last_loss = value
        run.set_step(current)

    def log(self, run: BaseTrackerRun, loss_value: torch.Tensor) -> None:
        self._loss_reader.push(self._stepper.current_step, loss_value)
        last_step = self._stepper.current_step + 1 >= self._stepper.total_steps
        self._emit_losses(run, force=last_step or self._due())
        if not self._due():
            return
        for name, value in flatten_metric_tree(self._collector.collect_results()).items():
            run.scalar(name, value)

    def flush(self, run: BaseTrackerRun) -> None:
        self._emit_losses(run, force=True)

    def state_dict(self) -> dict[str, Any]:
        return {"tracker": state_dict_main_process(self._ctx, self._tracker)}

    def load_state_dict(self, state_dict: dict[str, Any]) -> None:
        load_state_dict_main_process(self._ctx, self._tracker, state_dict["tracker"])

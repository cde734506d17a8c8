from __future__ import annotations

from pathlib import Path

from tqdm import tqdm

from d9d_b200.core.dist_context import DeviceMeshParameters
from d9d_b200.internals.pipeline_state import PipelineStateHandler
from d9d_b200.loop import component as parts
from d9d_b200.loop import control
from d9d_b200.loop.config import TrainerConfig
from d9d_b200.loop.event.catalogue import common as shared_events
from d9d_b200.loop.event.catalogue import train as events
from d9d_b200.loop.state import TrainJobState
from d9d_b200.metric.impl.container import ComposeMetric

from ._assembly import build_housekeeping, lay_foundation


class TrainingConfigurator:
    """Assembles a :class:`Trainer` from the mesh, the trainer config and the user's providers
    (reference ``d9d/loop/run/train.py:68-248``)."""

    def __init__(self, mesh: DeviceMeshParameters, parameters: TrainerConfig, task_provider: control.TrainTaskProvider,
                 model_provider: control.ModelProvider, data_provider: control.DatasetProvider, optimizer_provider: control.OptimizerProvider,
                 lr_scheduler_provider: control.LRSchedulerProvider):
        self._mesh = mesh
        self._parameters = parameters
        self._task_provider = task_provider
        self._model_provider = model_provider
        self._data_provider = data_provider
        self._optimizer_provider = optimizer_provider
        self._lr_scheduler_provider = lr_scheduler_provider

    def _build_state(self) -> TrainJobState:
        cfg = self._parameters
        base = lay_foundation(self._mesh, cfg, lambda ctx: self._task_provider(control.TrainTaskProviderContext(dist_context=ctx)),
                              self._model_provider, cfg.batching, cfg.pipelining, events.EVENT_TRAIN_CONFIG_STARTED)
        ctx, bus, maths, task = base.ctx, base.bus, base.maths, base.task

        loader = parts.DataLoaderFactory(dist_context=ctx, provider=self._data_provider, config_data_loading=cfg.data_loading,
                                         batch_maths=maths).build_dataloader_for_train_job()
        bus.trigger(events.EVENT_TRAIN_DATA_LOADER_READY, shared_events.EventDataLoaderReadyContext(data_loader=loader))
        # one step consumes a whole accumulation group (the reference counts loader batches here, which overstates
        # the number of optimizer steps by the accumulation factor)
        stepper = parts.Stepper(initial_step=0, total_steps=len(loader) // maths.num_microbatches_gradient_accumulation)

        pipeline_state = PipelineStateHandler(sharding_spec={}, num_shards=maths.num_microbatches_pipelining)
        schedule, modules = parts.ModelStageFactory(
            model_provider=self._model_provider, dist_context=ctx, batch_maths=maths, config_model=cfg.model_stage_factory,
            config_pipelining=cfg.pipelining, pipeline_callback=parts.LossComputer(state=pipeline_state, task=task, stepper=stepper),
        ).build_pipeline_and_modules()
        bus.trigger(events.EVENT_TRAIN_MODEL_STAGES_READY, shared_events.EventModelStagesReadyContext(modules=modules.modules))
        metrics = ComposeMetric(task.create_metrics(control.CreateMetricsContext()).metrics)

        optimizer, scheduler = parts.OptimizerFactory(
            dist_context=ctx, tracked_modules=modules, optimizer_provider=self._optimizer_provider,
            lr_scheduler_provider=self._lr_scheduler_provider, stepper=stepper,
        ).build_optimizer_and_scheduler()
        bus.trigger(events.EVENT_TRAIN_OPTIMIZER_READY, events.EventOptimizerReadyContext(optimizer=optimizer))
        bus.trigger(events.EVENT_TRAIN_LR_SCHEDULER_READY, events.EventLRSchedulerReadyContext(lr_scheduler=scheduler))

        # gradients: the manager hands its 1/sum(w) scale to optimizers that can fold it into their update kernel, and the
        # clipper multiplies its coefficient into the same pending scalar
        grad_manager = parts.GradientManager(dist_context=ctx, tracked_modules=modules, batch_maths=maths, config=cfg.gradient_manager)
        grad_manager.bind_optimizer(optimizer)
        clipper = parts.GradientClipper(dist_context=ctx, tracked_modules=modules, config=cfg.gradient_clipping, stepper=stepper)
        clipper.bind_gradient_manager(grad_manager)

        house = build_housekeeping(ctx, cfg, stepper, run_name=cfg.run.name)
        hparams = {"task": task.dump_hparams(), "model": self._model_provider.dump_hparams()}
        return TrainJobState(
            dist_context=ctx, event_bus=bus, task=task, batch_maths=maths, data_loader=loader, stepper=stepper, tracked_modules=modules,
            task_operator=parts.TrainTaskOperator(dist_context=ctx, task=task, pipeline=schedule, pipeline_state=pipeline_state,
                                                  metrics=metrics),
            metrics=metrics, optimizer=optimizer, lr_scheduler=scheduler, gradient_manager=grad_manager, gradient_clipper=clipper,
            logger=parts.JobLogger(dist_context=ctx, config=cfg.logging, metrics=metrics, stepper=stepper, run_config=cfg.run,
                                   additional_hparams=hparams),
            exporter=parts.ModelStageExporter(model_provider=self._model_provider, dist_context=ctx, modules=modules),
            garbage_collector=house.gc, checkpointer=house.checkpointer, profiler=house.profiler, timeout_manager=base.timeout,
            expert_bias_balancer=parts.ExpertBiasBalancer(dist_context=ctx, tracked_modules=modules, config=cfg.expert_bias_balancing)
            if cfg.expert_bias_balancing is not None else None,
            moe_aux_loss=parts.MoEAuxLoss(dist_context=ctx, tracked_modules=modules, config=cfg.moe_aux_loss)
            if cfg.moe_aux_loss is not None else None,
            lm_loss=parts.LMLoss(dist_context=ctx, tracked_modules=modules, config=cfg.lm_loss)
            if cfg.lm_loss is not None else None,
        )

    def configure(self) -> "Trainer":
        return Trainer(self._build_state())


class Trainer:
    """Runs the training loop over a prepared :class:`TrainJobState` (reference ``run/train.py:251-376``).

    One iteration == one optimizer step: forward/backward over the accumulation group (gradient buckets all-reduce
    on the side stream as they fill), metric sync kicked off asynchronously, gradient wait + ``1/sum(w)`` scaling,
    clipping, optimizer, expert-bias balancing (when configured), LR scheduler, logging (+ the MoE auxiliary losses and
    the LM loss terms when configured), ``zero_grad``, housekeeping, post-step checkpoint.
    """

    def __init__(self, state: TrainJobState):
        self._state = state

    @property
    def state(self) -> TrainJobState:
        return self._state

    def train(self) -> None:
        s = self._state
        s.dist_context.wait_world()
        s.dist_context.logger.info("Trying to load last checkpoint before doing anything else")
        s.checkpointer.load_last_checkpoint(s)
        if s.stepper.current_step >= s.stepper.total_steps:
            s.dist_context.logger.info("Already trained fully, will do nothing")
            return
        s.dist_context.wait_world()
        step_ctx = shared_events.EventStepContext(stepper=s.stepper)
        with (
            tqdm(desc="Training", total=s.stepper.total_steps, initial=s.stepper.current_step,
                 disable=not s.dist_context.is_local_main_process) as bar,
            s.logger.new_run() as run,
            s.garbage_collector as gc,
            s.profiler.open() as profiler,
            s.gradient_manager.install(),
            s.gradient_clipper.install(),
            s.logger.install(),
        ):
            run.set_context({"stage": "train"})
            s.event_bus.trigger(events.EVENT_TRAIN_READY, events.EventTrainReadyContext(run=run))
            for batch_group in s.data_loader:
                run.set_step(s.stepper.current_step)
                s.event_bus.trigger(events.EVENT_TRAIN_STEP_PRE, step_ctx)
                if s.expert_bias_balancer is not None:
                    s.expert_bias_balancer.reset_counters()
                if s.moe_aux_loss is not None:
                    s.moe_aux_loss.reset()
                if s.lm_loss is not None:
                    s.lm_loss.reset()
                with s.event_bus.bounded(events.EVENT_TRAIN_FORWARD_BACKWARD_PRE, events.EVENT_TRAIN_FORWARD_BACKWARD_POST, step_ctx):
                    for batch in batch_group:
                        result = s.task_operator.forward_backward(batch)
                        if result is not None:
                            s.gradient_manager.add_loss_with_weight(result.loss, result.loss_weight)
                s.logger.trigger_sync()
                s.gradient_manager.sync_and_scale()
                s.gradient_clipper.clip_and_log(run)
                with s.event_bus.bounded(events.EVENT_TRAIN_OPTIMIZER_STEP_PRE, events.EVENT_TRAIN_OPTIMIZER_STEP_POST, step_ctx):
                    s.optimizer.step()
                if s.expert_bias_balancer is not None:
                    s.expert_bias_balancer.update()
                s.lr_scheduler.step()
                s.logger.log(run, loss_value=s.gradient_manager.compute_global_loss())
                if s.moe_aux_loss is not None and s.logger.is_due():
                    s.moe_aux_loss.log(run)
                if s.lm_loss is not None and s.logger.is_due():
                    s.lm_loss.log(run)
                s.gradient_manager.zero_grad()
                gc.collect_periodic()
                if profiler:
                    profiler.step()
                s.timeout_manager.set_periodic()
                s.event_bus.trigger(events.EVENT_TRAIN_STEP_POST, step_ctx)
                s.stepper.step()
                s.checkpointer.checkpoint_if_needed(s)
                bar.update()
                if s.stepper.current_step >= s.stepper.total_steps:
                    break
            s.checkpointer.wait_pending()
            s.logger.flush(run)
            s.task.finalize(control.FinalizeContext())
            s.event_bus.trigger(events.EVENT_TRAIN_FINISHED, events.EventTrainFinishedContext())

    def export(self, export_to: Path, load_checkpoint: bool) -> None:
        if load_checkpoint:
            self._state.checkpointer.load_last_checkpoint(self._state)
        self._state.exporter.export(Path(export_to))

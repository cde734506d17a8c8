"""Auxiliary-loss-free load balancing: the update rule on hand-made counts, two gloo ranks against one process, and the
Trainer option on a tiny DeepSeek-V3 (balancing, exact resume, unchanged checkpoint structure when off)."""

import pytest
import torch

from tests.dist_utils import run_distributed
from tests.helpers_train import LMProvider, SFTTask, SyntheticDataProvider, VOCAB, trainer_config


def _moe(E=4, k=2, bias=True, dtype=torch.float32):
    from d9d_b200.module.block.moe import MoELayer, RouterParameters

    layer = MoELayer(hidden_dim=16, intermediate_dim_grouped=8, num_grouped_experts=E, top_k=k, router_renormalize_probabilities=True,
                     router=RouterParameters(score_function="sigmoid", enable_expert_bias=bias))
    layer.reset_parameters()
    return layer.to(dtype)


def test_update_rule_on_hand_made_counts():
    from d9d_b200.module.block.moe import update_expert_bias

    biased, plain = _moe(), _moe(bias=False)
    biased.tokens_per_expert.copy_(torch.tensor([5, 1, 3, 3]))
    plain.tokens_per_expert.copy_(torch.tensor([7, 0, 1, 0]))
    plain_state = {k: v.clone() for k, v in plain.state_dict().items()}
    update_expert_bias([torch.nn.ModuleList([biased, plain])], 0.01)
    # mean 3: over-loaded expert 0 goes down, under-loaded expert 1 goes up, balanced experts stay
    assert biased.router.expert_bias.tolist() == pytest.approx([-0.01, 0.01, 0.0, 0.0])
    assert biased.tokens_per_expert.tolist() == [0, 0, 0, 0]
    # the layer without a bias is left alone, counter included
    assert plain.tokens_per_expert.tolist() == [7, 0, 1, 0]
    for k, v in plain.state_dict().items():
        assert torch.equal(v, plain_state[k]), k


def test_equal_counts_leave_the_bias_unchanged():
    from d9d_b200.module.block.moe import update_expert_bias

    layer = _moe()
    layer.router.expert_bias.copy_(torch.tensor([0.5, -0.25, 0.0, 1.0]))
    layer.tokens_per_expert.fill_(6)
    update_expert_bias([layer], 0.1)
    assert layer.router.expert_bias.tolist() == [0.5, -0.25, 0.0, 1.0]
    assert int(layer.tokens_per_expert.sum()) == 0


def test_uniform_overcounting_changes_nothing():
    from d9d_b200.module.block.moe import update_expert_bias

    once, twice = _moe(), _moe()
    once.tokens_per_expert.copy_(torch.tensor([4, 2, 1, 1]))
    twice.tokens_per_expert.copy_(torch.tensor([8, 4, 2, 2]))
    update_expert_bias([once], 1e-3)
    update_expert_bias([twice], 1e-3)
    assert torch.equal(once.router.expert_bias, twice.router.expert_bias)


def test_fp32_master_survives_a_bf16_buffer():
    from d9d_b200.module.block.moe import update_expert_bias
    from d9d_b200.module.block.moe.balancing import expert_bias_master

    layer = _moe(dtype=torch.bfloat16)
    assert layer.router.expert_bias.dtype == torch.bfloat16
    layer.router.expert_bias.fill_(0.5)
    for _ in range(10):
        layer.tokens_per_expert.copy_(torch.tensor([0, 2, 2, 2]))  # expert 0 under-loaded: +1e-3 per step
        update_expert_bias([layer], 1e-3)
    master = expert_bias_master(layer)
    assert master.dtype == torch.float32
    assert master[0].item() == pytest.approx(0.51, abs=1e-6)
    # a bf16 value at 0.5 cannot take a 1e-3 step (its spacing is 2^-8): without the master it would never have moved
    assert layer.router.expert_bias[0].item() == torch.tensor(0.51).bfloat16().item() != 0.5
    # weights loaded into the buffer from elsewhere become the new master
    layer.router.expert_bias.fill_(-1.0)
    layer.tokens_per_expert.fill_(3)
    update_expert_bias([layer], 1e-3)
    assert expert_bias_master(layer).tolist() == [-1.0] * 4


def _gloo_worker(rank, world, out, mesh_kwargs):
    import torch.distributed as dist

    from d9d_b200.core.dist_context import BATCH_DOMAIN, DeviceMeshParameters
    from d9d_b200.module.block.moe import update_expert_bias

    mesh = DeviceMeshParameters(**mesh_kwargs).build()
    torch.manual_seed(0)
    layer = _moe(E=8, k=2)
    x = torch.randn(2, 24, 16)
    group = mesh.mesh_for(BATCH_DOMAIN)["dp", "cp", "tp"]._flatten().get_group()  # noqa: SLF001
    for step in range(3):
        layer.reset_stats()
        with torch.no_grad():
            shard = x[:, step:step + 12] if "tensor_parallel" in mesh_kwargs else x[rank]
            layer(shard[None] if shard.dim() == 2 else shard)
        update_expert_bias([layer], 0.01, group)
    if rank == 0:
        torch.save(layer.router.expert_bias.clone(), out)
    dist.barrier()


@pytest.mark.dist
def test_two_data_parallel_ranks_match_one_process(tmp_path):
    from d9d_b200.module.block.moe import update_expert_bias

    out = tmp_path / "bias.pt"
    run_distributed(_gloo_worker, 2, str(out), {"data_parallel_replicate": 2})
    torch.manual_seed(0)
    layer = _moe(E=8, k=2)
    x = torch.randn(2, 24, 16)
    for _ in range(3):
        layer.reset_stats()
        with torch.no_grad():
            layer(x)  # the global batch: both ranks' tokens
        update_expert_bias([layer], 0.01)
    assert torch.equal(torch.load(out), layer.router.expert_bias)
    assert layer.router.expert_bias.abs().sum() > 0


def _deepseek_params():
    from d9d_b200.module.model.deepseek_v3 import (
        DeepseekV3ForCausalLMParameters,
        DeepseekV3LayerParameters,
        DeepseekV3Parameters,
        deepseek_v3_router,
    )

    layer = DeepseekV3LayerParameters.model_validate({
        "hidden_size": 32, "intermediate_size": 64, "moe_intermediate_size": 16, "num_attention_heads": 4,
        "rms_norm_eps": 1e-6, "kv_lora_rank": 16, "q_lora_rank": None, "qk_nope_head_dim": 8, "qk_rope_head_dim": 8,
        "v_head_dim": 8, "num_experts": 8, "experts_top_k": 2, "num_shared_experts": 1,
        "first_k_dense_replace": 1, "router_renormalize_probabilities": True,
        "router": deepseek_v3_router(n_group=4, topk_group=2, routed_scaling_factor=2.5).model_dump(),
    })
    return DeepseekV3ForCausalLMParameters(model=DeepseekV3Parameters(
        layer=layer, num_hidden_layers=3, rope_base=10000, max_position_ids=64, split_vocab_size=VOCAB,
        split_vocab_order=["regular", "special"]))


class _DeepseekProvider(LMProvider):
    def initialize_model_stage(self, context):
        from d9d_b200.model_state.mapper.adapters import identity_mapper_from_module
        from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode
        from d9d_b200.module.model.deepseek_v3 import DeepseekV3ForCausalLM
        from d9d_b200.loop.control import InitializeModelStageResult

        model = DeepseekV3ForCausalLM(self._params, context.stage, HiddenStatesAggregationMode.no, False).to(self._dtype)
        return InitializeModelStageResult(model=model, state_mapper=identity_mapper_from_module(model))

    def parallelize_model_stage(self, context):
        pass


def _deepseek_trainer(tmp, balancing=True, ckpt_period="disable"):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import AdamWOptimizerConfig
    from d9d_b200.loop.config import TrainerConfig
    from d9d_b200.loop.run import TrainingConfigurator

    cfg = trainer_config(tmp, ckpt_period=ckpt_period, log_dir=tmp / "logs").model_dump()
    cfg["gradient_manager"]["grad_dtype"] = None  # bf16 model, as the recipes cast it: bf16 gradients
    if balancing:
        cfg["expert_bias_balancing"] = {"update_rate": 1e-2}
    cfg = TrainerConfig.model_validate(cfg)
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=DeviceMeshParameters(), parameters=cfg, task_provider=lambda ctx: SFTTask(ctx.dist_context),
        model_provider=_DeepseekProvider(_deepseek_params(), dtype=torch.bfloat16), data_provider=SyntheticDataProvider(num_samples=48),
        optimizer_provider=AutoOptimizerProvider(AdamWOptimizerConfig(lr=3e-3, weight_decay=0.0)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched),
    ).configure()


def _biases(trainer):
    return {k: v.clone() for k, v in trainer.state.tracked_modules.modules[0].state_dict().items() if k.endswith("expert_bias")}


def _losses(tmp):
    import json

    (f,) = list((tmp / "logs").glob("*.jsonl"))
    return {r["step"]: r["value"] for r in map(json.loads, f.read_text().splitlines()) if r.get("name") == "loss"}


def test_trainer_balances_expert_bias_and_resumes_exactly(tmp_path):
    full = _deepseek_trainer(tmp_path / "full")
    biases = _biases(full)
    assert len(biases) == 2 and all(v.dtype == torch.bfloat16 and not v.any() for v in biases.values())
    counts = {}
    from d9d_b200.module.block.moe import MoELayer

    layers = [m for m in full.state.tracked_modules.modules[0].modules() if isinstance(m, MoELayer)]
    real_update = full.state.expert_bias_balancer.update

    def recording_update():
        counts.setdefault(len(counts), [layer.tokens_per_expert.clone() for layer in layers])
        real_update()

    full.state.expert_bias_balancer.update = recording_update
    full.train()
    trained = _biases(full)
    assert all(v.any() for v in trained.values())
    # every step's update pushes each expert against its own imbalance: the total signed movement of the biases opposes
    # the accumulated over-selection
    for i, name in enumerate(sorted(trained)):
        excess = sum((c[i] - c[i].float().mean()).float() for c in counts.values())
        assert float((trained[name].float() * excess).sum()) < 0, (name, excess, trained[name])

    class _Stop(Exception):
        pass

    from d9d_b200.loop.event.catalogue.train import EVENT_TRAIN_STEP_PRE

    part = _deepseek_trainer(tmp_path / "cut", ckpt_period=1)

    def stop_at_3(ctx):
        if ctx.stepper.current_step == 3:
            raise _Stop

    part.state.event_bus.subscribe(EVENT_TRAIN_STEP_PRE, stop_at_3)
    with pytest.raises(_Stop):
        part.train()
    resumed = _deepseek_trainer(tmp_path / "cut", ckpt_period=1)
    resumed.train()
    for name, value in _biases(resumed).items():
        assert torch.equal(value, trained[name]), name
    full_masters = full.state.expert_bias_balancer.state_dict()["masters"]
    for name, value in resumed.state.expert_bias_balancer.state_dict()["masters"].items():
        assert torch.equal(value, full_masters[name]), name
    ref_losses, got_losses = _losses(tmp_path / "full"), _losses(tmp_path / "cut")
    assert all(got_losses[s] == ref_losses[s] for s in ref_losses if s >= 3) and len(ref_losses) == 6


def test_balancing_off_keeps_the_checkpoint_structure(tmp_path):
    from d9d_b200.loop.state import TrainJobState

    off = _deepseek_trainer(tmp_path / "off", balancing=False)
    assert off.state.expert_bias_balancer is None
    keys = set(off.state.state_dict())
    assert keys == {"stepper", "tracked_modules", "data_loader", "logger", "task", "metrics", "optimizer", "lr_scheduler"}
    assert keys == set(TrainJobState.CHECKPOINTED) - {"expert_bias_balancer"}
    off.train()
    assert all(not v.any() for v in _biases(off).values())  # nothing moves the bias when balancing is off
    on = _deepseek_trainer(tmp_path / "on")
    assert set(on.state.state_dict()) == keys | {"expert_bias_balancer"}

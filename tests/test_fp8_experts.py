"""fp8 expert block on CPU: the PyTorch emulation of the recipe against fp64 products of its own quantised operands, the
quantiser emulations' rules, and the Trainer option ``model_stage_factory.fp8_experts`` (refusals, conversion, training,
exact resume, and bitwise-unchanged training when it is off)."""

import pytest
import torch

from d9d_b200.kernel import fp8
from d9d_b200.kernel.moe import fp8_grouped_linear_reference, grouped_swiglu_fp8_reference

from .helpers_train import LMProvider, SFTTask, SyntheticDataProvider, moe_params, trainer_config


def _deq_rows(x):
    q, s = fp8.quantize_rowwise_reference(x)
    return q.double() * s.double()[:, None]


def test_segment_quantiser_emulation_zeroes_pads_and_scales_empty_experts():
    x = torch.randn(512, 24).bfloat16()
    x[5:128] = float("nan")  # pad rows of expert 0 (1 token)
    qt, s = fp8.quantize_segments_t_reference(x, [0, 128, 128, 384], [1, 0, 200, 0])
    assert qt.shape == (24, 512) and s.shape == (4, 24)
    assert (s[1] == 1).all() and (s[3] == 1).all()
    assert not qt[:, 1:128].float().any() and not qt[:, 328:].float().any()
    torch.testing.assert_close(qt[:, 128:328].float() * s[2][:, None], x[128:328].float().t(), rtol=0.07, atol=0)
    qb, sb = fp8.quantize_colwise_t_batched_reference(x[:384].view(3, 128, 24))
    assert qb.shape == (3, 24, 128) and torch.equal(qb[1].float(), fp8.quantize_colwise_t_reference(x[128:256])[0].float())


def test_emulated_grouped_linear_matches_fp64_on_its_quantised_operands():
    torch.manual_seed(0)
    starts, counts = [0, 128, 256, 384], [100, 0, 128, 7]
    x = torch.randn(512, 64, dtype=torch.float64).bfloat16().requires_grad_()
    w = (torch.randn(4, 64, 48) * 0.1).bfloat16().requires_grad_()
    y = fp8_grouped_linear_reference(x, w, starts, counts)
    dy = torch.randn(512, 48).bfloat16()
    y.backward(dy)
    for e, (s0, n) in enumerate(zip(starts, counts)):
        rows = slice(s0, s0 + n)
        if n == 0:
            assert not w.grad[e].any()
            continue
        # forward: Q_row(x) . Q_colT(W[e]); dgrad: Q_row(dy) . Q_row(W[e])^T; wgrad: Q_seg(x)^T . Q_seg(dy)
        y64 = _deq_rows(x[rows].detach()) @ _deq_rows(w[e].detach().t()).t()
        dx64 = _deq_rows(dy[rows]) @ _deq_rows(w[e].detach()).t()
        dw64 = _deq_rows(x[rows].detach().t()) @ _deq_rows(dy[rows].t()).t()
        for got, want in ((y[rows], y64), (x.grad[rows], dx64), (w.grad[e], dw64)):
            torch.testing.assert_close(got.double(), want, rtol=2**-7, atol=1e-6 * float(want.abs().max()))
    pads = torch.ones(512, dtype=torch.bool)
    for s0, n in zip(starts, counts):
        pads[s0 : s0 + n] = False
    assert not y[pads].any() and not x.grad[pads].any()


def test_emulated_block_close_to_exact_block():
    torch.manual_seed(0)
    starts, counts = [0, 128, 256], [90, 128, 30]
    xp = torch.randn(384, 64)
    pp = torch.rand(384)
    w = [torch.randn(3, a, b) * 0.1 for a, b in ((64, 32), (64, 32), (32, 64))]
    leaves = [xp.clone().requires_grad_(), pp.clone().requires_grad_()] + [t.clone().requires_grad_() for t in w]
    y = grouped_swiglu_fp8_reference(*leaves, starts, counts)
    y.square().sum().backward()
    exact = [t.detach().double().requires_grad_() for t in (xp, pp, *w)]
    out = torch.zeros(384, 64, dtype=torch.float64)
    for e, (s0, n) in enumerate(zip(starts, counts)):
        r = slice(s0, s0 + n)
        h = torch.nn.functional.silu(exact[0][r] @ exact[2][e]) * (exact[0][r] @ exact[3][e]) * exact[1][r, None]
        out = out.index_put((torch.arange(s0, s0 + n),), h @ exact[4][e])
    out.square().sum().backward()
    for a, b in zip([y] + [t.grad for t in leaves], [out] + [t.grad for t in exact]):
        assert float((a.double() - b).norm() / b.norm()) < 0.08


def test_grouped_swiglu_module_fp8_flag_and_refusals():
    from d9d_b200.module.block.moe import GroupedSwiGLU

    m = GroupedSwiGLU(64, 32, 3)
    m.enable_fp8()
    assert m.fp8
    x, p = torch.randn(40, 64), torch.rand(40)
    y = m(x, p, torch.tensor([10, 0, 30]))  # composed per-expert path -> emulation of the recipe
    assert y.shape == (40, 64) and torch.isfinite(y).all()
    with pytest.raises(ValueError, match="multiples of 16"):
        GroupedSwiGLU(64, 24, 3).enable_fp8()
    wrapped = GroupedSwiGLU(64, 32, 3)
    wrapped.gate_proj = torch.nn.Identity()  # stands in for an adapter-wrapped projection
    with pytest.raises(ValueError, match="LoRA"):
        wrapped.enable_fp8()


# ------------------------------------------------------------------------------------------ Trainer option
def _trainer(tmp, fp8_experts, moe=None, ckpt_period="disable", mesh=None, provider=None):
    """``fp8_experts=None`` leaves the option unset (the configuration a job without it has)."""
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import AdamWOptimizerConfig
    from d9d_b200.loop.run import TrainingConfigurator

    cfg = trainer_config(tmp, log_dir=tmp / "logs", ckpt_period=ckpt_period)
    if fp8_experts is not None:
        cfg.model_stage_factory.fp8_experts = fp8_experts
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=mesh or DeviceMeshParameters(), parameters=cfg, task_provider=lambda ctx: SFTTask(ctx.dist_context),
        model_provider=provider or LMProvider(moe or moe_params(2), moe=True), data_provider=SyntheticDataProvider(num_samples=64),
        optimizer_provider=AutoOptimizerProvider(AdamWOptimizerConfig(lr=3e-3, weight_decay=0.0)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched)).configure()


def _losses(tmp):
    from .test_trainer import _read_losses

    return _read_losses(tmp)[0]


def test_fp8_experts_off_is_bitwise_today_and_on_trains(tmp_path):
    from d9d_b200.module.block.moe import GroupedSwiGLU

    off = _trainer(tmp_path / "off", False)
    assert not any(m.fp8 for m in off.state.tracked_modules.modules[0].modules() if isinstance(m, GroupedSwiGLU))
    off.train()
    default = _trainer(tmp_path / "default", None)
    assert "fp8_experts" not in trainer_config(tmp_path / "x").model_stage_factory.model_fields_set  # the unset arm
    default.train()
    assert _losses(tmp_path / "off") == _losses(tmp_path / "default")

    on = _trainer(tmp_path / "on", True)
    blocks = [m for m in on.state.tracked_modules.modules[0].modules() if isinstance(m, GroupedSwiGLU)]
    assert blocks and all(b.fp8 for b in blocks)
    on.train()
    losses = _losses(tmp_path / "on")
    assert losses[max(losses)] < losses[min(losses)]


def test_fp8_experts_refuses_sizes_and_tensor_parallelism(tmp_path):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.module.model.qwen3_moe import Qwen3MoEForCausalLMParameters, Qwen3MoELayerParameters, Qwen3MoEParameters

    from .helpers_train import VOCAB

    odd = Qwen3MoEForCausalLMParameters(model=Qwen3MoEParameters(
        layer=Qwen3MoELayerParameters(hidden_size=32, intermediate_size=24, num_experts=4, experts_top_k=2, num_attention_heads=4,
                                      num_key_value_heads=2, rms_norm_eps=1e-6, head_dim=8),
        num_hidden_layers=1, rope_base=10000, max_position_ids=64, split_vocab_size=VOCAB,
        split_vocab_order=["regular", "special"]))
    with pytest.raises(ValueError, match="multiples of 16"):
        _trainer(tmp_path / "odd", True, moe=odd)
    # tensor parallelism: the factory's conversion step against a stand-in context of a TP-2 mesh
    from types import SimpleNamespace

    from d9d_b200.loop.component.model_stage_factory import ModelStageFactory
    from d9d_b200.module.block.moe import GroupedSwiGLU

    factory = ModelStageFactory.__new__(ModelStageFactory)
    factory._config_model = SimpleNamespace(fp8_experts=True)
    factory._ctx = SimpleNamespace(mesh_params=DeviceMeshParameters(tensor_parallel=2), logger=None)
    block = GroupedSwiGLU(32, 16, 4)
    with pytest.raises(NotImplementedError, match="tensor parallelism"):
        factory._apply_fp8_experts(torch.nn.Sequential(block))
    assert not block.fp8


def test_fp8_experts_resumes_exactly(tmp_path):
    from d9d_b200.loop.event.catalogue.train import EVENT_TRAIN_STEP_PRE

    full = _trainer(tmp_path / "a", True)
    full.train()
    want = {k: v.clone() for k, v in full.state.tracked_modules.modules[0].state_dict().items()}

    class _Stop(Exception):
        pass

    part = _trainer(tmp_path / "b", True, ckpt_period=1)

    def stop_at_3(ctx):
        if ctx.stepper.current_step == 3:
            raise _Stop

    part.state.event_bus.subscribe(EVENT_TRAIN_STEP_PRE, stop_at_3)
    with pytest.raises(_Stop):
        part.train()
    resumed = _trainer(tmp_path / "b", True, ckpt_period=1)
    resumed.train()
    for k, v in resumed.state.tracked_modules.modules[0].state_dict().items():
        torch.testing.assert_close(v, want[k], rtol=0, atol=0, msg=lambda m, k=k: f"{k}: {m}")


def test_fp8_experts_refuses_lora_on_the_experts(tmp_path):
    from d9d_b200.loop.control import InitializeModelStageResult
    from d9d_b200.model_state.mapper.compose import ModelStateMapperSequential
    from d9d_b200.peft import inject_peft_and_freeze
    from d9d_b200.peft.all import peft_method_from_config
    from d9d_b200.peft.lora.config import LoRAConfig

    class ExpertLoRAProvider(LMProvider):
        def initialize_model_stage(self, context):
            built = super().initialize_model_stage(context)
            method = peft_method_from_config(LoRAConfig.model_validate(
                {"kind": "lora", "module_name_pattern": r".*grouped_experts\.(gate_proj|up_proj)",
                 "params": {"r": 4, "alpha": 8, "dropout": 0.0}}))
            redirect = inject_peft_and_freeze(method, built.model)
            return InitializeModelStageResult(model=built.model, state_mapper=ModelStateMapperSequential([built.state_mapper, redirect]))

    with pytest.raises(ValueError, match="LoRA"):
        _trainer(tmp_path / "lora", True, provider=ExpertLoRAProvider(moe_params(2), moe=True))

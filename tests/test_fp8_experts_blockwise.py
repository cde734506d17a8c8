"""The blockwise fp8 recipe of the MoE expert block on CPU: the quantiser emulations against the fp64 models of
``fp8_reference``, token groups that stay inside expert segments, the emulated grouped linear against fp64 products of its
own quantised operands, the outlier property that motivates the recipe, the module's recipe switch and the Trainer option
``model_stage_factory.fp8_experts_recipe``."""

import pytest
import torch

from d9d_b200.kernel import fp8
from d9d_b200.kernel.moe import fp8_grouped_linear_reference, grouped_swiglu_fp8_reference

from .fp8_reference import assert_codes_admissible, check_scales, flush
from .helpers_train import LMProvider, SFTTask, SyntheticDataProvider, moe_params, trainer_config

E4M3_MIN_NORMAL = 2.0**-6


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def _blocks_amax(w, rows_per_group, cols_per_group):
    """amax of every rows_per_group x cols_per_group block of the 2-D ``w`` (fp64, flushed), repeated to ``w``'s shape."""
    R, C = w.shape
    Rb, Cb = -(-R // rows_per_group), -(-C // cols_per_group)
    pad = torch.nn.functional.pad(flush(w).abs(), (0, Cb * cols_per_group - C, 0, Rb * rows_per_group - R))
    amax = pad.view(Rb, rows_per_group, Cb, cols_per_group).amax(dim=(1, 3))
    return amax.repeat_interleave(rows_per_group, 0).repeat_interleave(cols_per_group, 1)[:R, :C]


def test_expert_weight_blocks_follow_the_scale_rule_in_both_orientations():
    torch.manual_seed(0)
    E, n_in, n_out = 3, 272, 160  # tails in both dims
    w = (torch.randn(E, n_in, n_out) * torch.logspace(-30, 30, E, base=2)[:, None, None]).bfloat16()
    w[1, :128, :128] = 0  # an all-zero block: scale 1
    qt, st = fp8.quantize_expert_weight_blocks_reference(w, True)
    q, s = fp8.quantize_expert_weight_blocks_reference(w, False)
    assert qt.shape == (E, n_out, n_in) and st.shape == (E, 3, n_out)
    assert q.shape == (E, n_in, n_out) and s.shape == (E, 2, n_in)
    for e in range(E):
        assert torch.equal(qt[e].view(torch.uint8), q[e].t().view(torch.uint8))  # one block scale, both copies
        amax = _blocks_amax(w[e].float(), 128, 128)  # [in, out]
        # plain copy: s[e, out-block, in-row]; transposed: s[e, in-block, out-row]
        s_full = s[e].t().repeat_interleave(128, dim=1)[:, :n_out]
        st_full = st[e].repeat_interleave(128, dim=0)[:n_in]
        check_scales(s_full, amax, f"expert {e} plain")
        check_scales(st_full, amax, f"expert {e} transposed")
        assert torch.equal(s_full, st_full)
        assert_codes_admissible(w[e], q[e], s_full, f"expert {e}")
    assert (st[1, 0, :128] == 1).all()


def test_token_groups_stay_inside_expert_segments_and_pads_quantise_to_zero():
    torch.manual_seed(1)
    starts, counts = [0, 128, 384, 512], [1, 200, 0, 128]
    x = torch.randn(768, 48).bfloat16()
    x[1:128] = float("nan")  # pad rows of expert 0
    x[328:384] = 1e30  # pad rows of expert 1
    x[640:] = float("nan")  # unused capacity
    qt, st = fp8.quantize_blockwise_segments_t_reference(x, starts, counts)
    assert qt.shape == (48, 768) and st.shape == (6, 48)
    valid = torch.zeros(768, dtype=torch.bool)
    for s0, n in zip(starts, counts):
        valid[s0 : s0 + n] = True
    assert not qt.float()[:, ~valid].any()
    xv = torch.where(valid[:, None], x.float(), torch.zeros(()))
    for g in range(6):  # every 128-token group lies in one segment (segments start on 128-row boundaries)
        rows = slice(128 * g, 128 * g + 128)
        amax = flush(xv[rows]).abs().amax(dim=0)
        check_scales(st[g], amax, f"group {g}")
        assert_codes_admissible(xv[rows].t(), qt[:, rows], st[g][:, None], f"group {g}")
    assert (st[3] == 1).all() and (st[5] == 1).all()  # no rows: scale 1
    q, s = fp8.quantize_blockwise_segments_reference(x, starts, counts)
    assert q.shape == (768, 48) and s.shape == (1, 768)
    assert not q.float()[~valid].any() and (s[0, ~valid] == 1).all()
    assert_codes_admissible(xv, q, s.t(), "row groups")


def _deq_blockwise_rows(x):
    q, s = fp8.quantize_blockwise_reference(x)
    return q.double() * s.double().t().repeat_interleave(128, dim=1)[:, : x.shape[1]]


def _blockwise_product(aq, sa, bq, sb):
    """fp64 sum over 128-deep k-blocks of exact products times the block scales (the promoted accumulation)."""
    K = aq.shape[1]
    out = torch.zeros(aq.shape[0], bq.shape[0], dtype=torch.float64)
    for kb in range(-(-K // 128)):
        ks = slice(128 * kb, min(K, 128 * kb + 128))
        out += (aq[:, ks].double() @ bq[:, ks].double().t()) * sa[kb].double()[:, None] * sb[kb].double()[None, :]
    return out


def test_emulated_grouped_linear_matches_fp64_on_its_quantised_operands():
    torch.manual_seed(2)
    starts, counts = [0, 128, 384, 512], [100, 0, 128, 7]
    n_in, n_out = 144, 272  # K and N tails
    x = torch.randn(640, n_in).bfloat16().requires_grad_()
    w = (torch.randn(4, n_in, n_out) * 0.1).bfloat16().requires_grad_()
    y = fp8_grouped_linear_reference(x, w, starts, counts, recipe="blockwise")
    dy = torch.randn(640, n_out).bfloat16()
    y.backward(dy)
    for e, (s0, n) in enumerate(zip(starts, counts)):
        rows = slice(s0, s0 + n)
        if n == 0:
            assert not w.grad[e].any()
            continue
        xe, we = x[rows].detach(), w[e].detach()
        y64 = _blockwise_product(*fp8.quantize_blockwise_reference(xe), *fp8.quantize_weight_blocks_reference(we, True))
        dx64 = _blockwise_product(*fp8.quantize_blockwise_reference(dy[rows]), *fp8.quantize_weight_blocks_reference(we))
        dw64 = _blockwise_product(*fp8.quantize_blockwise_t_reference(xe), *fp8.quantize_blockwise_t_reference(dy[rows]))
        for got, want in ((y[rows], y64), (x.grad[rows], dx64), (w.grad[e], dw64)):
            torch.testing.assert_close(got.double(), want, rtol=2**-7, atol=1e-5 * float(want.abs().max()))
        # and close to the exact product of the bf16 operands
        assert _rel(y[rows], xe.double() @ we.double()) < 0.08
    pads = torch.ones(640, dtype=torch.bool)
    for s0, n in zip(starts, counts):
        pads[s0 : s0 + n] = False
    assert not y[pads].any() and not x.grad[pads].any()


def test_unknown_recipes_are_refused():
    x, w = torch.randn(128, 16).bfloat16(), torch.randn(1, 16, 16).bfloat16()
    with pytest.raises(ValueError, match="unknown fp8 expert recipe"):
        fp8_grouped_linear_reference(x, w, [0], [128], recipe="mx")
    with pytest.raises(ValueError, match="unknown fp8 expert recipe"):
        grouped_swiglu_fp8_reference(x, torch.rand(128), w, w, w, [0], [128], recipe="tensorwise")


def test_an_outlier_token_only_costs_its_own_token_group():
    """One token of one expert 2^16 times the typical magnitude in every channel: under the blockwise recipe the expert's
    other 128-token groups keep e4m3 precision; the row-wise segment quantiser (one scale per channel over all of the
    expert's tokens) pushes them below e4m3's smallest normal."""
    torch.manual_seed(3)
    starts, counts = [0, 512], [500, 60]
    x = torch.randn(640, 32)
    x[500:512] = 0  # pad rows
    x[10] = 2.0**16  # expert 0, token group 0
    qt, st = fp8.quantize_blockwise_segments_t_reference(x, starts, counts)
    deq = qt.float() * st.repeat_interleave(128, dim=0).t()
    for g in (1, 2):
        rows = slice(128 * g, 128 * g + 128)
        assert _rel(deq[:, rows], x[rows].t()) < 0.04
    typical = x[:500].abs() <= 2  # within two standard deviations: 2 * 448 / 2^16 < 2^-6
    assert torch.all(qt[:, :128].float().t()[typical[:128]].abs() < E4M3_MIN_NORMAL)  # the outlier's own group pays
    qr, _ = fp8.quantize_segments_t_reference(x, starts, counts)
    assert torch.all(qr[:, 128:500].float().t()[typical[128:500]].abs() < E4M3_MIN_NORMAL)
    # the other expert is untouched by either recipe
    assert _rel(deq[:, 512:572], x[512:572].t()) < 0.04


def test_module_recipe_switch_and_refusals():
    from d9d_b200.module.block.moe import GroupedSwiGLU

    m = GroupedSwiGLU(64, 32, 3)
    m.enable_fp8()
    assert m.fp8 and m.fp8_recipe == "rowwise"
    b = GroupedSwiGLU(64, 32, 3)
    b.load_state_dict(m.state_dict())
    b.enable_fp8("blockwise")
    assert b.fp8 and b.fp8_recipe == "blockwise"
    x, p, groups = torch.randn(40, 64), torch.rand(40), torch.tensor([10, 0, 30])
    ym, yb = m(x, p, groups), b(x, p, groups)  # composed per-expert path -> emulation of each recipe
    assert yb.shape == (40, 64) and torch.isfinite(yb).all() and not torch.equal(ym, yb)
    starts, counts = [0, 10, 10], [10, 0, 30]
    ref = grouped_swiglu_fp8_reference(x, p, b.gate_proj.weight, b.up_proj.weight, b.down_proj.weight, starts, counts, "blockwise")
    assert torch.equal(yb, ref)
    with pytest.raises(ValueError, match="unknown recipe"):
        GroupedSwiGLU(64, 32, 3).enable_fp8("mx")
    with pytest.raises(ValueError, match="multiples of 16"):
        GroupedSwiGLU(64, 24, 3).enable_fp8("blockwise")
    wrapped = GroupedSwiGLU(64, 32, 3)
    wrapped.gate_proj = torch.nn.Identity()  # stands in for an adapter-wrapped projection
    with pytest.raises(ValueError, match="LoRA"):
        wrapped.enable_fp8("blockwise")
    assert not wrapped.fp8


# ------------------------------------------------------------------------------------------ Trainer option
def _trainer(tmp, recipe=None):
    """``recipe=None`` leaves ``fp8_experts_recipe`` unset (the configuration a job without it has)."""
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import AdamWOptimizerConfig
    from d9d_b200.loop.run import TrainingConfigurator

    cfg = trainer_config(tmp, log_dir=tmp / "logs")
    cfg.model_stage_factory.fp8_experts = True
    if recipe is not None:
        cfg.model_stage_factory.fp8_experts_recipe = recipe
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=DeviceMeshParameters(), parameters=cfg, task_provider=lambda ctx: SFTTask(ctx.dist_context),
        model_provider=LMProvider(moe_params(2), moe=True), data_provider=SyntheticDataProvider(num_samples=64),
        optimizer_provider=AutoOptimizerProvider(AdamWOptimizerConfig(lr=3e-3, weight_decay=0.0)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched)).configure()


def _losses(tmp):
    from .test_trainer import _read_losses

    return _read_losses(tmp)[0]


def _blocks(trainer):
    from d9d_b200.module.block.moe import GroupedSwiGLU

    return [m for m in trainer.state.tracked_modules.modules[0].modules() if isinstance(m, GroupedSwiGLU)]


def test_trainer_recipe_option(tmp_path):
    from d9d_b200.loop.config.config import ModelStageFactoryConfig

    assert ModelStageFactoryConfig.model_fields["fp8_experts_recipe"].default == "rowwise"
    default = _trainer(tmp_path / "default")
    assert all(b.fp8 and b.fp8_recipe == "rowwise" for b in _blocks(default))
    default.train()
    rowwise = _trainer(tmp_path / "rowwise", "rowwise")
    rowwise.train()
    assert _losses(tmp_path / "default") == _losses(tmp_path / "rowwise")  # the option absent: row-wise, bitwise

    blockwise = _trainer(tmp_path / "blockwise", "blockwise")
    blocks = _blocks(blockwise)
    assert blocks and all(b.fp8 and b.fp8_recipe == "blockwise" for b in blocks)
    blockwise.train()
    losses = _losses(tmp_path / "blockwise")
    assert losses[max(losses)] < losses[min(losses)]
    assert losses != _losses(tmp_path / "rowwise")
    with pytest.raises(ValueError):
        _trainer(tmp_path / "mx", "mx")

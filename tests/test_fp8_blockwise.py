"""The blockwise fp8 recipe on CPU: scale rules of the quantiser emulations, the outlier property that motivates it,
the emulated linear layer's autograd (joint backward, and the split backward of all three recipes) and a Trainer run with
``Fp8LinearConfig(recipe="blockwise")``."""

import pytest
import torch

from d9d_b200.kernel import fp8

E4M3_MIN_NORMAL = 2.0**-6


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def test_row_groups_cover_partial_tails_and_zero_groups():
    torch.manual_seed(0)
    x = torch.randn(5, 200)
    x[2] = 0
    x[3, 128:] = 0
    q, s = fp8.quantize_blockwise_reference(x)
    assert q.shape == (5, 200) and q.dtype == fp8.FP8 and s.shape == (2, 5)
    assert torch.equal(s[0], x[:, :128].abs().amax(dim=1) / 448 + (x[:, :128].abs().amax(dim=1) == 0).float())
    # the tail group has 72 valid elements: its scale is their amax
    assert torch.allclose(s[1, [0, 1, 4]], x[[0, 1, 4], 128:].abs().amax(dim=1) / 448, rtol=0, atol=0)
    assert s[0, 2] == 1 and s[1, 2] == 1 and s[1, 3] == 1 and not q[2].float().any() and not q[3, 128:].float().any()
    deq = q.float().view(5, 200) * s.t().repeat_interleave(128, dim=1)[:, :200]
    assert _rel(deq, x) < 0.04


def test_token_groups_are_the_row_groups_of_the_transpose():
    torch.manual_seed(1)
    x = torch.randn(130, 48)  # 130 tokens: a 2-token tail group per channel
    qt, s = fp8.quantize_blockwise_t_reference(x)
    assert qt.shape == (48, 130) and s.shape == (2, 48)
    assert torch.equal(s[1], x[128:].abs().amax(dim=0) / 448)
    q2, s2 = fp8.quantize_blockwise_reference(x.t().contiguous())
    assert torch.equal(qt.view(torch.uint8), q2.view(torch.uint8)) and torch.equal(s, s2)


def test_weight_block_scales_are_constant_per_128x128_block_and_transposes_are_bitwise():
    torch.manual_seed(2)
    w = torch.randn(272, 400) * torch.logspace(-1, 1, 272)[:, None]
    q, s = fp8.quantize_weight_blocks_reference(w)
    qt, st = fp8.quantize_weight_blocks_reference(w, transpose=True)
    assert q.shape == (272, 400) and s.shape == (4, 272) and qt.shape == (400, 272) and st.shape == (3, 400)
    for nb in range(3):
        rows = slice(nb * 128, min(272, nb * 128 + 128))
        for kb in range(4):
            cols = slice(kb * 128, min(400, kb * 128 + 128))
            block = w[rows, cols].abs().amax() / 448
            assert torch.all(s[kb, rows] == block)  # repeated on each of the block's rows
            assert torch.all(st[nb, cols] == block)  # and on each row of the transposed copy
    assert torch.equal(qt.view(torch.uint8), q.view(torch.uint8).t())


def test_an_outlier_only_costs_its_own_group():
    """Values 2^16 times the typical magnitude in one 128-group of a row: blockwise keeps the row's other groups at e4m3
    precision, one scale per row pushes them below e4m3's smallest normal (subnormal or zero)."""
    torch.manual_seed(3)
    x = torch.randn(16, 512)
    x[5, 10:13] = 2.0**16
    qb, sb = fp8.quantize_blockwise_reference(x)
    deq = qb.float() * sb.t().repeat_interleave(128, dim=1)
    assert _rel(deq[5, 128:], x[5, 128:]) < 0.04
    typical = x[5].abs() <= 2  # within two standard deviations: 2 * 448 / 2^16 < 2^-6
    assert torch.all(qb[5, :128][typical[:128]].float().abs() < E4M3_MIN_NORMAL)  # the outlier's own group pays
    qr, _ = fp8.quantize_rowwise_reference(x)
    assert torch.all(qr[5, 128:][typical[128:]].float().abs() < E4M3_MIN_NORMAL)
    # the same along tokens, for the weight gradient's operands: one channel, one 128-token group
    xt = torch.randn(384, 32)
    xt[200, 7] = 2.0**16
    qt, st = fp8.quantize_blockwise_t_reference(xt)
    deq_t = qt.float() * st.t().repeat_interleave(128, dim=1)
    assert _rel(deq_t[7, :128], xt[:128, 7]) < 0.04 and _rel(deq_t[7, 256:], xt[256:, 7]) < 0.04


def test_blockwise_mm_reference_promotes_every_k_block():
    torch.manual_seed(4)
    a, b = torch.randn(40, 300), torch.randn(24, 300)
    aq, sa = fp8.quantize_blockwise_reference(a)
    bq, sb = fp8.quantize_weight_blocks_reference(b)
    want = torch.zeros(40, 24, dtype=torch.float64)
    for kb in range(3):
        ks = slice(kb * 128, min(300, kb * 128 + 128))
        want += (aq[:, ks].double() * sa[kb].double()[:, None]) @ (bq[:, ks].double() * sb[kb].double()[:, None]).t()
    got = fp8.blockwise_mm(aq, sa, bq, sb, out_dtype=torch.float32)
    assert got.dtype == torch.float32 and torch.allclose(got.double(), want, rtol=1e-5, atol=1e-4)
    assert _rel(got, a @ b.t()) < 0.06


def _layer_inputs(seed=5):
    torch.manual_seed(seed)
    x = torch.randn(3, 50, 256)  # 150 tokens: not a multiple of 128
    w = torch.randn(144, 256) * 0.05  # out 144: a partial 128-row weight block
    return x, w


def test_blockwise_linear_autograd_close_to_fp32():
    x, w = _layer_inputs()
    x1, w1 = x.clone().requires_grad_(), w.clone().requires_grad_()
    y = fp8.fp8_linear(x1, w1, recipe="blockwise")
    g = torch.randn(y.shape)
    y.float().backward(g)
    x2, w2 = x.clone().requires_grad_(), w.clone().requires_grad_()
    y2 = x2 @ w2.t()
    y2.backward(g)
    assert y.shape == (3, 50, 144)
    assert _rel(y, y2) < 0.05
    assert _rel(x1.grad, x2.grad) < 0.06
    assert _rel(w1.grad, w2.grad) < 0.06


def _assert_split_backward_equals_the_joint_backward(recipe, x, w):
    from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection

    g = torch.randn(*x.shape[:-1], w.shape[0])
    x1, w1 = x.clone().requires_grad_(), w.clone().requires_grad_()
    fp8.fp8_linear(x1, w1, recipe=recipe).float().backward(g)
    x2, w2 = x.clone().requires_grad_(), w.clone().requires_grad_()
    y = fp8.fp8_linear(x2, w2, recipe=recipe).float()
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.inputs):
        y.backward(g, retain_graph=True)
    assert w2.grad is None and torch.equal(x2.grad, x1.grad)
    x2.grad = None
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.weight):
        y.backward(g)
    assert x2.grad is None and torch.equal(w2.grad, w1.grad)


def test_split_backward_equals_the_joint_backward():
    _assert_split_backward_equals_the_joint_backward("blockwise", *_layer_inputs(6))


@pytest.mark.parametrize("recipe", ["rowwise", "mx"])
def test_split_backward_of_the_other_recipes_equals_the_joint_backward(recipe):
    """The fp8 linear layer runs every recipe through one autograd function: the same split backward for each."""
    if recipe == "mx":  # token and feature counts multiples of 128
        torch.manual_seed(6)
        x, w = torch.randn(2, 128, 256), torch.randn(128, 256) * 0.05
    else:
        x, w = _layer_inputs(6)
    _assert_split_backward_equals_the_joint_backward(recipe, x, w)


def test_blockwise_sizes_and_conversion():
    w = torch.randn(48, 40)
    with pytest.raises(ValueError):
        fp8.fp8_linear(torch.randn(3, 40), w, recipe="blockwise")  # in = 40: not a multiple of 16
    assert fp8.fp8_linear(torch.randn(7, 48), torch.randn(32, 48), recipe="blockwise").shape == (7, 32)  # 7 tokens are fine
    with pytest.raises(ValueError):
        fp8.fp8_linear(torch.randn(7, 48), torch.randn(32, 48), recipe="block")
    m = torch.nn.Sequential(torch.nn.Linear(32, 48), torch.nn.ReLU(), torch.nn.Linear(48, 10))
    assert fp8.convert_linears_to_fp8(m, recipe="blockwise") == 1 and m[0].fp8_recipe == "blockwise" and type(m[2]) is torch.nn.Linear
    assert m(torch.randn(5, 32)).shape == (5, 10)


def test_trainer_with_the_blockwise_recipe(tmp_path):
    """``Fp8LinearConfig(recipe="blockwise")`` converts the selected projections and the job trains (emulation on CPU)."""
    import json

    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.kernel.fp8 import Fp8Linear
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import AdamWOptimizerConfig
    from d9d_b200.loop.config import Fp8LinearConfig
    from d9d_b200.loop.run import TrainingConfigurator
    from tests.helpers_train import LMProvider, SFTTask, SyntheticDataProvider, dense_params, trainer_config

    cfg = trainer_config(tmp_path, log_dir=tmp_path / "logs")
    cfg.model_stage_factory.fp8_linear = Fp8LinearConfig(include=r"self_attn|mlp", recipe="blockwise")
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    trainer = TrainingConfigurator(
        mesh=DeviceMeshParameters(), parameters=cfg, task_provider=lambda ctx: SFTTask(ctx.dist_context),
        model_provider=LMProvider(dense_params(2)), data_provider=SyntheticDataProvider(num_samples=64),
        optimizer_provider=AutoOptimizerProvider(AdamWOptimizerConfig(lr=3e-3, weight_decay=0.0)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched)).configure()
    model = trainer.state.tracked_modules.modules[0]
    converted = [m for m in model.modules() if isinstance(m, Fp8Linear)]
    assert converted and all(m.fp8_recipe == "blockwise" for m in converted)
    trainer.train()
    files = list((tmp_path / "logs").glob("*.jsonl"))
    assert len(files) == 1
    losses = {r["step"]: r["value"] for r in map(json.loads, files[0].read_text().splitlines()) if r.get("name") == "loss"}
    assert losses[max(losses)] < losses[min(losses)]

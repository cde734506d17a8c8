"""The sequence-wise balance loss on the PyTorch path (the numerics oracle of the fused kernels): the definition on
hand-made inputs, the attached gradient against autograd on an fp64 transcription of DeepSeek-V3 eqs. 17-20 for softmax
and sigmoid routers under every routing option, refused inputs and meshes, token weighting and activation recomputation,
and the Trainer option: a DeepSeek-V3-style run that logs and trains it, bitwise unchanged when its coefficient is 0, and
a two-stage pipeline run equal to one process."""

import json

import pytest
import torch

from d9d_b200.kernel.router import route_topk
from tests.dist_utils import run_distributed

W_TOK = 1e-3


def _seq_objective_fp64(logits, chosen, k, S, coef, w, score_function):
    """``w S coef sum_b A_b`` and ``A [B]`` from the written definition, in fp64 (``chosen`` carries no gradient)."""
    x = logits.double().reshape(-1, logits.shape[-1])
    T, E = x.shape
    B = T // S
    if score_function == "softmax":
        s = torch.softmax(x, dim=-1)
    else:
        sig = torch.sigmoid(x)
        s = sig / sig.sum(-1, keepdim=True)
    c = torch.stack([torch.bincount(chosen.reshape(B, -1)[b], minlength=E) for b in range(B)]).double()
    P = s.reshape(B, S, E).sum(1)
    A = E / (k * S * S) * (c * P).sum(-1)
    return w * S * coef * A.sum(), A


def _route(logits, k, coef, S, sums=None, score_function="softmax", **opts):
    return route_topk(logits, k, opts.pop("renormalize", True), score_function=score_function, sequence_balance_coef=coef,
                      sequence_length=S, token_loss_weight=W_TOK, sequence_balance_sums=sums, **opts)


def _logged_A(sums):
    return sums[0].item() / sums[1].item()


# ---- definition ----

@pytest.mark.parametrize("score_function", ["softmax", "sigmoid"])
def test_uniform_logits_give_one(score_function):
    E, k, S, B = 8, 2, 6, 3
    sums = torch.zeros(2)
    logits = torch.zeros(B * S, E, requires_grad=True)
    _, p = _route(logits, k, 1.0, S, sums, score_function)
    p.sum().backward()
    # every score is 1/E, so A_b = E / (k S^2) * (S / E) * sum_e c[b, e] = 1 whatever the selection
    assert _logged_A(sums) == pytest.approx(1.0, rel=1e-6)
    assert sums[1].item() == pytest.approx(W_TOK * B * S)


@pytest.mark.parametrize("score_function", ["softmax", "sigmoid"])
def test_balanced_selections_give_exactly_one(score_function):
    E, k, S, B = 8, 2, 4, 2
    # within each sequence, token t selects experts (2t, 2t + 1): every expert once per sequence, scores uniform over
    # the picked pair (softmax) or flat (sigmoid: 0 vs -30 is sigma 0.5 vs ~0, normalised to 1/2 per picked expert)
    logits = torch.full((B * S, E), -30.0)
    for t in range(B * S):
        logits[t, (2 * t) % E] = logits[t, (2 * t + 1) % E] = 0.0
    logits = logits.requires_grad_()
    sums = torch.zeros(2)
    idx, p = _route(logits, k, 1.0, S, sums, score_function)
    p.sum().backward()
    _, A = _seq_objective_fp64(logits.detach(), idx, k, S, 1.0, W_TOK, score_function)
    assert torch.allclose(A, torch.ones_like(A), rtol=0, atol=1e-12)
    assert _logged_A(sums) == pytest.approx(1.0, rel=1e-6)


def test_split_experts_batch_is_balanced_but_every_sequence_collapsed():
    E, k, S, B = 4, 2, 8, 4
    logits = torch.full((B, S, E), -20.0)
    logits[0::2, :, :2] = 10.0  # even sequences route everything to experts {0, 1}
    logits[1::2, :, 2:] = 10.0  # odd ones to {2, 3}
    logits = logits.reshape(B * S, E).requires_grad_()
    seq_sums, batch_sums = torch.zeros(2), torch.zeros(3)
    _, p = route_topk(logits, k, True, load_balancing_coef=1.0, token_loss_weight=W_TOK, aux_loss_sums=batch_sums,
                      sequence_balance_coef=1.0, sequence_length=S, sequence_balance_sums=seq_sums)
    p.sum().backward()
    assert batch_sums[0].item() / batch_sums[2].item() == pytest.approx(1.0, rel=1e-5)
    assert E / k * 0.999 < _logged_A(seq_sums) <= E / k * (1 + 1e-6)


def test_one_sequence_is_the_batch_load_balancing_loss():
    torch.manual_seed(0)
    T, E, k, c = 24, 16, 4, 0.3
    logits = torch.randn(T, E) * 2
    dprobs = torch.randn(T, k)
    grads = []
    for kwargs in ({"load_balancing_coef": c}, {"sequence_balance_coef": c, "sequence_length": T}):
        x = logits.clone().requires_grad_()
        _, p = route_topk(x, k, True, token_loss_weight=W_TOK, **kwargs)
        (p * dprobs).sum().backward()
        grads.append(x.grad)
    torch.testing.assert_close(grads[1], grads[0], rtol=1e-6, atol=1e-9)


# ---- gradient against autograd on the fp64 definition ----

OPTIONS = [
    {},
    {"renormalize": False},
    {"expert_bias": "bias"},
    {"num_groups": 4, "topk_groups": 2},
    {"num_groups": 4, "topk_groups": 2, "expert_bias": "bias", "scaling_factor": 2.5},
    {"renormalize": False, "scaling_factor": 0.5},
]


@pytest.mark.parametrize("score_function", ["softmax", "sigmoid"])
@pytest.mark.parametrize("opts", OPTIONS, ids=lambda o: "-".join(f"{k}" for k in o) or "plain")
def test_attached_gradient_matches_autograd_on_the_fp64_definition(score_function, opts):
    torch.manual_seed(1)
    S, B, E, k, coef = 9, 4, 16, 3, 0.7
    opts = dict(opts)
    if opts.get("expert_bias") == "bias":
        opts["expert_bias"] = torch.randn(E) * 0.05
    logits = (torch.randn(B * S, E) * 2).requires_grad_()
    dprobs = torch.randn(B * S, k)
    sums = torch.zeros(2)
    idx, p = _route(logits, k, coef, S, sums, score_function, **dict(opts))
    (p * dprobs).sum().backward()

    base = logits.detach().clone().requires_grad_()
    idx0, p0 = route_topk(base, k, opts.pop("renormalize", True), score_function=score_function, **opts)
    assert torch.equal(idx0, idx)
    (p0 * dprobs).sum().backward()
    x64 = logits.detach().double().requires_grad_()
    obj, A = _seq_objective_fp64(x64, idx, k, S, coef, W_TOK, score_function)
    (seq_grad,) = torch.autograd.grad(obj, x64)
    torch.testing.assert_close(logits.grad.double(), base.grad.double() + seq_grad, rtol=1e-5, atol=1e-9)
    assert seq_grad.abs().max() > 1e-6  # the balance term is not negligible here
    assert sums[0].item() == pytest.approx(W_TOK * S * A.sum().item(), rel=1e-5)


def test_softmax_combined_with_the_batch_loss_and_z_loss():
    torch.manual_seed(2)
    S, B, E, k = 7, 3, 16, 4
    seq, lb, z = 0.4, 0.6, 0.2
    logits = (torch.randn(B * S, E) * 2).requires_grad_()
    dprobs = torch.randn(B * S, k)
    idx, p = route_topk(logits, k, True, num_groups=4, topk_groups=2, load_balancing_coef=lb, z_loss_coef=z,
                        token_loss_weight=W_TOK, sequence_balance_coef=seq, sequence_length=S)
    (p * dprobs).sum().backward()
    base = logits.detach().clone().requires_grad_()
    _, p0 = route_topk(base, k, True, num_groups=4, topk_groups=2)
    (p0 * dprobs).sum().backward()
    x64 = logits.detach().double().requires_grad_()
    obj, _ = _seq_objective_fp64(x64, idx, k, S, seq, W_TOK, "softmax")
    T = B * S
    s = torch.softmax(x64, -1)
    c = torch.bincount(idx.reshape(-1), minlength=E).double()
    A = E * ((c / (k * T)) * s.mean(0)).sum()
    Z = (torch.logsumexp(x64, -1) ** 2).mean()
    (grad,) = torch.autograd.grad(obj + W_TOK * T * (lb * A + z * Z), x64)
    torch.testing.assert_close(logits.grad.double(), base.grad.double() + grad, rtol=1e-5, atol=1e-9)


def test_coefficient_zero_is_the_plain_call():
    torch.manual_seed(3)
    logits = torch.randn(12, 8)
    a, b = logits.clone().requires_grad_(), logits.clone().requires_grad_()
    sums = torch.zeros(2)
    ia, pa = route_topk(a, 2, True, score_function="sigmoid")
    ib, pb = route_topk(b, 2, True, score_function="sigmoid", sequence_balance_coef=0.0, sequence_length=5,
                        token_loss_weight=W_TOK, sequence_balance_sums=sums)
    assert torch.equal(ia, ib) and torch.equal(pa, pb)
    pa.sum().backward()
    pb.sum().backward()
    assert torch.equal(a.grad, b.grad) and not sums.any()


# ---- refusals ----

def test_bad_inputs_are_refused():
    x = torch.randn(12, 8)
    with pytest.raises(ValueError, match="divisor"):
        route_topk(x, 2, True, sequence_balance_coef=0.1, sequence_length=5, token_loss_weight=W_TOK)
    with pytest.raises(ValueError, match="sequence_length"):
        route_topk(x, 2, True, sequence_balance_coef=0.1, token_loss_weight=W_TOK)
    with pytest.raises(ValueError, match="token_loss_weight"):
        route_topk(x, 2, True, sequence_balance_coef=0.1, sequence_length=4)
    with pytest.raises(ValueError, match="non-negative"):
        route_topk(x, 2, True, sequence_balance_coef=-0.1, sequence_length=4, token_loss_weight=W_TOK)
    for bad in (torch.zeros(3), torch.zeros(2, dtype=torch.float64), torch.zeros(1, 2)):
        with pytest.raises(ValueError, match="sequence_balance_sums"):
            route_topk(x, 2, True, sequence_balance_coef=0.1, sequence_length=4, token_loss_weight=W_TOK,
                       sequence_balance_sums=bad)
    # the batch terms stay softmax-only, with or without the sequence-wise loss
    with pytest.raises(ValueError, match="softmax"):
        route_topk(x, 2, True, score_function="sigmoid", load_balancing_coef=0.1, sequence_balance_coef=0.1,
                   sequence_length=4, token_loss_weight=W_TOK)


def test_moe_layer_needs_batched_sequences():
    from d9d_b200.module.block.moe import MoELayer, RouterParameters

    layer = MoELayer(hidden_dim=16, intermediate_dim_grouped=8, num_grouped_experts=8, top_k=2, router_renormalize_probabilities=True,
                     router=RouterParameters(score_function="sigmoid", enable_expert_bias=True))
    layer.reset_parameters()
    layer.router.set_sequence_balance_loss(0.1, W_TOK)
    layer.router.reset_aux_loss_sums()
    with pytest.raises(ValueError, match=r"\[batch, sequence, hidden\]"):
        layer(torch.randn(12, 16))
    layer(torch.randn(3, 4, 16)).sum().backward()
    assert layer.router.sequence_balance_sums[1].item() == pytest.approx(W_TOK * 12)


class _Modules:
    def __init__(self, modules):
        self.modules = modules


@pytest.mark.parametrize("mesh", [{"context_parallel_shard": 2}, {"context_parallel_replicate": 2}, {"tensor_parallel": 2}])
def test_trainer_refuses_meshes_that_split_sequences(mesh):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.component import MoEAuxLoss
    from d9d_b200.loop.config import MoEAuxLossConfig

    class _Ctx:  # the mesh alone: building it would need the ranks
        mesh_params = DeviceMeshParameters(**mesh)
        current_device = torch.device("cpu")

    with pytest.raises(ValueError, match="whole sequences"):
        MoEAuxLoss(_Ctx(), _Modules([]), MoEAuxLossConfig(sequence_balance_coef=1e-4))
    MoEAuxLoss(_Ctx(), _Modules([]), MoEAuxLossConfig(load_balancing_coef=1e-2))  # the batch terms need no whole sequences


def test_trainer_accepts_sigmoid_routers_for_the_sequence_loss_only():
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.component import MoEAuxLoss
    from d9d_b200.loop.config import MoEAuxLossConfig
    from d9d_b200.module.block.moe import MoELayer, RouterParameters

    layer = MoELayer(hidden_dim=16, intermediate_dim_grouped=8, num_grouped_experts=8, top_k=2, router_renormalize_probabilities=True,
                     router=RouterParameters(score_function="sigmoid", enable_expert_bias=True))
    ctx = DeviceMeshParameters().build()
    MoEAuxLoss(ctx, _Modules([torch.nn.ModuleList([layer])]), MoEAuxLossConfig(sequence_balance_coef=1e-4))
    assert layer.router.sequence_balance_coef == 1e-4
    with pytest.raises(ValueError, match="softmax router"):
        MoEAuxLoss(ctx, _Modules([torch.nn.ModuleList([layer])]),
                   MoEAuxLossConfig(sequence_balance_coef=1e-4, z_loss_coef=1e-3))


# ---- accounting ----

def test_microbatches_are_weighted_by_their_tokens():
    torch.manual_seed(4)
    E, k, coef = 8, 2, 0.5
    parts = [(torch.randn(2 * 5, E) * 2, 5), (torch.randn(3 * 7, E) * 2, 7)]
    sums = torch.zeros(2)
    want_value, want_weight = 0.0, 0.0
    for logits, S in parts:
        x = logits.clone().requires_grad_()
        idx, p = _route(x, k, coef, S, sums, "sigmoid")
        (p.sum() * 0).backward()
        x64 = logits.double().requires_grad_()
        obj, A = _seq_objective_fp64(x64, idx, k, S, coef, W_TOK, "sigmoid")
        torch.testing.assert_close(x.grad.double(), torch.autograd.grad(obj, x64)[0], rtol=1e-5, atol=1e-10)
        want_value += W_TOK * S * A.sum().item()
        want_weight += W_TOK * logits.shape[0]
    assert sums[1].item() == pytest.approx(want_weight)
    assert sums[0].item() == pytest.approx(want_value, rel=1e-5)


def _deepseek_model(recompute):
    from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode
    from d9d_b200.module.block.moe import MoELayer
    from d9d_b200.module.model.deepseek_v3 import DeepseekV3ForCausalLM
    from d9d_b200.pipelining.api import PipelineStageInfo
    from tests.test_expert_bias_balancing import _deepseek_params

    torch.manual_seed(5)
    model = DeepseekV3ForCausalLM(_deepseek_params(), PipelineStageInfo(0, 1), HiddenStatesAggregationMode.no, recompute)
    model.reset_parameters()
    layers = [m for m in model.modules() if isinstance(m, MoELayer)]
    for layer in layers:
        layer.router.set_sequence_balance_loss(0.3, W_TOK)
        layer.router.reset_aux_loss_sums()
    return model, layers


def test_activation_recomputation_counts_once():
    ids = torch.randint(0, 128, (3, 16), generator=torch.Generator().manual_seed(6))
    pos = torch.arange(16)[None].expand(3, -1)
    results = []
    for recompute in (False, True):
        model, layers = _deepseek_model(recompute)
        model.train()
        out = model(input_ids=ids, position_ids=pos, labels=ids)
        out["logps"].mean().backward()
        results.append(({n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None},
                        [layer.router.sequence_balance_sums.clone() for layer in layers]))
    (g0, s0), (g1, s1) = results
    assert g0.keys() == g1.keys() and s0
    for name in g0:
        torch.testing.assert_close(g1[name], g0[name], rtol=1e-5, atol=1e-7, msg=name)
    for a, b in zip(s0, s1):
        assert torch.equal(a, b)
        assert a[1].item() == pytest.approx(W_TOK * 48)


# ---- Trainer ----

def _deepseek_trainer(tmp, aux):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import AdamWOptimizerConfig
    from d9d_b200.loop.config import TrainerConfig
    from d9d_b200.loop.run import TrainingConfigurator
    from tests.helpers_train import SFTTask, SyntheticDataProvider, trainer_config
    from tests.test_expert_bias_balancing import _deepseek_params, _DeepseekProvider

    cfg = trainer_config(tmp, log_dir=tmp / "logs").model_dump()
    cfg["gradient_manager"]["grad_dtype"] = None  # bf16 model, as the recipes cast it: bf16 gradients
    if aux is not None:
        cfg["moe_aux_loss"] = aux
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=DeviceMeshParameters(), parameters=TrainerConfig.model_validate(cfg), task_provider=lambda ctx: SFTTask(ctx.dist_context),
        model_provider=_DeepseekProvider(_deepseek_params(), dtype=torch.bfloat16), data_provider=SyntheticDataProvider(num_samples=32),
        optimizer_provider=AutoOptimizerProvider(AdamWOptimizerConfig(lr=3e-3, weight_decay=0.0)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched),
    ).configure()


def _logged(tmp):
    (f,) = list((tmp / "logs").glob("*.jsonl"))
    out = {}
    for r in map(json.loads, f.read_text().splitlines()):
        if "name" in r and "value" in r:
            out.setdefault(r["name"], {})[r["step"]] = r["value"]
    return out


def _trained(trainer):
    trainer.train()
    return {k: v.clone() for k, v in trainer.state.tracked_modules.modules[0].state_dict().items()}


def test_trainer_trains_a_sigmoid_router_with_the_sequence_loss(tmp_path):
    on = _deepseek_trainer(tmp_path / "on", {"sequence_balance_coef": 0.05})
    trained = _trained(on)
    logs = _logged(tmp_path / "on")
    seq = logs["moe_sequence_balance_loss"]
    assert sorted(seq) == sorted(logs["l2_grad_norm_total"])  # only on logging steps
    assert "moe_load_balancing_loss" not in logs
    assert all(1.0 <= v <= 8 / 2 for v in seq.values()), seq  # 1 <= A_b <= E / k
    ref = _trained(_deepseek_trainer(tmp_path / "ref", None))
    assert any(not torch.equal(trained[n], ref[n]) for n in ref if n.endswith("router.gate.weight"))


def test_trainer_coefficient_zero_is_bitwise_the_plain_run(tmp_path):
    ref = _trained(_deepseek_trainer(tmp_path / "off", None))
    got = _trained(_deepseek_trainer(tmp_path / "zero", {"sequence_balance_coef": 0.0}))
    for name, value in ref.items():
        assert torch.equal(got[name], value), name
    assert _logged(tmp_path / "zero")["loss"] == _logged(tmp_path / "off")["loss"]
    assert "moe_sequence_balance_loss" not in _logged(tmp_path / "zero")


# ---- a pipeline-parallel run against one process (gloo) ----

SEQ_ON = {"sequence_balance_coef": 0.5}  # large enough to move the routers visibly in a few steps


def _pp_trainer(tmp, mesh_kwargs=None, schedule=None, source=None):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import SGDOptimizerConfig
    from d9d_b200.loop.config import TrainerConfig
    from d9d_b200.loop.run import TrainingConfigurator
    from tests.helpers_train import LMProvider, SFTTask, SyntheticDataProvider, moe_params, trainer_config

    cfg = trainer_config(tmp, total_batch=8, micro=2, schedule=schedule, log_dir=tmp / "logs", source=source).model_dump()
    cfg["moe_aux_loss"] = SEQ_ON
    cfg["logging"]["period_steps"] = 1
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=DeviceMeshParameters(**(mesh_kwargs or {})), parameters=TrainerConfig.model_validate(cfg),
        task_provider=lambda ctx: SFTTask(ctx.dist_context), model_provider=LMProvider(moe_params(), moe=True),
        data_provider=SyntheticDataProvider(num_samples=32), optimizer_provider=AutoOptimizerProvider(SGDOptimizerConfig(lr=0.5)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched),
    ).configure()


def _pp_worker(rank, world, tmp, mesh_kwargs, schedule, source):
    from pathlib import Path

    trainer = _pp_trainer(Path(tmp), mesh_kwargs, schedule, source=Path(source))
    trainer.train()
    trainer.export(Path(tmp) / "export", load_checkpoint=False)


@pytest.mark.dist
def test_pipeline_parallel_run_matches_one_process(tmp_path):
    from d9d_b200.model_state.io import load_model_state
    from d9d_b200.model_state.mapper.adapters import identity_mapper_from_module

    mesh_kwargs = {"pipeline_parallel": 2}
    schedule = {"schedule": "1f1b", "num_stages_per_rank": 1, "zero_bubble": False}
    _pp_trainer(tmp_path / "init").export(tmp_path / "init" / "export", load_checkpoint=False)  # one initial model for all
    source = tmp_path / "init" / "export"
    single = _pp_trainer(tmp_path / "one", source=source)
    single.train()
    ref_state = {k: v.clone() for k, v in single.state.tracked_modules.modules[0].state_dict().items()}
    run_distributed(_pp_worker, 2, str(tmp_path / "dist"), mesh_kwargs, schedule, str(source))
    model = _pp_trainer(tmp_path / "load").state.tracked_modules.modules[0]
    load_model_state(tmp_path / "dist" / "export", identity_mapper_from_module(model), "cpu", model, show_progress=False)

    ref, got = _logged(tmp_path / "one"), _logged(tmp_path / "dist")
    assert ref["moe_sequence_balance_loss"][0] > 1.0
    for name in ("loss", "moe_sequence_balance_loss"):
        assert sorted(got[name]) == sorted(ref[name]) == list(range(4)), name
        for step, value in ref[name].items():
            assert got[name][step] == pytest.approx(value, rel=1e-5, abs=1e-7), (name, step)
    for name, value in ref_state.items():
        torch.testing.assert_close(model.state_dict()[name], value, rtol=1e-4, atol=1e-6, msg=lambda m, n=name: f"{n}: {m}")

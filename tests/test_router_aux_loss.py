"""The softmax router's auxiliary losses on the PyTorch path (the numerics oracle of the fused kernels): the definitions on
hand-made inputs, the attached gradient against autograd on the explicit fp64 formula under every allowed routing option,
the token weighting across microbatches, activation recomputation, a router trained by the load-balancing term alone, the
refusal of sigmoid routers, and the Trainer option: bitwise unchanged when off, logged values when on, data-parallel and
pipeline-parallel (1F1B and zero-bubble) gloo runs equal to one process accumulating the same microbatches, and an
exact resume."""

import math

import pytest
import torch

from d9d_b200.kernel.router import route_topk
from tests.dist_utils import run_distributed

W_TOK = 1e-3


def _aux_objective_fp64(logits, chosen, k, lb, z, w):
    """``w T (lb A + z Z)`` from the written definitions, in fp64 (``chosen`` carries no gradient)."""
    x = logits.double().reshape(-1, logits.shape[-1])
    T, E = x.shape
    s = torch.softmax(x, dim=-1)
    c = torch.bincount(chosen.reshape(-1), minlength=E).double()
    A = E * ((c / (k * T)) * s.mean(0)).sum()
    Z = (torch.logsumexp(x, dim=-1) ** 2).mean()
    return w * T * (lb * A + z * Z), A, Z


def _route(logits, k, lb, z, sums=None, **opts):
    return route_topk(logits, k, opts.pop("renormalize", True), load_balancing_coef=lb, z_loss_coef=z, token_loss_weight=W_TOK,
                      aux_loss_sums=sums, **opts)


def test_uniform_logits_give_one():
    E, k, T = 8, 2, 16
    sums = torch.zeros(3)
    logits = torch.zeros(T, E, requires_grad=True)
    _, p = _route(logits, k, 1.0, 0.0, sums)
    p.sum().backward()
    # P_e = 1/E for every expert, so A = E * sum_e f_e / E = 1 whatever the selection
    assert sums[0].item() / sums[2].item() == pytest.approx(1.0, rel=1e-6)
    assert sums[2].item() == pytest.approx(W_TOK * T)


def test_balanced_selection_gives_exactly_one():
    E, k = 8, 2
    # token t selects experts (2t mod 8, 2t+1 mod 8): every expert is selected equally often; scores uniform
    T = 8
    logits = torch.full((T, E), -30.0)
    for t in range(T):
        logits[t, (2 * t) % E] = logits[t, (2 * t + 1) % E] = 0.0
    logits = logits.requires_grad_()
    sums = torch.zeros(3)
    idx, p = _route(logits, k, 1.0, 0.0, sums)
    assert torch.bincount(idx.reshape(-1), minlength=E).tolist() == [2] * E
    p.sum().backward()
    _, A, _ = _aux_objective_fp64(logits.detach(), idx, k, 1.0, 0.0, W_TOK)
    assert float(A) == pytest.approx(1.0, abs=1e-12)
    assert sums[0].item() / sums[2].item() == pytest.approx(1.0, rel=1e-6)


def test_collapse_onto_k_experts_approaches_e_over_k():
    E, k, T = 16, 4, 32
    logits = torch.full((T, E), -20.0)
    logits[:, :k] = 10.0
    logits = logits.requires_grad_()
    sums = torch.zeros(3)
    _, p = _route(logits, k, 1.0, 0.0, sums)
    p.sum().backward()
    A = sums[0].item() / sums[2].item()
    assert E / k * 0.999 < A <= E / k


def test_z_loss_is_the_mean_squared_logsumexp():
    torch.manual_seed(0)
    logits = (torch.randn(13, 24) * 3).requires_grad_()
    sums = torch.zeros(3)
    idx, p = _route(logits, 3, 0.0, 1.0, sums)
    p.sum().backward()
    _, A, Z = _aux_objective_fp64(logits.detach(), idx, 3, 0.0, 1.0, W_TOK)
    assert Z.item() == pytest.approx((torch.logsumexp(logits.detach().double(), -1) ** 2).mean().item(), rel=1e-12)
    assert sums[1].item() / sums[2].item() == pytest.approx(Z.item(), rel=1e-5)
    assert sums[0].item() / sums[2].item() == pytest.approx(A.item(), rel=1e-5)  # A is logged whatever the coefficients


OPTIONS = [
    {},
    {"renormalize": False},
    {"expert_bias": "bias"},
    {"num_groups": 4, "topk_groups": 2},
    {"num_groups": 4, "topk_groups": 2, "expert_bias": "bias", "scaling_factor": 2.5},
    {"renormalize": False, "scaling_factor": 0.5},
]


@pytest.mark.parametrize("opts", OPTIONS, ids=lambda o: "-".join(f"{k}" for k in o) or "plain")
@pytest.mark.parametrize("lb,z", [(0.7, 0.0), (0.0, 0.3), (0.7, 0.3)])
def test_attached_gradient_matches_autograd_on_the_fp64_formula(opts, lb, z):
    torch.manual_seed(1)
    T, E, k = 37, 16, 3
    opts = dict(opts)
    if opts.get("expert_bias") == "bias":
        opts["expert_bias"] = torch.randn(E) * 0.05
    logits = (torch.randn(T, E) * 2).requires_grad_()
    dprobs = torch.randn(T, k)
    idx, p = _route(logits, k, lb, z, **opts)
    (p * dprobs).sum().backward()
    got = logits.grad.clone()

    base = logits.detach().clone().requires_grad_()
    idx0, p0 = _route(base, k, 0.0, 0.0, **opts)
    assert torch.equal(idx0, idx)
    (p0 * dprobs).sum().backward()
    x64 = logits.detach().double().requires_grad_()
    obj, _, _ = _aux_objective_fp64(x64, idx, k, lb, z, W_TOK)
    (aux_grad,) = torch.autograd.grad(obj, x64)
    torch.testing.assert_close(got.double(), base.grad.double() + aux_grad, rtol=1e-5, atol=1e-8)
    assert aux_grad.abs().max() > 1e-6  # the auxiliary term is not negligible here


def test_microbatches_are_weighted_by_their_tokens():
    torch.manual_seed(2)
    E, k, lb, z = 8, 2, 0.5, 0.2
    parts = [torch.randn(5, E) * 2, torch.randn(19, E) * 2]
    x = [p.clone().requires_grad_() for p in parts]
    sums = torch.zeros(3)
    for xi in x:
        _, p = _route(xi, k, lb, z, sums)
        (p.sum() * 0).backward()
    grads, values, weights = [], [], []
    for xi in parts:
        x64 = xi.double().requires_grad_()
        idx, _ = route_topk(xi, k, True)
        obj, A, Z = _aux_objective_fp64(x64, idx, k, lb, z, W_TOK)
        grads.append(torch.autograd.grad(obj, x64)[0])
        values.append((A.item(), Z.item()))
        weights.append(W_TOK * xi.shape[0])
    for xi, g in zip(x, grads):
        torch.testing.assert_close(xi.grad.double(), g, rtol=1e-5, atol=1e-9)
    assert sums[2].item() == pytest.approx(sum(weights))
    assert sums[0].item() == pytest.approx(sum(w * a for w, (a, _) in zip(weights, values)), rel=1e-5)
    assert sums[1].item() == pytest.approx(sum(w * zz for w, (_, zz) in zip(weights, values)), rel=1e-5)


def test_coefficients_zero_are_the_plain_call():
    torch.manual_seed(3)
    logits = torch.randn(11, 8)
    a, b = logits.clone().requires_grad_(), logits.clone().requires_grad_()
    sums = torch.zeros(3)
    ia, pa = route_topk(a, 2, True)
    ib, pb = route_topk(b, 2, True, load_balancing_coef=0.0, z_loss_coef=0.0, token_loss_weight=W_TOK, aux_loss_sums=sums)
    assert torch.equal(ia, ib) and torch.equal(pa, pb)
    pa.sum().backward()
    pb.sum().backward()
    assert torch.equal(a.grad, b.grad) and not sums.any()


def test_sigmoid_router_with_a_coefficient_is_refused():
    from d9d_b200.module.block.moe import MoELayer, RouterParameters

    with pytest.raises(ValueError, match="softmax"):
        route_topk(torch.randn(4, 8), 2, True, score_function="sigmoid", load_balancing_coef=0.1, token_loss_weight=W_TOK)
    layer = MoELayer(hidden_dim=16, intermediate_dim_grouped=8, num_grouped_experts=8, top_k=2, router_renormalize_probabilities=True,
                     router=RouterParameters(score_function="sigmoid", enable_expert_bias=True))
    with pytest.raises(ValueError, match="softmax router"):
        layer.router.set_aux_loss(0.0, 1e-3, W_TOK)
    layer.router.set_aux_loss(0.0, 0.0, W_TOK)  # off is allowed


def test_load_balancing_term_alone_balances_a_collapsed_router():
    from d9d_b200.module.block.moe.router import TopKRouter

    torch.manual_seed(4)
    E, k, D, T = 8, 2, 16, 256
    router = TopKRouter(dim=D, num_experts=E, top_k=k, renormalize_probabilities=True)
    router.reset_parameters()
    with torch.no_grad():
        router.gate.weight.mul_(0.1)
        router.gate.weight[:k, 0] = 1.0  # a constant input feature sends most tokens to experts 0 and 1
    router.set_aux_loss(1.0, 0.0, 1.0 / T)  # unit weight per call
    x = torch.randn(T, D)
    x[:, 0] = 2.0
    opt = torch.optim.SGD(router.parameters(), lr=2.0)
    history = []
    for _ in range(200):
        router.reset_aux_loss_sums()
        routing = router(x)
        opt.zero_grad()
        (routing.selected_probabilities.sum() * 0).backward()  # the auxiliary gradient alone
        opt.step()
        history.append(router.aux_loss_sums[0].item() / router.aux_loss_sums[2].item())
    assert history[0] > 2.0, history[0]
    assert history[-1] < 1.2, history[-10:]


def _qwen_moe(recompute: bool):
    from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode
    from d9d_b200.module.block.moe import MoELayer
    from d9d_b200.module.model.qwen3_moe import Qwen3MoEForCausalLM
    from d9d_b200.pipelining.api import PipelineStageInfo
    from tests.helpers_train import moe_params

    torch.manual_seed(5)
    model = Qwen3MoEForCausalLM(moe_params(), PipelineStageInfo(0, 1), HiddenStatesAggregationMode.no, recompute)
    model.reset_parameters()
    layers = [m for m in model.modules() if isinstance(m, MoELayer)]
    for layer in layers:
        layer.router.set_aux_loss(0.3, 0.1, W_TOK)
        layer.router.reset_aux_loss_sums()
    return model, layers


def test_activation_recomputation_counts_once():
    ids = torch.randint(0, 128, (2, 16), generator=torch.Generator().manual_seed(6))
    pos = torch.arange(16)[None].expand(2, -1)
    results = []
    for recompute in (False, True):
        model, layers = _qwen_moe(recompute)
        model.train()
        out = model(input_ids=ids, position_ids=pos, labels=ids)
        out["logps"].mean().backward()
        results.append(({n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None},
                        [layer.router.aux_loss_sums.clone() for layer in layers]))
    (g0, s0), (g1, s1) = results
    assert g0.keys() == g1.keys()
    for name in g0:
        torch.testing.assert_close(g1[name], g0[name], rtol=1e-5, atol=1e-7, msg=name)
    for a, b in zip(s0, s1):
        assert torch.equal(a, b)
        assert a[2].item() == pytest.approx(W_TOK * 32)


def _moe_trainer(tmp, aux):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import AdamWOptimizerConfig
    from d9d_b200.loop.config import TrainerConfig
    from d9d_b200.loop.run import TrainingConfigurator
    from tests.helpers_train import LMProvider, SFTTask, SyntheticDataProvider, moe_params, trainer_config

    cfg = trainer_config(tmp, log_dir=tmp / "logs").model_dump()
    if aux is not None:
        cfg["moe_aux_loss"] = aux
    cfg = TrainerConfig.model_validate(cfg)
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=DeviceMeshParameters(), parameters=cfg, task_provider=lambda ctx: SFTTask(ctx.dist_context),
        model_provider=LMProvider(moe_params(), moe=True), data_provider=SyntheticDataProvider(num_samples=32),
        optimizer_provider=AutoOptimizerProvider(AdamWOptimizerConfig(lr=3e-3, weight_decay=0.0)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched),
    ).configure()


def _logged(tmp):
    import json

    (f,) = list((tmp / "logs").glob("*.jsonl"))
    out = {}
    for r in map(json.loads, f.read_text().splitlines()):
        if "name" in r and "value" in r:
            out.setdefault(r["name"], {})[r["step"]] = r["value"]
    return out


def _trained(trainer):
    trainer.train()
    return {k: v.clone() for k, v in trainer.state.tracked_modules.modules[0].state_dict().items()}


def test_trainer_off_and_zero_coefficients_are_bitwise_the_plain_run(tmp_path):
    off = _moe_trainer(tmp_path / "off", None)
    assert off.state.moe_aux_loss is None
    ref = _trained(off)
    zero = _moe_trainer(tmp_path / "zero", {"load_balancing_coef": 0.0, "z_loss_coef": 0.0})
    got = _trained(zero)
    for name, value in ref.items():
        assert torch.equal(got[name], value), name
    assert _logged(tmp_path / "zero")["loss"] == _logged(tmp_path / "off")["loss"]
    assert set(zero.state.state_dict()) == set(off.state.state_dict())  # no checkpoint state


def test_trainer_logs_the_token_weighted_losses(tmp_path):
    on = _moe_trainer(tmp_path / "on", {"load_balancing_coef": 0.05, "z_loss_coef": 1e-3})
    trained = _trained(on)
    logs = _logged(tmp_path / "on")
    lb, z = logs["moe_load_balancing_loss"], logs["moe_router_z_loss"]
    assert sorted(lb) == sorted(z) == sorted(logs["l2_grad_norm_total"])  # only on logging steps
    assert all(1.0 <= v <= 2.0 for v in lb.values()), lb  # E / k = 2 bounds A
    assert all(v > 0 and math.isfinite(v) for v in z.values()), z
    ref = _trained(_moe_trainer(tmp_path / "ref", None))
    assert any(not torch.equal(trained[n], ref[n]) for n in ref if "router" in n)


def test_trainer_refuses_sigmoid_routers():
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.component import MoEAuxLoss
    from d9d_b200.loop.config import MoEAuxLossConfig
    from d9d_b200.module.block.moe import MoELayer, RouterParameters

    class _Modules:
        def __init__(self, modules):
            self.modules = modules

    layer = MoELayer(hidden_dim=16, intermediate_dim_grouped=8, num_grouped_experts=8, top_k=2, router_renormalize_probabilities=True,
                     router=RouterParameters(score_function="sigmoid", enable_expert_bias=True))
    with pytest.raises(ValueError, match="softmax router"):
        MoEAuxLoss(DeviceMeshParameters().build(), _Modules([torch.nn.ModuleList([layer])]), MoEAuxLossConfig(load_balancing_coef=1e-2))


# ---- distributed runs against one process that accumulates the same microbatches (gloo) ----

AUX_ON = {"load_balancing_coef": 0.5, "z_loss_coef": 0.05}  # large enough to move the router visibly in a few steps
SAMPLES, GLOBAL_BATCH, MICRO = 32, 8, 2


class _OrderedSamples:
    """The synthetic dataset read in a given order (``order[i]`` is the sample served at position ``i``)."""

    def __init__(self, data, order):
        self._data, self._order = data, order

    def __len__(self):
        return len(self._order)

    def __getitem__(self, i):
        return self._data[self._order[i]]


class _OrderedProvider:
    def __init__(self, order=None):
        self._order = order

    def __call__(self, context):
        from d9d_b200.dataset import SyntheticTokenDataset, shard_dataset_data_parallel
        from d9d_b200.loop.control import InitializeDatasetResult
        from tests.helpers_train import VOCAB

        data = SyntheticTokenDataset(SAMPLES, 16, sum(VOCAB.values()), seed=3, learnable=True)
        if self._order is not None:
            data = _OrderedSamples(data, self._order)
        return InitializeDatasetResult(dataset=shard_dataset_data_parallel(data, context.dist_context), collator=SyntheticTokenDataset.collate)


def _data_parallel_order(world):
    """The sample order under which one process accumulates, step by step, rank 0's microbatches, then rank 1's, ...:
    the same token split as ``world`` data-parallel ranks."""
    from d9d_b200.dataset.sharded import ShardedDataset, ShardIndexingMode

    shards = [ShardedDataset(list(range(SAMPLES)), total_shards=world, current_shard=r, indexing_mode=ShardIndexingMode.sequential,
                             pad_to_equal_size_across_shards=True) for r in range(world)]
    per_rank = GLOBAL_BATCH // world
    order = []
    for step in range(SAMPLES // GLOBAL_BATCH):
        for shard in shards:
            order += [shard[i] for i in range(step * per_rank, (step + 1) * per_rank)]
    return order


def _aux_trainer(tmp, mesh_kwargs=None, schedule=None, order=None, ckpt_period="disable", source=None):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import SGDOptimizerConfig
    from d9d_b200.loop.config import TrainerConfig
    from d9d_b200.loop.run import TrainingConfigurator
    from tests.helpers_train import LMProvider, SFTTask, moe_params, trainer_config

    cfg = trainer_config(tmp, total_batch=GLOBAL_BATCH, micro=MICRO, schedule=schedule, ckpt_period=ckpt_period,
                         log_dir=tmp / "logs", source=source).model_dump()
    cfg["moe_aux_loss"] = AUX_ON
    cfg["logging"]["period_steps"] = 1
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=DeviceMeshParameters(**(mesh_kwargs or {})), parameters=TrainerConfig.model_validate(cfg),
        task_provider=lambda ctx: SFTTask(ctx.dist_context), model_provider=LMProvider(moe_params(), moe=True),
        data_provider=_OrderedProvider(order), optimizer_provider=AutoOptimizerProvider(SGDOptimizerConfig(lr=0.5)),
        lr_scheduler_provider=AutoLRSchedulerProvider(sched),
    ).configure()


def _aux_dist_worker(rank, world, tmp, mesh_kwargs, schedule, source):
    from pathlib import Path

    trainer = _aux_trainer(Path(tmp), mesh_kwargs, schedule, source=Path(source))
    trainer.train()
    trainer.export(Path(tmp) / "export", load_checkpoint=False)


def _exported(tmp):
    from d9d_b200.model_state.io import load_model_state
    from d9d_b200.model_state.mapper.adapters import identity_mapper_from_module

    model = _aux_trainer(tmp / "load").state.tracked_modules.modules[0]
    load_model_state(tmp / "export", identity_mapper_from_module(model), "cpu", model, show_progress=False)
    return model.state_dict()


def _assert_same_run(ref_dir, ref_state, got_dir, got_state):
    ref, got = _logged(ref_dir), _logged(got_dir)
    for name in ("loss", "moe_load_balancing_loss", "moe_router_z_loss"):
        assert sorted(got[name]) == sorted(ref[name]) == list(range(SAMPLES // GLOBAL_BATCH)), name
        for step, value in ref[name].items():
            assert got[name][step] == pytest.approx(value, rel=1e-5, abs=1e-7), (name, step)
    for name, value in ref_state.items():
        torch.testing.assert_close(got_state[name], value, rtol=1e-4, atol=1e-6, msg=lambda m, n=name: f"{n}: {m}")


@pytest.mark.dist
@pytest.mark.parametrize("mesh_kwargs,schedule,world", [
    ({"data_parallel_replicate": 2}, None, 2),
    ({"pipeline_parallel": 2}, {"schedule": "1f1b", "num_stages_per_rank": 1, "zero_bubble": False}, 2),
    ({"pipeline_parallel": 2}, {"schedule": "1f1b", "num_stages_per_rank": 1, "zero_bubble": True}, 2),
], ids=["dp2", "pp2-1f1b", "pp2-zero-bubble"])
def test_distributed_run_matches_one_process(tmp_path, mesh_kwargs, schedule, world):
    dp = mesh_kwargs.get("data_parallel_replicate", 1)
    _aux_trainer(tmp_path / "init").export(tmp_path / "init" / "export", load_checkpoint=False)  # one initial model for all
    source = tmp_path / "init" / "export"
    single = _aux_trainer(tmp_path / "one", order=_data_parallel_order(dp) if dp > 1 else None, source=source)
    single.train()
    ref_state = {k: v.clone() for k, v in single.state.tracked_modules.modules[0].state_dict().items()}
    assert _logged(tmp_path / "one")["moe_load_balancing_loss"][0] > 1.0
    run_distributed(_aux_dist_worker, world, str(tmp_path / "dist"), mesh_kwargs, schedule, str(source))
    _assert_same_run(tmp_path / "one", ref_state, tmp_path / "dist", _exported(tmp_path / "dist"))


def test_resumed_run_continues_the_same_trajectory(tmp_path):
    from d9d_b200.loop.event.catalogue.train import EVENT_TRAIN_STEP_PRE

    full = _aux_trainer(tmp_path / "full")
    full.train()
    ref_state = {k: v.clone() for k, v in full.state.tracked_modules.modules[0].state_dict().items()}

    class _Stop(Exception):
        pass

    def stop_at_2(ctx):
        if ctx.stepper.current_step == 2:
            raise _Stop

    part = _aux_trainer(tmp_path / "cut", ckpt_period=1)
    part.state.event_bus.subscribe(EVENT_TRAIN_STEP_PRE, stop_at_2)
    with pytest.raises(_Stop):
        part.train()
    resumed = _aux_trainer(tmp_path / "cut", ckpt_period=1)
    resumed.train()
    for name, value in resumed.state.tracked_modules.modules[0].state_dict().items():
        assert torch.equal(value, ref_state[name]), name
    ref, got = _logged(tmp_path / "full"), _logged(tmp_path / "cut")
    for name in ("loss", "moe_load_balancing_loss", "moe_router_z_loss"):
        assert got[name] == ref[name], name

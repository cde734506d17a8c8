"""Label smoothing and the z-loss in the fused linear cross-entropy, on the CPU: the reference against
``F.cross_entropy(label_smoothing) + zeta lse^2`` and its autograd, the chunked code path (through PyTorch stand-ins of
the native ops) against the reference over split blocks and small scratch budgets, refused coefficients, coefficients 0
bitwise the plain call, the logged sums, and the Trainer option: logged keys, per-step sums, a two-stage pipeline run
equal to one process, and ``lm_loss: null`` bitwise the plain run."""

import math

import pytest
import torch
import torch.nn.functional as F

from d9d_b200.kernel.cce import main as cce
from d9d_b200.kernel.cce.main import LinearCrossEntropy, linear_cross_entropy, linear_cross_entropy_reference
from tests.dist_utils import run_distributed

REGS = [(0.1, 0.0), (0.0, 0.1), (0.1, 1e-4), (1.0, 0.05)]  # (label_smoothing, z_loss_coef)


def _problem(T=96, K=32, sizes=(700, 24), seed=0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    e = (torch.randn(T, K, generator=g) * 0.5).to(dtype).requires_grad_()
    ws = [(torch.randn(s, K, generator=g) * 0.2).to(dtype).requires_grad_() for s in sizes]
    tgt = torch.randint(0, sum(sizes), (T,), generator=g)
    tgt[::5] = -100
    tgt[1] = sum(sizes) - 1  # a target inside the last (tiny) block
    return e, ws, tgt


@pytest.mark.parametrize("eps,zeta", REGS)
@pytest.mark.parametrize("softcap,with_bias", [(None, False), (5.0, True)])
def test_reference_is_the_definition_and_its_gradient(eps, zeta, softcap, with_bias):
    e, ws, tgt = _problem(dtype=torch.float64)
    w = torch.cat(ws).detach().requires_grad_()
    bias = (torch.randn(w.shape[0], dtype=torch.float64) * 0.3).requires_grad_() if with_bias else None
    loss, lse = linear_cross_entropy_reference(e, w, tgt, bias, -100, softcap, eps, zeta)
    # the written definition: (1 - eps) nll + eps (lse - mean_j z_j) + zeta lse^2, 0 at ignored targets
    z = e.double() @ w.double().t() + (bias if with_bias else 0)
    if softcap:
        z = softcap * torch.tanh(z / softcap)
    nll = torch.logsumexp(z, -1) - z.gather(1, tgt.clamp_min(0)[:, None])[:, 0]
    want = ((1 - eps) * nll + eps * (torch.logsumexp(z, -1) - z.mean(-1)) + zeta * torch.logsumexp(z, -1) ** 2)
    want = torch.where(tgt == -100, 0.0, want)
    torch.testing.assert_close(loss.double(), want, rtol=1e-5, atol=1e-5)  # the reference computes in fp32
    torch.testing.assert_close(lse.double(), torch.logsumexp(z, -1), rtol=1e-5, atol=1e-5)
    # the gradient w.r.t. the logits that the kernels write: (1 + 2 zeta lse) p - (1 - eps) onehot - eps / V
    zl = z.detach().requires_grad_()
    lsel = torch.logsumexp(zl, -1)
    (F.cross_entropy(zl, tgt, reduction="none", label_smoothing=eps) + zeta * lsel**2 * (tgt != -100)).sum().backward()
    p = torch.softmax(z.detach(), -1)
    onehot = F.one_hot(tgt.clamp_min(0), z.shape[1]).double()
    dz = ((1 + 2 * zeta * lsel.detach())[:, None] * p - (1 - eps) * onehot - eps / z.shape[1]) * (tgt != -100)[:, None]
    torch.testing.assert_close(zl.grad, dz, rtol=1e-9, atol=1e-12)
    # and the reference's autograd reproduces it
    loss.sum().backward()
    dzdx = (1 - (z.detach() / softcap) ** 2) if softcap else 1.0
    torch.testing.assert_close(e.grad.double(), (dz * dzdx) @ w.detach(), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("eps,zeta", REGS)
@pytest.mark.parametrize("sizes", [(700,), (700, 24), (300, 260, 8)])
@pytest.mark.parametrize("budget", [1 << 30, 96 * 256 * 2 + 96 * 32 * 4])
@pytest.mark.parametrize("softcap,with_bias", [(None, False), (5.0, True)])
def test_chunked_path_matches_the_reference(monkeypatch, eps, zeta, sizes, budget, softcap, with_bias):
    monkeypatch.setattr(cce, "_CHUNK_BYTES", budget)
    e, ws, tgt = _problem(sizes=sizes)
    bias = (torch.randn(sum(sizes)) * 0.3).requires_grad_() if with_bias else None
    sums = torch.zeros(3)
    loss, lse = linear_cross_entropy(e, ws, tgt, bias=bias, softcap=softcap, reduction="sum", return_lse=True,
                                     _emulate=True, label_smoothing=eps, z_loss_coef=zeta, loss_sums=sums)
    loss.backward()
    got = [e.grad.clone(), *[w.grad.clone() for w in ws]] + ([bias.grad.clone()] if with_bias else [])

    e2 = e.detach().clone().requires_grad_()
    ws2 = [w.detach().clone().requires_grad_() for w in ws]
    b2 = bias.detach().clone().requires_grad_() if with_bias else None
    ref, lse_ref = linear_cross_entropy_reference(e2, torch.cat(ws2), tgt, b2, -100, softcap, eps, zeta)
    ref.sum().backward()
    want = [e2.grad, *[w.grad for w in ws2]] + ([b2.grad] if with_bias else [])
    assert torch.allclose(loss, ref.sum(), rtol=1e-4, atol=1e-4)
    assert torch.allclose(lse, lse_ref, rtol=1e-4, atol=1e-4)
    for a, b in zip(got, want):
        assert (a - b).norm() / (b.norm() + 1e-9) < 1e-2  # the emulated dlogits buffer is bf16 like the real one
    nll, _ = linear_cross_entropy_reference(e2.detach(), torch.cat(ws2).detach(), tgt, b2, -100, softcap)
    valid = tgt != -100
    torch.testing.assert_close(sums, torch.stack([nll[valid].sum(), (lse_ref[valid] ** 2).sum(), valid.sum().float()]),
                               rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("reduction", ["none", "sum", "mean"])
@pytest.mark.parametrize("emulate", [False, True])
def test_reductions_keep_their_meaning(reduction, emulate):
    e, ws, tgt = _problem()
    per_token = linear_cross_entropy(e, ws, tgt, reduction="none", _emulate=emulate, label_smoothing=0.2, z_loss_coef=0.01)
    got = linear_cross_entropy(e, ws, tgt, reduction=reduction, _emulate=emulate, label_smoothing=0.2, z_loss_coef=0.01)
    want = {"none": per_token, "sum": per_token.sum(), "mean": per_token.sum() / (tgt != -100).sum()}[reduction]
    torch.testing.assert_close(got, want)
    assert (per_token[tgt == -100] == 0).all()


@pytest.mark.parametrize("kw", [{"label_smoothing": -0.1}, {"label_smoothing": 1.01}, {"label_smoothing": math.nan},
                                {"z_loss_coef": -1e-4}, {"z_loss_coef": math.inf}, {"z_loss_coef": math.nan}])
def test_invalid_coefficients_are_refused(kw):
    e, ws, tgt = _problem()
    for emulate in (False, True):
        with pytest.raises(ValueError):
            linear_cross_entropy(e, ws, tgt, _emulate=emulate, **kw)
    with pytest.raises(ValueError):
        LinearCrossEntropy(**kw)(e, ws[0], tgt.clamp_max(ws[0].shape[0] - 1))
    with pytest.raises(ValueError, match="loss_sums"):
        linear_cross_entropy(e, ws, tgt, z_loss_coef=0.1, loss_sums=torch.zeros(3, dtype=torch.float64))


@pytest.mark.parametrize("emulate", [False, True])
def test_zero_coefficients_are_bitwise_the_plain_call(emulate):
    results = []
    for kw in ({}, {"label_smoothing": 0.0, "z_loss_coef": 0.0}):
        e, ws, tgt = _problem()
        loss, lse = linear_cross_entropy(e, ws, tgt, reduction="none", return_lse=True, _emulate=emulate, **kw)
        loss.sum().backward()
        results.append([loss.detach(), lse, e.grad, *[w.grad for w in ws]])
    for a, b in zip(*results):
        assert torch.equal(a, b)


def test_loss_sums_count_once_under_recomputation():
    from torch.utils.checkpoint import checkpoint

    e, ws, tgt = _problem()
    sums = [torch.zeros(3), torch.zeros(3)]
    fn = lambda x, s: linear_cross_entropy(x, ws, tgt, _emulate=True, z_loss_coef=0.1, loss_sums=s)  # noqa: E731
    fn(e, sums[0]).backward()
    checkpoint(fn, e, sums[1], use_reentrant=False).backward()
    assert torch.equal(sums[0], sums[1]) and sums[0][2].item() == (tgt != -100).sum().item()
    with torch.no_grad():
        fn(e, sums[1])  # a forward without backward adds nothing
    assert torch.equal(sums[0], sums[1])


def test_lm_head_regularisation_and_sums():
    from d9d_b200.module.block.head import SplitLanguageModellingHead

    torch.manual_seed(0)
    head = SplitLanguageModellingHead({"a": 50, "b": 14}, ["a", "b"], 16)
    h = torch.randn(2, 8, 16)
    labels = torch.randint(0, 64, (2, 8))
    labels[0, :3] = -100
    plain = head(h, labels)
    head.set_loss_regularisation(0.0, 0.0)
    torch.testing.assert_close(head(h, labels), plain, rtol=0, atol=0)
    head.set_loss_regularisation(0.1, 1e-3)
    h.requires_grad_()
    loss = head(h, labels)
    w = head.classifier_weight()
    ref, _ = linear_cross_entropy_reference(h.reshape(-1, 16), w, labels.reshape(-1), None, -100, None, 0.1, 1e-3)
    torch.testing.assert_close(loss.reshape(-1), ref)
    assert (head.lm_loss_sums == 0).all()  # accumulated in backward
    loss.sum().backward()
    assert head.lm_loss_sums[2].item() == 13
    torch.testing.assert_close(head.lm_loss_sums[0], plain.sum())
    head.reset_loss_sums()
    assert (head.lm_loss_sums == 0).all()
    with pytest.raises(ValueError):
        head.set_loss_regularisation(1.5, 0.0)


# ---- Trainer ----

LM_ON = {"label_smoothing": 0.1, "z_loss_coef": 0.01}


def _lm_trainer(tmp, lm_loss, mesh_kwargs=None, schedule=None, source=None, micro=4, period=2):
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d_b200.loop.auto.auto_lr_scheduler import PiecewiseConfig
    from d9d_b200.loop.auto.auto_optimizer import SGDOptimizerConfig
    from d9d_b200.loop.config import TrainerConfig
    from d9d_b200.loop.run import TrainingConfigurator
    from tests.helpers_train import LMProvider, SFTTask, SyntheticDataProvider, dense_params, trainer_config

    cfg = trainer_config(tmp, total_batch=8, micro=micro, schedule=schedule, log_dir=tmp / "logs", source=source).model_dump()
    if lm_loss is not None:
        cfg["lm_loss"] = lm_loss
    cfg["logging"]["period_steps"] = period
    sched = PiecewiseConfig.model_validate({"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
        {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})
    return TrainingConfigurator(
        mesh=DeviceMeshParameters(**(mesh_kwargs or {})), parameters=TrainerConfig.model_validate(cfg),
        task_provider=lambda ctx: SFTTask(ctx.dist_context), model_provider=LMProvider(dense_params()),
        data_provider=SyntheticDataProvider(num_samples=32), optimizer_provider=AutoOptimizerProvider(SGDOptimizerConfig(lr=0.5)),
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


def test_trainer_null_is_bitwise_the_plain_run(tmp_path):
    from tests.helpers_train import LMProvider, dense_params  # noqa: F401

    off = _lm_trainer(tmp_path / "off", None)
    assert off.state.lm_loss is None
    ref = _trained(off)
    zero = _lm_trainer(tmp_path / "zero", {"label_smoothing": 0.0, "z_loss_coef": 0.0})
    got = _trained(zero)
    for name, value in ref.items():
        assert torch.equal(got[name], value), name
    assert _logged(tmp_path / "zero")["loss"] == _logged(tmp_path / "off")["loss"]
    assert "lm_nll" not in _logged(tmp_path / "off")
    assert set(zero.state.state_dict()) == set(off.state.state_dict())  # no checkpoint state


def test_trainer_logs_the_lm_terms_and_restarts_the_sums_every_step(tmp_path):
    on = _lm_trainer(tmp_path / "on", LM_ON, period=1)
    seen = []

    from d9d_b200.loop.event.catalogue.train import EVENT_TRAIN_STEP_PRE

    head = on.state.tracked_modules.modules[0].lm_head
    on.state.event_bus.subscribe(EVENT_TRAIN_STEP_PRE, lambda ctx: seen.append(head.lm_loss_sums.clone()))
    trained = _trained(on)
    logs = _logged(tmp_path / "on")
    nll, z = logs["lm_nll"], logs["lm_z_loss"]
    assert sorted(nll) == sorted(z) == sorted(logs["loss"]) == list(range(4))
    assert all(0 < v < 10 and math.isfinite(v) for v in nll.values()), nll
    assert all(v > 0 and math.isfinite(v) for v in z.values()), z
    assert all(logs["loss"][step] != nll[step] for step in nll)  # the logged loss is the regularised objective
    # one step's tokens only: 8 sequences of 16 tokens, their labels unmasked
    assert head.lm_loss_sums[2].item() == 8 * 16
    assert len(seen) == 4 and all(s[2].item() in (0.0, 8 * 16) for s in seen)
    ref = _trained(_lm_trainer(tmp_path / "ref", None))
    assert any(not torch.equal(trained[n], ref[n]) for n in ref)


def test_trainer_refuses_a_last_stage_without_lm_head():
    from d9d_b200.core.dist_context import DeviceMeshParameters
    from d9d_b200.loop.component import LMLoss
    from d9d_b200.loop.config import LMLossConfig
    from d9d_b200.pipelining.api import PipelineStageInfo

    class _Modules:
        def __init__(self, modules):
            self.modules = modules

    class _LastStageWithoutHead(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self._stage = PipelineStageInfo(0, 1)

    with pytest.raises(ValueError, match="LM head"):
        LMLoss(DeviceMeshParameters().build(), _Modules([_LastStageWithoutHead()]), LMLossConfig(z_loss_coef=1e-4))
    with pytest.raises(ValueError):
        LMLossConfig(label_smoothing=1.5)
    with pytest.raises(ValueError):
        LMLossConfig(z_loss_coef=-1.0)


def _pp_worker(rank, world, tmp, mesh_kwargs, schedule, source):
    from pathlib import Path

    trainer = _lm_trainer(Path(tmp), LM_ON, mesh_kwargs, schedule, source=Path(source), micro=2, period=1)
    trainer.train()
    trainer.export(Path(tmp) / "export", load_checkpoint=False)


@pytest.mark.dist
def test_pipeline_parallel_run_matches_one_process(tmp_path):
    from d9d_b200.model_state.io import load_model_state
    from d9d_b200.model_state.mapper.adapters import identity_mapper_from_module

    mesh_kwargs = {"pipeline_parallel": 2}
    schedule = {"schedule": "1f1b", "num_stages_per_rank": 1, "zero_bubble": False}
    _lm_trainer(tmp_path / "init", LM_ON).export(tmp_path / "init" / "export", load_checkpoint=False)  # one initial model
    source = tmp_path / "init" / "export"
    single = _lm_trainer(tmp_path / "one", LM_ON, source=source, micro=2, period=1)
    single.train()
    ref_state = {k: v.clone() for k, v in single.state.tracked_modules.modules[0].state_dict().items()}
    run_distributed(_pp_worker, 2, str(tmp_path / "dist"), mesh_kwargs, schedule, str(source))
    model = _lm_trainer(tmp_path / "load", LM_ON).state.tracked_modules.modules[0]
    load_model_state(tmp_path / "dist" / "export", identity_mapper_from_module(model), "cpu", model, show_progress=False)

    ref, got = _logged(tmp_path / "one"), _logged(tmp_path / "dist")
    for name in ("loss", "lm_nll", "lm_z_loss"):
        assert sorted(got[name]) == sorted(ref[name]) == list(range(4)), name
        for step, value in ref[name].items():
            assert got[name][step] == pytest.approx(value, rel=1e-5, abs=1e-7), (name, step)
    for name, value in ref_state.items():
        torch.testing.assert_close(model.state_dict()[name], value, rtol=1e-4, atol=1e-6, msg=lambda m, n=name: f"{n}: {m}")

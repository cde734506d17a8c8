"""The fused router kernel with the DeepSeek routing options (sigmoid scores, group-limited selection, weight scaling)
against ``route_topk_general``, and against the written selection rule where ``torch.topk``'s tie order is unspecified."""

import pytest
import torch

pytestmark = pytest.mark.gpu

# every bf16 value with magnitude in [0.25, 4): 2 signs x 4 binades x 128 mantissas = 1024 distinct logits, adjacent ones
# far enough apart that softmax / sigmoid scores never tie within fp32 rounding
_LOGIT_POOL = None


def _logit_pool() -> torch.Tensor:
    global _LOGIT_POOL
    if _LOGIT_POOL is None:
        mags = torch.tensor([(1 + m / 128) * 2.0 ** ex for ex in range(-2, 2) for m in range(128)])
        _LOGIT_POOL = torch.cat([mags, -mags]).bfloat16()
    return _LOGIT_POOL


def _distinct_logits(T: int, E: int, gen: torch.Generator) -> torch.Tensor:
    pool = _logit_pool()
    rows = [pool[torch.randperm(pool.numel(), generator=gen)[:E]] for _ in range(T)]
    return torch.stack(rows) if rows else torch.empty(0, E, dtype=torch.bfloat16)


def _well_separated(logits, bias, score, k, G, topk_groups) -> torch.Tensor:
    """Rows whose k-th / (k+1)-th key and topk_groups-th / next group score differ clearly (fp64 keys)."""
    x = logits.double()
    s = torch.softmax(x, -1) if score == "softmax" else torch.sigmoid(x)
    keys = s if bias is None else s + bias.double()
    ok = torch.ones(x.shape[0], dtype=torch.bool)
    if G > 1:
        per = keys.view(x.shape[0], G, x.shape[1] // G)
        gs = per.topk(min(2, per.shape[-1]), -1).values.sum(-1)
        top = gs.sort(-1, descending=True).values
        if topk_groups < G:
            ok &= (top[:, topk_groups - 1] - top[:, topk_groups]) > 1e-5 * top[:, 0].abs()
        keep = torch.zeros_like(gs, dtype=torch.bool).scatter_(-1, gs.topk(topk_groups, -1).indices, True)
        keys = per.masked_fill(~keep.unsqueeze(-1), float("-inf")).view_as(keys)
    top = keys.sort(-1, descending=True).values
    if k < keys.shape[-1]:
        ok &= (top[:, k - 1] - top[:, k]) > 1e-5 * top[:, 0].abs()
    return ok


def _inputs(T, E, k, G, topk_groups, score, with_bias, seed):
    gen = torch.Generator().manual_seed(seed)
    # non-negative bias: eligible keys stay positive, so experts of dropped groups (key 0.0) are never picked and the
    # selection is unique (the masked-zero semantics have their own test)
    bias = (torch.rand(E, generator=gen) * 0.1) if with_bias else None
    logits = _distinct_logits(T, E, gen)
    for _ in range(20):
        bad = ~_well_separated(logits, bias, score, k, G, topk_groups)
        if not bad.any():
            break
        logits[bad] = _distinct_logits(int(bad.sum()), E, gen)
    else:
        raise AssertionError("could not draw well-separated router inputs")
    return logits.cuda(), (bias.cuda() if bias is not None else None)


def _sorted_by_expert(idx, probs):
    order = idx.argsort(-1)
    return idx.gather(-1, order), probs.gather(-1, order), order


def _compare(logits, bias, k, renorm, score, G, topk_groups, scale):
    from d9d_b200.kernel.router import route_topk, route_topk_general

    a = logits.clone().requires_grad_()
    b = logits.clone().float().requires_grad_()
    idx, probs = route_topk(a, k, renorm, bias, score, G, topk_groups, scale)
    ridx, rprobs = route_topk_general(b, k, renorm, bias, score, G, topk_groups, scale)
    assert idx.shape == ridx.shape and probs.dtype == torch.float32
    idx_s, probs_s, order = _sorted_by_expert(idx, probs)
    ridx_s, rprobs_s, rorder = _sorted_by_expert(ridx, rprobs)
    assert torch.equal(idx_s, ridx_s)
    torch.testing.assert_close(probs_s, rprobs_s, rtol=1e-5, atol=0)
    w = torch.randn(*idx.shape, device="cuda")
    (probs_s * w).sum().backward()
    (rprobs_s * w).sum().backward()
    if logits.shape[0] == 0:
        return
    torch.testing.assert_close(a.grad.float(), b.grad, rtol=2e-2, atol=2e-3 * float(b.grad.abs().max()))


CASES = [  # E, k, G, topk_groups
    (256, 8, 8, 4),    # DeepSeek-V3
    (160, 6, 8, 3),    # group size 20: not a multiple of 32
    (384, 8, 1, 1),    # Kimi-K2-like (with sigmoid), 16 experts per lane
    (64, 6, 1, 1),
    (8, 3, 4, 2),      # the transformers parity config
    (32, 4, 32, 8),    # one expert per group
    (1024, 32, 32, 8),
]


@pytest.mark.parametrize("E,k,G,topk_groups", CASES)
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
@pytest.mark.parametrize("renorm", [True, False])
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("scale", [1.0, 2.5])
def test_native_router_matches_general(E, k, G, topk_groups, score, renorm, with_bias, scale):
    logits, bias = _inputs(777, E, k, G, topk_groups, score, with_bias, seed=E * 31 + k)
    _compare(logits, bias, k, renorm, score, G, topk_groups, scale)


@pytest.mark.parametrize("T", [0, 1])
@pytest.mark.parametrize("score", ["softmax", "sigmoid"])
def test_native_router_tiny_token_counts(T, score):
    logits, bias = _inputs(T, 256, 8, 8, 4, score, True, seed=T)
    _compare(logits, bias, 8, True, score, 8, 4, 2.5)


def test_native_router_batched_input():
    from d9d_b200.kernel.router import route_topk, route_topk_general

    logits, bias = _inputs(2 * 129, 256, 8, 8, 4, "sigmoid", True, seed=5)
    x = logits.view(2, 129, 256)
    idx, probs = route_topk(x, 8, True, bias, "sigmoid", 8, 4, 2.5)
    ridx, rprobs = route_topk_general(x.float(), 8, True, bias, "sigmoid", 8, 4, 2.5)
    assert idx.shape == (2, 129, 8) and probs.shape == (2, 129, 8)
    i, p, _ = _sorted_by_expert(idx, probs)
    ri, rp, _ = _sorted_by_expert(ridx, rprobs)
    assert torch.equal(i, ri)
    torch.testing.assert_close(p, rp, rtol=1e-5, atol=0)


def _native(logits, bias, k, G, topk_groups, score="sigmoid", renorm=False, scale=1.0):
    from d9d_b200.kernel.router import route_topk

    return route_topk(logits.cuda(), k, renorm, None if bias is None else bias.cuda(), score, G, topk_groups, scale)


def test_equal_keys_go_to_the_lower_expert():
    # all logits equal: every key ties, the k lowest expert indices win
    logits = torch.zeros(3, 64, dtype=torch.bfloat16)
    idx, _ = _native(logits, None, 5, 1, 1)
    assert idx.cpu().tolist() == [[0, 1, 2, 3, 4]] * 3
    # equal group scores: the lower groups win; within them the lower experts
    idx, _ = _native(logits, None, 6, 8, 2)
    assert sorted(idx[0].cpu().tolist()) == [0, 1, 2, 3, 4, 5]
    bias = torch.zeros(64)
    bias[40:48] = 0.25  # group 5 is clearly best; the second group is a tie between all others -> group 0
    idx, _ = _native(logits, bias, 10, 8, 2)
    assert sorted(idx[0].cpu().tolist()) == [0, 1, 40, 41, 42, 43, 44, 45, 46, 47]


def test_experts_of_dropped_groups_get_key_zero():
    # sigmoid(0) = 0.5, so the keys are 0.5 + bias: all negative.  Group 0 (experts 0, 1) has the best group score and is
    # the only one kept; the experts of the dropped groups 1-3 get key 0.0, which outranks the kept negative keys, so they
    # are picked first, lower index first, as the written rule says.
    E, G = 8, 4
    logits = torch.zeros(1, E, dtype=torch.bfloat16)
    bias = torch.tensor([-0.9, -0.8, -1.0, -1.0, -1.0, -1.0, -1.0, -1.0])
    idx, probs = _native(logits, bias, 3, G, 1)
    assert idx[0].cpu().tolist() == [2, 3, 4]
    torch.testing.assert_close(probs.cpu(), torch.full((1, 3), 0.5))
    # when fewer than k experts remain with key 0.0, the best negative keys of the kept group follow
    idx, _ = _native(logits, bias, 8, G, 1)
    assert idx[0].cpu().tolist() == [2, 3, 4, 5, 6, 7, 1, 0]


def test_deepseek_v3_moe_layer_native_matches_general(monkeypatch):
    from d9d_b200.kernel import router as router_kernels
    from d9d_b200.module.block.moe import MoELayer
    from d9d_b200.module.block.moe import router as router_module
    from d9d_b200.module.model.deepseek_v3 import deepseek_v3_router

    E, k, H, F = 64, 6, 256, 192
    torch.manual_seed(7)
    layer = MoELayer(hidden_dim=H, intermediate_dim_grouped=F, num_grouped_experts=E, top_k=k, router_renormalize_probabilities=True,
                     router=deepseek_v3_router(n_group=8, topk_group=4, routed_scaling_factor=2.5))
    layer.reset_parameters()
    layer = layer.cuda().bfloat16()
    with torch.no_grad():
        layer.router.expert_bias.copy_(torch.randperm(E).float() * 2.0 ** -9)
    x0 = torch.randn(2, 64, H, device="cuda").bfloat16()

    def run():
        layer.zero_grad(set_to_none=True)
        layer.reset_stats()
        x = x0.clone().requires_grad_()
        routing = layer.router(x.view(-1, H))
        y = layer(x)
        (y.float() * torch.linspace(-1, 1, H, device="cuda")).sum().backward()
        return (routing.selected_expert_indices.sort(-1).values, y.detach().float(), x.grad.float(),
                layer.router.gate.weight.grad.float(), layer.tokens_per_expert.clone())

    native = run()
    monkeypatch.setattr(router_module, "route_topk", router_kernels.route_topk_general)
    general = run()
    assert torch.equal(native[0], general[0])
    assert torch.equal(native[4], general[4])
    for got, ref in zip(native[1:4], general[1:4]):
        torch.testing.assert_close(got, ref, rtol=2e-2, atol=2e-2 * float(ref.abs().max()))

"""Multi-head latent attention on the native flash attention kernels at DeepSeek-V2 / V3's head dims (qk 128 nope + 64 rope
= 192, v 128): a DeepSeek-V2 model against its fp32 CPU copy, the packed-batch entry point without a host sync, and the
ring attention block plan emulated on one GPU."""

import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

DQK, DV = 192, 128


def _tiny_deepseek_v2():
    from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode
    from d9d_b200.module.model.deepseek_v2 import (DeepseekV2ForCausalLM, DeepseekV2ForCausalLMParameters,
                                                   DeepseekV2LayerParameters, DeepseekV2Parameters)
    from d9d_b200.pipelining.api import PipelineStageInfo

    p = DeepseekV2ForCausalLMParameters(model=DeepseekV2Parameters(
        layer=DeepseekV2LayerParameters(hidden_size=256, rms_norm_eps=1e-6, num_attention_heads=4, qk_nope_head_dim=128,
                                        qk_rope_head_dim=64, v_head_dim=128, kv_lora_rank=128, q_lora_rank=None,
                                        intermediate_size=192, first_k_dense_replace=1, moe_intermediate_size=192, num_experts=8,
                                        experts_top_k=2, num_shared_experts=1),
        num_hidden_layers=2, rope_base=10000, max_position_ids=256,
        split_vocab_size={"regular": 1000, "special": 24}, split_vocab_order=["regular", "special"]))
    return DeepseekV2ForCausalLM(p, PipelineStageInfo(0, 1), HiddenStatesAggregationMode.no, False)


def _cos(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return torch.nn.functional.cosine_similarity(a, b, dim=0).item()


def test_deepseek_v2_native_vs_oracle(monkeypatch):
    """Loss and every gradient of the bf16 CUDA model (native attention at (192, 128)) against the fp32 CPU model."""
    import d9d_b200.kernel.flash_attn.native as native

    calls = []
    real = native.flash_attention

    def counting(q, k, v, *a, **kw):
        calls.append((q.shape[-1], k.shape[-1], v.shape[-1]))
        return real(q, k, v, *a, **kw)

    def no_sdpa(*a, **kw):
        raise AssertionError("SDPA ran on the latent attention path")

    torch.manual_seed(0)
    ref = _tiny_deepseek_v2()
    ref.reset_parameters()
    ref = ref.bfloat16().float()
    ref.model.rope_provider.reset_parameters()
    gpu = copy.deepcopy(ref).bfloat16().cuda()
    gpu.model.rope_provider.reset_parameters()

    ids = torch.randint(0, 1024, (2, 128))
    labels = torch.randint(0, 1024, (2, 128))
    labels[0, :5] = -100
    pos = torch.arange(128)[None].expand(2, -1).contiguous()

    out_ref = ref(input_ids=ids, position_ids=pos, labels=labels)
    monkeypatch.setattr(native, "flash_attention", counting)
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", no_sdpa)
    out_gpu = gpu(input_ids=ids.cuda(), position_ids=pos.cuda(), labels=labels.cuda())
    assert calls == [(DQK, DQK, DV)] * 2, calls
    l_ref, l_gpu = out_ref["logps"].sum() / 251, out_gpu["logps"].sum() / 251
    assert abs(l_ref.item() - l_gpu.item()) < 3e-2, (l_ref.item(), l_gpu.item())
    l_ref.backward()
    l_gpu.backward()
    bad = []
    for (n, p_ref), (_, p_gpu) in zip(ref.named_parameters(), gpu.named_parameters()):
        assert p_gpu.grad is not None, n
        c = _cos(p_ref.grad, p_gpu.grad.cpu())
        ratio = (p_gpu.grad.float().norm().item() + 1e-12) / (p_ref.grad.norm().item() + 1e-12)
        if c < 0.98 or not (0.9 < ratio < 1.1):
            bad.append((n, c, ratio))
    assert not bad, bad


def test_latent_attention_sdpa_fallback_pads_v():
    """Head dims without a native kernel take SDPA on V padded to the qk head dim; the caller still sees out [..., Dv]."""
    from d9d_b200.kernel.flash_attn import attention_reference, flash_attn_func

    torch.manual_seed(3)
    q = torch.randn(2, 100, 4, 96, device="cuda").bfloat16()
    k = torch.randn(2, 100, 4, 96, device="cuda").bfloat16()
    v = torch.randn(2, 100, 4, 64, device="cuda").bfloat16()
    out, _ = flash_attn_func(q, k, v, causal=True)
    assert out.shape == (2, 100, 4, 64)
    want, _ = attention_reference(q.float(), k.float(), v.float(), None, True)
    torch.testing.assert_close(out.float(), want, rtol=2e-2, atol=2e-2)


def test_varlen_makes_no_host_sync():
    from d9d_b200.kernel.flash_attn import flash_attn_varlen_func

    lens = [100, 300, 7, 257]
    total = sum(lens)
    cu = torch.tensor([0] + [sum(lens[: i + 1]) for i in range(len(lens))], dtype=torch.int32, device="cuda")
    q = torch.randn(total, 4, DQK, device="cuda").bfloat16().requires_grad_()
    k = torch.randn(total, 1, DQK, device="cuda").bfloat16().requires_grad_()
    v = torch.randn(total, 1, DV, device="cuda").bfloat16().requires_grad_()
    dout = torch.randn(total, 4, DV, device="cuda").bfloat16()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out, _ = flash_attn_varlen_func(q, k, v, cu, cu, max(lens), max(lens), causal=True)
        dq, dk, dv = torch.autograd.grad(out, (q, k, v), dout)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert out.shape == (total, 4, DV) and dq.shape == q.shape and dk.shape == k.shape and dv.shape == v.shape
    assert bool(torch.isfinite(out.float()).all()) and bool(torch.isfinite(dq.float()).all())


@pytest.mark.parametrize("causal", [True, False])
def test_ring_block_plan_at_192_128(causal):
    """Every "rank" walks all K/V blocks with the ring's call plan / merge / gradient routines, on the (192, 128) kernels,
    against fp32 attention over the whole sequence."""
    from d9d_b200.kernel.context_parallel import ContextParallelLayout, local_sequence_indices, shard_sequence
    from d9d_b200.kernel.context_parallel import ring
    from d9d_b200.kernel.flash_attn import attention_reference

    world, batch, seq, heads = 4, 2, 2048, 4
    layout = ContextParallelLayout.zigzag
    torch.manual_seed(0)
    q = (torch.randn(batch, seq, heads, DQK, device="cuda") * 0.5).bfloat16()
    k = (torch.randn(batch, seq, heads, DQK, device="cuda") * 0.5).bfloat16()
    v = (torch.randn(batch, seq, heads, DV, device="cuda") * 0.5).bfloat16()
    w = torch.randn(batch, seq, heads, DV, device="cuda").bfloat16()
    assert ring._use_plan("auto", q, k, v)  # noqa: SLF001
    qr, kr, vr = (t.float().requires_grad_() for t in (q, k, v))
    out_ref, _ = attention_reference(qr, kr, vr, None, causal)
    (out_ref * w.float()).sum().backward()

    positions = torch.stack([local_sequence_indices(seq, world, r, layout) for r in range(world)])
    shards = [[shard_sequence(t, 1, world, r, layout).contiguous() for t in (q, k, v, w)] for r in range(world)]
    scale = DQK ** -0.5
    dk_total = [torch.zeros_like(shards[r][1], dtype=torch.float32) for r in range(world)]
    dv_total = [torch.zeros_like(shards[r][2], dtype=torch.float32) for r in range(world)]
    for rank in range(world):
        plan = ring._BlockPlan(positions, rank, causal)  # noqa: SLF001
        masks = ring._Masks(positions, rank, causal, q.device, {})  # noqa: SLF001
        ql, _, _, wl = shards[rank]
        out = lse = None
        for src in range(world):
            if masks.get(src) is False:
                continue
            calls = plan.calls(src)
            assert calls is not None
            o_b, l_b = ring._plan_forward(ql, shards[src][1], shards[src][2], scale, calls)  # noqa: SLF001
            out, lse = ring._merge(out, lse, o_b, l_b)  # noqa: SLF001
        result = out.to(q.dtype)
        assert result.shape[-1] == DV
        want = shard_sequence(out_ref.detach(), 1, world, rank, layout)
        assert ((result.float() - want).norm() / want.norm()).item() < 2e-2
        delta = (wl.float() * result.float()).sum(-1).transpose(1, 2)
        dq = torch.zeros_like(ql, dtype=torch.float32)
        for src in range(world):
            if masks.get(src) is False:
                continue
            dq_b, dk_b, dv_b = ring._plan_backward(ql, shards[src][1], shards[src][2], wl, result, lse, delta, scale, plan.calls(src))  # noqa: SLF001
            dq += dq_b
            dk_total[src] += dk_b
            dv_total[src] += dv_b
        want_dq = shard_sequence(qr.grad, 1, world, rank, layout)
        assert ((dq - want_dq).norm() / want_dq.norm()).item() < 3e-2
    for r in range(world):
        want_dk = shard_sequence(kr.grad, 1, world, r, layout)
        want_dv = shard_sequence(vr.grad, 1, world, r, layout)
        assert ((dk_total[r] - want_dk).norm() / want_dk.norm()).item() < 3e-2
        assert ((dv_total[r] - want_dv).norm() / want_dv.norm()).item() < 3e-2

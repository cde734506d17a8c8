"""Ring attention's block plan on the native wgmma flash-attention kernels, emulated on ONE GPU: every "rank" walks all
K/V blocks with the same call plan / merge / gradient routines the distributed ring uses (`kernel/context_parallel/ring.py`),
and the result is compared with fp32 attention over the whole sequence."""

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("layout_name", ["zigzag", "contiguous"])
@pytest.mark.parametrize("causal", [True, False])
def test_ring_block_plan_on_native_kernels(layout_name, causal):
    from d9d_b200.kernel.context_parallel import ContextParallelLayout, local_sequence_indices, shard_sequence
    from d9d_b200.kernel.context_parallel import ring
    from d9d_b200.kernel.flash_attn import attention_reference

    world, batch, seq, heads, kv_heads, dim = 4, 2, 2048, 8, 2, 128
    layout = ContextParallelLayout(layout_name)
    torch.manual_seed(0)
    q = (torch.randn(batch, seq, heads, dim, device="cuda") * 0.5).bfloat16()
    k = (torch.randn(batch, seq, kv_heads, dim, device="cuda") * 0.5).bfloat16()
    v = (torch.randn(batch, seq, kv_heads, dim, device="cuda") * 0.5).bfloat16()
    w = torch.randn(batch, seq, heads, dim, device="cuda").bfloat16()
    qr, kr, vr = (t.float().requires_grad_() for t in (q, k, v))
    out_ref, _ = attention_reference(qr, kr, vr, None, causal)
    (out_ref * w.float()).sum().backward()

    positions = torch.stack([local_sequence_indices(seq, world, r, layout) for r in range(world)])
    shards = [[shard_sequence(t, 1, world, r, layout).contiguous() for t in (q, k, v, w)] for r in range(world)]
    scale = dim ** -0.5
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

"""fp8 expert block on the H100: the batched and segment-wise transposing quantisers against their PyTorch emulations,
the grouped e4m3 GEMMs (GROUPED_M / GROUPED_K) against an fp64 product of their dequantised operands with a per-element
bound, and ``grouped_swiglu(fp8=True)`` against the emulation of the same recipe and against the bf16 block."""

import math

import pytest
import torch

from d9d_b200.kernel import fp8

pytestmark = pytest.mark.gpu

U_CHAIN = 2.0**-13  # assumed unit roundoff of the tensor core's e4m3 accumulation inside one 128-deep k-block
U_F32 = 2.0**-24
U_BF16 = 2.0**-8


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _layout_from_counts(counts, device="cuda"):
    """A MoE layout ([E] counts -> 128-aligned segments, tile table) built on the host, for exact control of the sizes."""
    from d9d_b200.kernel.moe.layout import ALIGN, MoELayout

    E = len(counts)
    aligned = [(c + ALIGN - 1) // ALIGN * ALIGN for c in counts]
    seg = [0]
    for a in aligned:
        seg.append(seg[-1] + a)
    cap = seg[-1] + 2 * ALIGN  # two unused tiles at the end (tile_group -1)
    tiles = [-1] * (cap // ALIGN)
    for e in range(E):
        for t in range(seg[e] // ALIGN, seg[e + 1] // ALIGN):
            tiles[t] = e
    i32 = dict(dtype=torch.int32, device=device)
    return MoELayout(torch.tensor(counts, **i32), torch.tensor(seg, **i32), torch.empty(0, **i32), torch.tensor(tiles, **i32),
                     0, 1, E, cap)


def _mismatch_ok(q, qr):
    # the kernels multiply by a fast-math reciprocal of the scale, the emulation divides: at most one e4m3 step apart,
    # and only rarely
    a, b = q.float(), qr.float()
    diff = a != b
    if diff.any():
        step = (a - b).abs()[diff] / b.abs()[diff].clamp_min(2.0**-9)
        assert float(step.max()) <= 0.125 + 1e-6
    return float(diff.float().mean())


# ------------------------------------------------------------------------------------------ quantisers
@pytest.mark.parametrize("E,R,C", [(1, 256, 96), (8, 576, 768), (128, 64, 48)])
def test_batched_transposing_quantiser(ops, E, R, C):
    x = (torch.randn(E, R, C, device="cuda") * torch.logspace(-2, 2, C, device="cuda")).bfloat16()
    x[0, :, 3] = 0
    q, s = ops.quantize_colwise_t_batched(x)
    qr, sr = fp8.quantize_colwise_t_batched_reference(x)
    assert q.shape == (E, C, R) and s.shape == (E, C)
    torch.testing.assert_close(s, sr, rtol=1e-6, atol=0)
    assert float(s[0, 3]) == 1.0 and not q[0, 3].float().any()
    assert _mismatch_ok(q, qr) < 0.02


def test_segment_quantiser_sizes_pads_and_empty_experts(ops):
    counts = [0, 1, 127, 128, 129, 0, 300, 5]
    lay = _layout_from_counts(counts)
    C = 80
    x = (torch.randn(lay.capacity, C, device="cuda") * 3).bfloat16()
    seg = lay.seg_offsets.tolist()
    for e, n in enumerate(counts):  # pad rows hold NaN and huge values: they must come out as zeros
        x[seg[e] + n : seg[e + 1]] = float("nan")
        if seg[e + 1] > seg[e] + n + 1:
            x[seg[e] + n + 1] = 1e30
    x[seg[-1]:] = float("nan")
    x[seg[6] : seg[6] + 300, 7] = 0  # an all-zero column of one expert: scale 1
    torch.cuda.synchronize()
    with torch.cuda.graph(torch.cuda.CUDAGraph()):  # capturable: no host synchronisation inside
        ops.quantize_segments_t(x, lay.tile_group, lay.seg_offsets, lay.counts)
    q, s = ops.quantize_segments_t(x, lay.tile_group, lay.seg_offsets, lay.counts)
    qr, sr = fp8.quantize_segments_t_reference(x, seg[:-1], counts)
    torch.testing.assert_close(s, sr, rtol=1e-6, atol=0)
    assert (s[0] == 1).all() and (s[5] == 1).all() and float(s[6, 7]) == 1.0
    valid = torch.zeros(lay.capacity, dtype=torch.bool, device="cuda")
    for e, n in enumerate(counts):
        valid[seg[e] : seg[e] + n] = True
    assert not q[:, ~valid].float().any()  # exact zeros outside the experts' rows
    assert torch.isfinite(q.float()).all()
    assert _mismatch_ok(q, qr) < 0.02


def test_segment_quantiser_one_expert_holds_all_tokens(ops):
    counts = [0, 16000, 0]
    lay = _layout_from_counts(counts)
    x = torch.randn(lay.capacity, 64, device="cuda").bfloat16()
    q, s = ops.quantize_segments_t(x, lay.tile_group, lay.seg_offsets, lay.counts)
    qr, sr = fp8.quantize_segments_t_reference(x, lay.seg_offsets[:-1].tolist(), counts)
    torch.testing.assert_close(s, sr, rtol=1e-6, atol=0)
    assert _mismatch_ok(q, qr) < 0.02


# ------------------------------------------------------------------------------------------ grouped GEMMs
def _bound(a_abs_dot, k_blocks):
    """Per-element bound on |D - exact| from the accumulation, given sum_k |a_k b_k| (scaled): in-chain accumulation at
    U_CHAIN per 128-deep k-block, fp32 across k-blocks and for the scaling.  Callers add the output rounding."""
    chain = 128 * U_CHAIN * a_abs_dot
    across = (k_blocks + 3) * U_F32 * a_abs_dot
    return chain + across


def _check(d, exact, absdot, k_blocks, out_bf16, what):
    bound = _bound(absdot, k_blocks) + (U_BF16 * exact.abs() if out_bf16 else 0) + 1e-30
    ratio = float(((d.double() - exact).abs() / bound).max())
    print(f"{what}: worst err / bound = {ratio:.3f}")
    assert ratio <= 1.0, what
    return ratio


def _grouped_m_reference(aq, sa, bq, sb, tiles, N):
    a = aq.double() * sa.double()[:, None]
    out = torch.zeros(aq.shape[0], N, dtype=torch.float64, device=aq.device)
    absd = torch.zeros_like(out)
    for t, e in enumerate(tiles.tolist()):
        if e < 0:
            continue
        rows = slice(128 * t, 128 * t + 128)
        b = bq[e].double() * sb.view(-1, N)[e].double()[:, None]
        out[rows] = a[rows] @ b.t()
        absd[rows] = a[rows].abs() @ b.abs().t()
    return out, absd


@pytest.mark.parametrize("E,counts,K,N", [(4, [300, 0, 1, 129], 576, 576), (128, None, 256, 768)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_grouped_m_against_fp64(ops, E, counts, K, N, accumulate):
    g = torch.Generator().manual_seed(E + K)
    if counts is None:
        counts = torch.randint(0, 40, (E,), generator=g).tolist()
        counts[3] = 0
    lay = _layout_from_counts(counts)
    cap = lay.capacity
    a = torch.randn(cap, K, device="cuda").bfloat16()
    w = (torch.randn(E, N, K, device="cuda") * 0.05).bfloat16()
    aq, sa = ops.quantize_rowwise(a)
    bq, sb = ops.quantize_rowwise(w.view(E * N, K))
    bq = bq.view(E, N, K)
    canary = 7.0
    d = torch.full((cap, N), canary, device="cuda", dtype=torch.bfloat16)
    base = d.clone()
    if accumulate:
        d.normal_()
        base = d.clone()
    ops.gemm_fp8_grouped_m(aq, sa, bq, sb, d, lay.tile_group, accumulate)
    exact, absd = _grouped_m_reference(aq, sa, bq, sb, lay.tile_group, N)
    used = lay.tile_group.repeat_interleave(128) >= 0
    assert torch.equal(d[~used], base[~used])  # -1 tiles are never written
    k_blocks = math.ceil(K / 128)
    if accumulate:
        # TMA reduce-add: rn(D + rn_bf16(acc))
        exact_acc = exact[used] + base[used].double()
        bound = _bound(absd[used], k_blocks) + U_BF16 * (exact[used].abs() + exact_acc.abs()) + 1e-30
        ratio = float(((d[used].double() - exact_acc).abs() / bound).max())
        print(f"grouped_m acc: worst err / bound = {ratio:.3f}")
        assert ratio <= 1.0
    else:
        _check(d[used], exact[used], absd[used], k_blocks, True, f"grouped_m E={E} K={K} N={N}")
    d2 = torch.full_like(d, canary) if not accumulate else base.clone()
    ops.gemm_fp8_grouped_m(aq, sa, bq, sb, d2, lay.tile_group, accumulate)
    assert torch.equal(d, d2)  # bitwise reproducible


@pytest.mark.parametrize("counts,M,N", [([300, 0, 1, 129, 128], 576, 768), ([16000], 128, 192), ([0] * 60 + [5] * 68, 256, 64)])
@pytest.mark.parametrize("dtype,accumulate", [(torch.float32, False), (torch.float32, True), (torch.bfloat16, False),
                                              (torch.bfloat16, True)])
def test_grouped_k_against_fp64(ops, counts, M, N, dtype, accumulate):
    lay = _layout_from_counts(counts)
    E, cap = len(counts), lay.capacity
    x = torch.randn(cap, M, device="cuda").bfloat16()
    dy = torch.randn(cap, N, device="cuda").bfloat16()
    xq, sx = ops.quantize_segments_t(x, lay.tile_group, lay.seg_offsets, lay.counts)
    dq, sd = ops.quantize_segments_t(dy, lay.tile_group, lay.seg_offsets, lay.counts)
    d = torch.randn(E, M, N, device="cuda").to(dtype)
    base = d.clone()
    ops.gemm_fp8_grouped_k(xq, sx, dq, sd, d, lay.seg_offsets, accumulate)
    seg = lay.seg_offsets.tolist()
    worst = 0.0
    for e in range(E):
        rows = slice(seg[e], seg[e + 1])
        a = xq[:, rows].double() * sx[e].double()[:, None]
        b = dq[:, rows].double() * sd[e].double()[:, None]
        exact, absd = a @ b.t(), a.abs() @ b.abs().t()
        if counts[e] == 0:
            want = base[e] if accumulate else torch.zeros_like(base[e])
            assert torch.equal(d[e], want), e
            continue
        kb = (seg[e + 1] - seg[e]) // 128
        got = d[e].double()
        target = exact + (base[e].double() if accumulate else 0)
        bound = _bound(absd, kb) + 1e-30
        if dtype == torch.bfloat16:
            bound = bound + U_BF16 * (exact.abs() + target.abs())
        elif accumulate:
            bound = bound + U_F32 * target.abs()
        worst = max(worst, float(((got - target).abs() / bound).max()))
    print(f"grouped_k counts={len(counts)} experts M={M} N={N} {dtype} acc={accumulate}: worst err / bound = {worst:.3f}")
    assert worst <= 1.0
    d2 = base.clone()
    ops.gemm_fp8_grouped_k(xq, sx, dq, sd, d2, lay.seg_offsets, accumulate)
    assert torch.equal(d, d2)


def test_grouped_k_long_reduction_error_is_that_of_promoted_accumulation(ops):
    """Norm-wise error of fp32 weight gradients against fp64, per expert.  With random inputs and round-to-nearest at
    U_CHAIN inside a chain, a chain of n products has an rms error of U_CHAIN * sqrt(sum_i i / 3) in units of one product's
    rms, so relative to the result's rms (sqrt(k) products):
      promoted (n = 128 per k-block, fp32 across blocks)   rel ~= U_CHAIN * sqrt(129 / 6)       (independent of k)
      one chain over all k tokens                          rel ~= U_CHAIN * sqrt((k + 1) / 6)
    At k = 16 000 the second is 11x the first.  The test allows 3x the promoted value, which also catches any per-expert
    scale mistake (an O(1) relative error)."""
    counts = [16000, 130, 0, 1000]
    lay = _layout_from_counts(counts)
    M, N = 128, 192
    x = torch.randn(lay.capacity, M, device="cuda").bfloat16()
    dy = torch.randn(lay.capacity, N, device="cuda").bfloat16()
    xq, sx = ops.quantize_segments_t(x, lay.tile_group, lay.seg_offsets, lay.counts)
    dq, sd = ops.quantize_segments_t(dy, lay.tile_group, lay.seg_offsets, lay.counts)
    d = torch.empty(len(counts), M, N, device="cuda")
    ops.gemm_fp8_grouped_k(xq, sx, dq, sd, d, lay.seg_offsets, False)
    seg = lay.seg_offsets.tolist()
    promoted = U_CHAIN * math.sqrt(129 / 6)
    for e, n in enumerate(counts):
        if n < 128:
            continue
        rows = slice(seg[e], seg[e + 1])
        exact = (xq[:, rows].double() * sx[e].double()[:, None]) @ (dq[:, rows].double() * sd[e].double()[:, None]).t()
        rel = float((d[e].double() - exact).norm() / exact.norm())
        one_chain = U_CHAIN * math.sqrt((n + 1) / 6)
        print(f"grouped_k {n} tokens: rel err {rel:.2e}; model: promoted {promoted:.2e}, one chain {one_chain:.2e}")
        assert rel <= 3 * promoted, (n, rel)


def test_grouped_ops_refuse_bad_operands(ops):
    lay = _layout_from_counts([128, 0])
    cap = lay.capacity
    aq, sa = ops.quantize_rowwise(torch.randn(cap, 64, device="cuda").bfloat16())
    bq, sb = ops.quantize_rowwise(torch.randn(2 * 32, 64, device="cuda").bfloat16())
    bq = bq.view(2, 32, 64)
    d = torch.zeros(cap, 32, device="cuda", dtype=torch.bfloat16)
    bad = [
        lambda: ops.gemm_fp8_grouped_m(aq.float(), sa, bq, sb, d, lay.tile_group, False),  # dtype
        lambda: ops.gemm_fp8_grouped_m(aq, sa[:-1], bq, sb, d, lay.tile_group, False),  # sa length
        lambda: ops.gemm_fp8_grouped_m(aq, sa, bq, sb[:-1], d, lay.tile_group, False),  # sb length E*N
        lambda: ops.gemm_fp8_grouped_m(aq, sa, bq, sb, d, lay.tile_group[:-1], False),  # tile table size
        lambda: ops.gemm_fp8_grouped_m(aq, sa, bq, sb, d[:, :24], lay.tile_group, False),  # output shape
        lambda: ops.gemm_fp8_grouped_m(aq, sa, bq, sb.cpu(), d, lay.tile_group, False),  # device
        lambda: ops.gemm_fp8_grouped_k(aq.t(), sa, aq.t(), sa, torch.zeros(2, 64, 64, device="cuda"), lay.seg_offsets, False),
        lambda: ops.gemm_fp8_grouped_k(aq.t().contiguous(), sa[:128], aq.t().contiguous(), sa[:128],
                                       torch.zeros(2, 64, 64, device="cuda"), lay.seg_offsets[:-1], False),  # offsets
        lambda: ops.gemm_fp8_grouped_k(aq.t().contiguous(), sa[:127], aq.t().contiguous(), sa[:128],
                                       torch.zeros(2, 64, 64, device="cuda"), lay.seg_offsets, False),  # sa length E*M
        lambda: ops.gemm_fp8_grouped_k(aq.t().contiguous(), sa[:128], aq.t().contiguous(), sa[:128],
                                       torch.zeros(2, 64, 64, device="cuda", dtype=torch.float16), lay.seg_offsets, False),
    ]
    for i, f in enumerate(bad):
        with pytest.raises((RuntimeError, ValueError)):
            f()
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ expert block
def _block_inputs(T=512, H=256, F=192, E=8, k=2, seed=0):
    from d9d_b200.kernel.moe import build_moe_layout, moe_permute

    torch.manual_seed(seed)
    x = torch.randn(T, H, device="cuda").bfloat16()
    ids = torch.stack([torch.randperm(E, device="cuda")[:k] for _ in range(T)])
    ids[ids == 5] = 6  # expert 5 gets no tokens
    probs = torch.rand(T, k, device="cuda")
    layout = build_moe_layout(ids, E)
    xp, pp = moe_permute(x, probs, layout)
    w = [(torch.randn(E, a, b, device="cuda") * 0.05).bfloat16() for a, b in ((H, F), (H, F), (F, H))]
    return xp.detach(), pp.detach(), w, layout


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cos(a, b):
    return float(torch.nn.functional.cosine_similarity(a.double().flatten(), b.double().flatten(), dim=0))


def test_fp8_block_against_emulation_and_bf16():
    from d9d_b200.kernel.moe import grouped_swiglu, grouped_swiglu_fp8_reference

    xp, pp, w, layout = _block_inputs()
    dy = torch.randn(xp.shape[0], w[2].shape[2], device="cuda").bfloat16()
    starts, counts = layout.seg_offsets[:-1].tolist(), layout.counts.tolist()
    valid = torch.zeros(xp.shape[0], dtype=torch.bool, device="cuda")
    for s0, n in zip(starts, counts):
        valid[s0 : s0 + n] = True

    def run(kind):
        leaves = [xp.clone().requires_grad_(), pp.clone().requires_grad_()] + [t.clone().requires_grad_() for t in w]
        if kind == "emu":
            y = grouped_swiglu_fp8_reference(*leaves, starts, counts)
        else:
            y = grouped_swiglu(*leaves, layout, fp8=(kind == "fp8"))
        (y[valid].float() * dy[valid].float()).sum().backward()
        return [y] + [t.grad for t in leaves]

    fp8_, emu, bf16 = run("fp8"), run("emu"), run("bf16")
    for name, a, b, c in zip(("y", "dx", "dprobs", "dwg", "dwu", "dwd"), fp8_, emu, bf16):
        if name in ("y", "dx", "dprobs"):
            a, b, c = a[valid], b[valid], c[valid]
        # the emulation rounds the same intermediates to bf16 but may round a handful of them the other way, which can move
        # an e4m3 operand by one step: a few per cent of one element, far less over a whole tensor
        assert _rel(a, b) < 2e-2, (name, _rel(a, b))
        assert _cos(a, c) >= 0.99, (name, _cos(a, c))


def test_fp8_block_buffers_split_backward_and_fused_wgrad():
    from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection
    from d9d_b200.kernel._native import FUSED_WGRAD_ATTR
    from d9d_b200.kernel.moe import grouped_swiglu

    xp, pp, w, layout = _block_inputs(seed=3)
    used = int(layout.seg_offsets[-1])
    cap, H = xp.shape
    out_buf = torch.zeros(cap + 256, H, device="cuda", dtype=torch.bfloat16)
    dx_buf = torch.zeros(cap + 256, H, device="cuda", dtype=torch.bfloat16)
    dy = torch.randn(cap, H, device="cuda").bfloat16()

    leaves = [xp.clone().requires_grad_(), pp.clone().requires_grad_()] + [t.clone().requires_grad_() for t in w]
    y = grouped_swiglu(leaves[0], leaves[1], *leaves[2:], layout, out_buf, dx_buf, fp8=True)
    assert y.data_ptr() == out_buf.data_ptr()
    y.backward(dy)
    assert torch.equal(leaves[0].grad[:used], dx_buf[:used])
    whole = [t.grad.clone() for t in leaves]

    leaves2 = [xp.clone().requires_grad_(), pp.clone().requires_grad_()] + [t.clone().requires_grad_() for t in w]
    y2 = grouped_swiglu(leaves2[0], leaves2[1], *leaves2[2:], layout, fp8=True)
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.inputs):
        dx, dp = torch.autograd.grad(y2, leaves2[:2], dy, retain_graph=True)
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.weight):
        dws = torch.autograd.grad(y2, leaves2[2:], dy, allow_unused=True)
    assert torch.equal(dx[:used], whole[0][:used]) and torch.equal(dp[:used], whole[1][:used])
    for a, b in zip(dws, whole[2:]):
        assert torch.equal(a.float(), b.float())

    # fused wgrad: two microbatches accumulate straight into pre-allocated fp32 gradients, as autograd accumulates the
    # fp32 gradients of the same parameters without the fused path
    fused, plain = [torch.nn.Parameter(t.clone()) for t in w], [torch.nn.Parameter(t.clone()) for t in w]
    for p in fused + plain:
        p.grad_dtype = torch.float32
    for p in fused:
        p.grad = torch.zeros(p.shape, device="cuda", dtype=torch.float32)
        setattr(p, FUSED_WGRAD_ATTR, True)
    for params in (fused, plain):
        for _ in range(2):
            grouped_swiglu(xp, pp, *params, layout, fp8=True).backward(dy)
    for a, b in zip(fused, plain):
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-6, atol=0)


def test_fp8_block_with_frozen_experts_quantises_no_weight_gradient_operands():
    from d9d_b200.kernel._native import native_ops
    from d9d_b200.kernel.moe import grouped_swiglu

    xp, pp, w, layout = _block_inputs(seed=5)
    ops = native_ops()
    calls = []
    real = ops.quantize_segments_t
    ops._cache["quantize_segments_t"] = lambda *a, **k: (calls.append(1), real(*a, **k))[1]
    try:
        x = xp.clone().requires_grad_()
        grouped_swiglu(x, pp, *w, layout, fp8=True).backward(torch.randn(xp.shape[0], w[2].shape[2], device="cuda").bfloat16())
        assert x.grad is not None and not calls  # frozen weights: no transposing quantiser runs
        w[0].requires_grad_()
        grouped_swiglu(x, pp, *w, layout, fp8=True).backward(torch.randn(xp.shape[0], w[2].shape[2], device="cuda").bfloat16())
        assert w[0].grad is not None and len(calls) == 2  # the gate gradient only: x and d(gate)
    finally:
        ops._cache["quantize_segments_t"] = real


def test_fp8_experts_model_trains_like_bf16():
    """A small Qwen3-MoE (hidden 256, 8 experts of 128) trained 50 steps from one seed with and without fp8 experts."""
    from d9d_b200.kernel._native import native_launch_count
    from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode
    from d9d_b200.module.block.moe import GroupedSwiGLU
    from d9d_b200.module.model.qwen3_moe import (
        Qwen3MoEForCausalLM, Qwen3MoEForCausalLMParameters, Qwen3MoELayerParameters, Qwen3MoEParameters)
    from d9d_b200.pipelining.api import PipelineStageInfo

    params = Qwen3MoEForCausalLMParameters(model=Qwen3MoEParameters(
        layer=Qwen3MoELayerParameters(hidden_size=256, intermediate_size=128, num_experts=8, experts_top_k=2, num_attention_heads=4,
                                      num_key_value_heads=2, rms_norm_eps=1e-6, head_dim=64),
        num_hidden_layers=2, rope_base=10000, max_position_ids=256, split_vocab_size={"regular": 512},
        split_vocab_order=["regular"]))

    def train(fp8_experts):
        torch.manual_seed(0)
        model = Qwen3MoEForCausalLM(params, PipelineStageInfo(0, 1), HiddenStatesAggregationMode.no, False)
        model.reset_parameters()
        model = model.bfloat16().cuda()
        model.model.rope_provider.reset_parameters()
        blocks = [m for m in model.modules() if isinstance(m, GroupedSwiGLU)]
        if fp8_experts:
            for b in blocks:
                b.enable_fp8()
        opt = torch.optim.AdamW(model.parameters(), lr=2e-3)
        gen = torch.Generator(device="cuda").manual_seed(1)
        losses = []
        for _ in range(50):
            ids = torch.randint(0, 512, (4, 128), device="cuda", generator=gen)
            ids[:, 1::2] = (ids[:, 0::2] * 7 + 3) % 512  # learnable: every second token follows from the one before
            labels = torch.roll(ids, -1, 1)
            out = model(input_ids=ids, position_ids=torch.arange(128, device="cuda")[None].expand(4, -1), labels=labels)
            loss = out["logps"].mean()
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(float(loss))
        return losses, blocks

    ref, _ = train(False)
    before = native_launch_count()
    got, blocks = train(True)
    assert native_launch_count() > before and all(b.fp8 for b in blocks)
    print("bf16 losses", [round(v, 4) for v in ref[::10]], "fp8 losses", [round(v, 4) for v in got[::10]])
    assert got[-1] < 0.7 * got[0]
    assert abs(got[-1] - ref[-1]) <= 0.05 * ref[0]  # within 5 % of the starting loss of the bf16 run

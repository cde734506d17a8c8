"""The blockwise fp8 recipe of the MoE expert block on the H100: the expert-weight and MoE-layout quantisers code by code and
scale by scale, the six grouped BLOCKWISE GEMM instances on exact operands against fp64, random operands within the
promoted-accumulation bound, and ``grouped_swiglu(fp8=True, recipe="blockwise")`` against its emulation and bf16."""

import pytest
import torch

from d9d_b200.kernel import fp8

from .fp8_reference import assert_codes_admissible, check_scales, flush, gemm_bound

pytestmark = pytest.mark.gpu

NAN_CODE = 0x7F


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _layout_from_counts(counts, device="cuda"):
    """A MoE layout ([E] counts -> 128-aligned segments, tile table) with two unused tiles (tile_group -1) at the end."""
    from d9d_b200.kernel.moe.layout import ALIGN, MoELayout

    E = len(counts)
    seg = [0]
    for c in counts:
        seg.append(seg[-1] + (c + ALIGN - 1) // ALIGN * ALIGN)
    cap = seg[-1] + 2 * ALIGN
    tiles = [-1] * (cap // ALIGN)
    for e in range(E):
        for t in range(seg[e] // ALIGN, seg[e + 1] // ALIGN):
            tiles[t] = e
    i32 = dict(dtype=torch.int32, device=device)
    return MoELayout(torch.tensor(counts, **i32), torch.tensor(seg, **i32), torch.empty(0, **i32), torch.tensor(tiles, **i32),
                     0, 1, E, cap)


def _used_rows(layout):
    return (layout.tile_group >= 0).repeat_interleave(128)


def _valid_rows(layout):
    valid = torch.zeros(layout.capacity, dtype=torch.bool, device="cuda")
    for s0, n in zip(layout.seg_offsets[:-1].tolist(), layout.counts.tolist()):
        valid[s0 : s0 + n] = True
    return valid


def _blocks_amax(w, rb, cb, flushed=True):
    """amax of every rb x cb block of the 2-D ``w`` in fp64 (elements below 2^-126 flushed), repeated to ``w``'s shape."""
    R, C = w.shape
    Rb, Cb = -(-R // rb), -(-C // cb)
    pad = torch.nn.functional.pad((flush(w) if flushed else w.double()).abs(), (0, Cb * cb - C, 0, Rb * rb - R))
    return pad.view(Rb, rb, Cb, cb).amax(dim=(1, 3)).repeat_interleave(rb, 0).repeat_interleave(cb, 1)[:R, :C]


# ------------------------------------------------------------------------------------------ quantisers
@pytest.mark.parametrize("E,n_in,n_out", [(1, 144, 272), (8, 768, 576), (3, 2048, 16)])
def test_expert_weight_blocks(ops, E, n_in, n_out):
    torch.manual_seed(0)
    # the full fp32 exponent range across the experts, an all-zero block
    w = (torch.randn(E, n_in, n_out, device="cuda") * torch.logspace(-120, 120, E, base=2, device="cuda")[:, None, None]).bfloat16()
    w[0, :16, :16] = 0
    w[0, :128, :128] = 0
    qt, st = ops.quantize_expert_weight_blocks(w, True)
    q, s = ops.quantize_expert_weight_blocks(w, False)
    assert qt.shape == (E, n_out, n_in) and st.shape == (E, -(-n_in // 128), n_out)
    assert q.shape == (E, n_in, n_out) and s.shape == (E, -(-n_out // 128), n_in)
    for e in range(E):
        assert torch.equal(qt[e].view(torch.uint8), q[e].t().view(torch.uint8)), e
        amax = _blocks_amax(w[e].float(), 128, 128)
        s_full = s[e].t().repeat_interleave(128, dim=1)[:, :n_out]
        st_full = st[e].repeat_interleave(128, dim=0)[:n_in]
        raw = _blocks_amax(w[e].float(), 128, 128, flushed=False)
        check_scales(s_full, amax, f"expert {e}", raw_amax=raw)
        assert torch.equal(s_full, st_full)
        assert_codes_admissible(w[e], q[e], s_full, f"expert {e}")
    assert (st[0, 0, :128] == 1).all()
    assert not s.as_strided((E, s.shape[1], s.stride(1)), s.stride())[..., n_in:].any()  # zero pitch padding


@pytest.mark.parametrize("counts,C", [([300, 0, 1, 129, 128], 96), ([16000], 272), ([0] * 60 + [5] * 68, 48)])
def test_layout_quantisers(ops, counts, C):
    torch.manual_seed(1)
    layout = _layout_from_counts(counts)
    cap = layout.capacity
    used, valid = _used_rows(layout), _valid_rows(layout)
    x = (torch.randn(cap, C, device="cuda") * torch.logspace(-120, 120, C, base=2, device="cuda")).bfloat16()
    x[:, 5] = 0
    x[~used] = float("nan")  # unused capacity: never initialised on the expert-parallel path
    xt_in = x.clone()
    xt_in[used & ~valid] = 1e30  # pad rows: the transposed groups end at the expert's last row
    q, s = ops.quantize_blockwise_tiles(x, layout.tile_group)
    qt, st = ops.quantize_blockwise_t_tiles(xt_in, layout.tile_group, layout.seg_offsets, layout.counts)
    assert q.shape == (cap, C) and s.shape == (-(-C // 128), cap)
    assert qt.shape == (C, cap) and st.shape == (cap // 128, C)
    # row groups: every row of a tile in use
    xu, qu, su = x[used], q[used], s[:, used]
    amax = _blocks_amax(xu.float(), 1, 128)
    s_full = su.t().repeat_interleave(128, dim=1)[:, :C]
    check_scales(s_full, amax, "row groups", raw_amax=_blocks_amax(xu.float(), 1, 128, flushed=False))
    assert_codes_admissible(xu, qu, s_full, "row groups")
    # token groups: the experts' rows, pad rows zero
    assert not qt[:, used & ~valid].float().any()
    xv = torch.where(valid[:, None], x.float(), torch.zeros((), device="cuda"))
    for g in (layout.tile_group >= 0).nonzero().flatten().tolist():
        rows = slice(128 * g, 128 * g + 128)
        check_scales(st[g], flush(xv[rows]).abs().amax(dim=0), f"token group {g}", raw_amax=xv[rows].abs().amax(dim=0))
        assert_codes_admissible(xv[rows].t(), qt[:, rows], st[g][:, None], f"token group {g}")


def test_layout_quantisers_are_reproducible(ops):
    layout = _layout_from_counts([300, 0, 129])
    x = torch.randn(layout.capacity, 64, device="cuda").bfloat16()
    a = ops.quantize_blockwise_t_tiles(x, layout.tile_group, layout.seg_offsets, layout.counts)
    b = ops.quantize_blockwise_t_tiles(x, layout.tile_group, layout.seg_offsets, layout.counts)
    used = _used_rows(layout)  # the skipped tiles' codes are never written
    assert torch.equal(a[0].view(torch.uint8)[:, used], b[0].view(torch.uint8)[:, used]) and torch.equal(a[1], b[1])


# ------------------------------------------------------------------------------------------ GEMMs on exact operands
def _codes(*shape, device="cuda"):
    return torch.randint(-1, 2, shape, device=device).float().to(fp8.FP8)


def _pow2(*shape):
    return torch.exp2(torch.randint(-2, 3, shape, device="cuda").float())


def _scales(*shape):
    """fp32 [..., groups, rows] view with the row pitch round_up(rows, 128), zero padding."""
    *lead, rows = shape
    pitch = -(-rows // 128) * 128
    return torch.zeros(*lead, pitch, device="cuda")[..., :rows]


def _grouped_m_ref(a, sa, b, sb, layout, N):
    """fp64 D[rows of e] = sum_kb (a[rows, kb] b[e, :, kb]^T) sa[kb, rows] sb[e, kb, :]"""
    K = a.shape[1]
    d = torch.zeros(a.shape[0], N, dtype=torch.float64, device="cuda")
    tiles = layout.tile_group.tolist()
    for e in set(t for t in tiles if t >= 0):
        rows = torch.tensor([r for r in range(a.shape[0]) if tiles[r // 128] == e], device="cuda")
        for kb in range(-(-K // 128)):
            ks = slice(128 * kb, min(K, 128 * kb + 128))
            part = a[rows][:, ks].double() @ b[e][:, ks].double().t()
            d[rows] += part * sa[kb, rows].double()[:, None] * sb[e, kb].double()[None, :]
    return d


@pytest.mark.parametrize("counts,K,N", [([300, 0, 1, 129], 576, 576), ([0, 2000, 0], 7168, 256), ([5] * 16, 256, 768)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_grouped_m_exact(ops, counts, K, N, accumulate):
    torch.manual_seed(2)
    layout = _layout_from_counts(counts)
    E, cap, kb = len(counts), layout.capacity, -(-K // 128)
    used = _used_rows(layout)
    a, b = _codes(cap, K), _codes(E, N, K)
    sa, sb = _scales(kb, cap), _scales(E, kb, N)
    sa.copy_(_pow2(kb, cap))
    sb.copy_(_pow2(E, kb, N))
    a.view(torch.uint8)[~used] = NAN_CODE  # unused tiles: never read
    sa[:, ~used] = float("nan")
    ref = _grouped_m_ref(a, sa, b, sb, layout, N)
    canary = torch.full((cap, N), 1234.0, device="cuda").bfloat16()
    prior = (torch.randint(-8, 9, (cap, N), device="cuda").float() / 4).bfloat16()
    prior[~used] = canary[~used]
    d = (prior if accumulate else canary).clone()
    ops.gemm_fp8_blockwise_grouped_m(a, sa, b, sb, d, layout.tile_group, accumulate)
    assert torch.equal(d[~used], canary[~used])  # unused tiles unwritten
    if accumulate:
        want = prior[used].double() + ref[used]
        # acc -> bf16 and the bf16 add: two roundings
        assert bool(((d[used].double() - want).abs() <= 2.0**-7 * (prior[used].double().abs() + ref[used].abs())).all())
    else:
        assert torch.equal(d[used], ref[used].to(torch.bfloat16))
    d2 = (prior if accumulate else canary).clone()
    ops.gemm_fp8_blockwise_grouped_m(a, sa, b, sb, d2, layout.tile_group, accumulate)
    assert torch.equal(d, d2)  # bitwise reproducible


def _grouped_k_ref(a, sa, b, sb, seg):
    E = len(seg) - 1
    d = torch.zeros(E, a.shape[0], b.shape[0], dtype=torch.float64, device="cuda")
    for e in range(E):
        for g in range(seg[e] // 128, seg[e + 1] // 128):
            ks = slice(128 * g, 128 * g + 128)
            d[e] += (a[:, ks].double() @ b[:, ks].double().t()) * sa[g].double()[:, None] * sb[g].double()[None, :]
    return d


@pytest.mark.parametrize("counts,M,N", [([300, 0, 1, 129, 128], 576, 768), ([16000], 128, 192), ([0] * 60 + [5] * 68, 256, 64)])
@pytest.mark.parametrize("dtype,accumulate", [(torch.float32, False), (torch.float32, True), (torch.bfloat16, False),
                                              (torch.bfloat16, True)])
def test_grouped_k_exact(ops, counts, M, N, dtype, accumulate):
    torch.manual_seed(3)
    layout = _layout_from_counts(counts)
    E, cap = len(counts), layout.capacity
    seg = layout.seg_offsets.tolist()
    used = _used_rows(layout)
    a, b = _codes(M, cap), _codes(N, cap)
    sa, sb = _scales(cap // 128, M), _scales(cap // 128, N)
    sa.copy_(_pow2(cap // 128, M))
    sb.copy_(_pow2(cap // 128, N))
    a.view(torch.uint8)[:, ~used] = NAN_CODE  # unused capacity: never read
    b.view(torch.uint8)[:, ~used] = NAN_CODE
    sa[(~used).view(-1, 128)[:, 0]] = float("nan")
    ref = _grouped_k_ref(a, sa, b, sb, seg)
    prior = (torch.randint(-8, 9, (E, M, N), device="cuda").float() / 4).to(dtype)
    d = prior.clone() if accumulate else torch.full((E, M, N), 1234.0, device="cuda", dtype=dtype)
    ops.gemm_fp8_blockwise_grouped_k(a, sa, b, sb, d, layout.seg_offsets, accumulate)
    empty = torch.tensor(counts, device="cuda") == 0
    if accumulate:
        assert torch.equal(d[empty], prior[empty])  # an expert without rows adds nothing
        want = prior.double() + ref
        tol = (2.0**-7 if dtype == torch.bfloat16 else 2.0**-23) * (prior.double().abs() + ref.abs())
        assert bool(((d.double() - want).abs() <= tol).all())
    else:
        assert not d[empty].any()  # ... and stores zeros
        assert torch.equal(d, ref.to(dtype))
    d2 = prior.clone() if accumulate else torch.zeros_like(d)
    ops.gemm_fp8_blockwise_grouped_k(a, sa, b, sb, d2, layout.seg_offsets, accumulate)
    assert torch.equal(d, d2)


# ------------------------------------------------------------------------------------------ random operands
def test_grouped_m_random_within_promoted_bound(ops):
    torch.manual_seed(4)
    layout = _layout_from_counts([300, 0, 1, 900])
    K, N = 7168, 576
    x = torch.randn(layout.capacity, K, device="cuda").bfloat16()
    w = (torch.randn(4, K, N, device="cuda") * 0.02).bfloat16()
    a, sa = ops.quantize_blockwise_tiles(x, layout.tile_group)
    b, sb = ops.quantize_expert_weight_blocks(w, True)
    d = torch.empty(layout.capacity, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm_fp8_blockwise_grouped_m(a, sa, b, sb, d, layout.tile_group)
    deq_a = a.double() * sa.double().t().repeat_interleave(128, dim=1)
    deq_b = b.double() * sb.double().transpose(1, 2).repeat_interleave(128, dim=2)[..., :K]
    used = _used_rows(layout)
    tiles = layout.tile_group.repeat_interleave(128)
    worst = 0.0
    for e in range(4):
        rows = (tiles == e).nonzero().flatten()
        if rows.numel() == 0:
            continue
        ref = deq_a[rows] @ deq_b[e].t()
        S = deq_a[rows].abs() @ deq_b[e].abs().t()
        bound = gemm_bound(ref, S, K, 128, torch.bfloat16)
        err = (d[rows].double() - ref).abs()
        assert bool((err <= bound).all()), e
        worst = max(worst, float((err / bound).max()))
    assert used.any()
    print(f"grouped_m K=7168: worst err / bound = {worst:.3f}")


def test_wgrad_over_16k_tokens_is_promoted(ops):
    """A 16 384-token fp32 expert weight gradient: the relative error against fp64 of the dequantised operands, next to the
    promoted-accumulation bound and the error one unpromoted chain would allow."""
    torch.manual_seed(5)
    layout = _layout_from_counts([16384])
    M, N = 576, 768
    x = torch.randn(layout.capacity, M, device="cuda").bfloat16()
    dy = torch.randn(layout.capacity, N, device="cuda").bfloat16()
    a, sa = ops.quantize_blockwise_t_tiles(x, layout.tile_group, layout.seg_offsets, layout.counts)
    b, sb = ops.quantize_blockwise_t_tiles(dy, layout.tile_group, layout.seg_offsets, layout.counts)
    d = torch.empty(1, M, N, device="cuda")
    ops.gemm_fp8_blockwise_grouped_k(a, sa, b, sb, d, layout.seg_offsets, False)
    K = int(layout.seg_offsets[-1])  # the unused tiles' codes and scales are never written or read
    deq_a = (a.double() * sa.double().t().repeat_interleave(128, dim=1))[:, :K]
    deq_b = (b.double() * sb.double().t().repeat_interleave(128, dim=1))[:, :K]
    ref = deq_a @ deq_b.t()
    S = deq_a.abs() @ deq_b.abs().t()
    bound = gemm_bound(ref, S, K, 128, torch.float32)
    err = (d[0].double() - ref).abs()
    assert bool((err <= bound).all())
    rel = float(err.norm() / ref.norm())
    rel_bound = float(bound.norm() / ref.norm())
    rel_chain = float(gemm_bound(ref, S, K, K, torch.float32).norm() / ref.norm())
    print(f"16384-token wgrad: relative error {rel:.2e}, promoted bound {rel_bound:.2e}, one chain {rel_chain:.2e}")
    assert rel <= rel_bound


def test_blockwise_grouped_ops_refuse_bad_operands(ops):
    layout = _layout_from_counts([130])
    cap, K, N = layout.capacity, 256, 128
    a, b = _codes(cap, K), _codes(1, N, K)
    sa, sb = _scales(2, cap), _scales(1, 2, N)
    d = torch.empty(cap, N, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="float8_e4m3fn"):
        ops.gemm_fp8_blockwise_grouped_m(a.view(torch.uint8), sa, b, sb, d, layout.tile_group)
    with pytest.raises(RuntimeError, match="sa has the wrong shape"):
        ops.gemm_fp8_blockwise_grouped_m(a, sa[:1], b, sb, d, layout.tile_group)
    with pytest.raises(RuntimeError, match="row pitch"):
        ops.gemm_fp8_blockwise_grouped_m(a, sa, b, torch.zeros(1, 2, 256, device="cuda")[..., :N], d, layout.tile_group)
    with pytest.raises(RuntimeError, match="tile_group"):
        ops.gemm_fp8_blockwise_grouped_m(a, sa, b, sb, d, layout.tile_group[:-1])
    with pytest.raises(RuntimeError, match="bf16"):
        ops.gemm_fp8_blockwise_grouped_m(a, sa, b, sb, d.float(), layout.tile_group)
    at, bt = _codes(64, cap), _codes(N, cap)
    dk = torch.empty(1, 64, N, device="cuda")
    gs = _scales(cap // 128, 64)
    with pytest.raises(RuntimeError, match="sb has the wrong shape"):
        ops.gemm_fp8_blockwise_grouped_k(at, gs, bt, gs, dk, layout.seg_offsets, False)
    with pytest.raises(RuntimeError, match="group_offsets"):
        ops.gemm_fp8_blockwise_grouped_k(at, gs, bt, _scales(cap // 128, N), dk, layout.seg_offsets[:1], False)
    with pytest.raises(RuntimeError, match="multiple of 128"):
        ops.quantize_blockwise_tiles(torch.zeros(100, 16, device="cuda").bfloat16(), layout.tile_group)
    with pytest.raises(RuntimeError, match="int32"):
        ops.quantize_blockwise_t_tiles(torch.zeros(cap, 16, device="cuda").bfloat16(), layout.tile_group.long(), layout.seg_offsets,
                                       layout.counts)
    with pytest.raises(RuntimeError, match="multiples of 16"):
        ops.quantize_expert_weight_blocks(torch.zeros(2, 24, 16, device="cuda").bfloat16(), True)
    with pytest.raises(RuntimeError, match="bf16"):
        ops.quantize_expert_weight_blocks(torch.zeros(2, 32, 16, device="cuda"), True)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ expert block
def _block_inputs(T, H, F, E, k, seed=0, empty=None):
    from d9d_b200.kernel.moe import build_moe_layout, moe_permute

    torch.manual_seed(seed)
    x = torch.randn(T, H, device="cuda").bfloat16()
    ids = torch.rand(T, E, device="cuda").topk(k, dim=1).indices
    if empty is not None:
        ids[ids == empty] = (empty + 1) % E  # this expert gets no tokens
    probs = torch.rand(T, k, device="cuda")
    layout = build_moe_layout(ids, E)
    xp, pp = moe_permute(x, probs, layout)
    w = [(torch.randn(E, a, b, device="cuda") * 0.02).bfloat16() for a, b in ((H, F), (H, F), (F, H))]
    return xp.detach(), pp.detach(), w, layout


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cos(a, b):
    return float(torch.nn.functional.cosine_similarity(a.double().flatten(), b.double().flatten(), dim=0))


@pytest.mark.parametrize("T,H,F,E,k", [(2048, 768, 576, 128, 8), (512, 7168, 2048, 32, 8)], ids=["flagship", "deepseek_v3"])
def test_blockwise_block_against_emulation_and_bf16(T, H, F, E, k):
    from d9d_b200.kernel.moe import grouped_swiglu, grouped_swiglu_fp8_reference

    xp, pp, w, layout = _block_inputs(T, H, F, E, k, empty=5)
    dy = torch.randn(xp.shape[0], H, device="cuda").bfloat16()
    starts, counts = layout.seg_offsets[:-1].tolist(), layout.counts.tolist()
    valid = _valid_rows(layout)

    def run(kind):
        leaves = [xp.clone().requires_grad_(), pp.clone().requires_grad_()] + [t.clone().requires_grad_() for t in w]
        if kind == "emu":
            y = grouped_swiglu_fp8_reference(*leaves, starts, counts, "blockwise")
        else:
            y = grouped_swiglu(*leaves, layout, fp8=(kind == "fp8"), recipe="blockwise")
        (y[valid].float() * dy[valid].float()).sum().backward()
        return [t.detach() for t in [y] + [t.grad for t in leaves]]

    got = run("fp8")
    emu = run("emu")
    bf16 = run("bf16")
    for name, a, b, c in zip(("y", "dx", "dprobs", "dwg", "dwu", "dwd"), got, emu, bf16):
        if name in ("y", "dx", "dprobs"):
            a, b, c = a[valid], b[valid], c[valid]
        print(f"{name}: rel to emulation {_rel(a, b):.2e}, cosine to bf16 {_cos(a, c):.5f}")
        assert _rel(a, b) < 2e-2, (name, _rel(a, b))
        assert _cos(a, c) >= 0.99, (name, _cos(a, c))
    assert not got[3][5].any() and not got[5][5].any()  # the empty expert's gradients: zeros


def test_blockwise_block_buffers_split_backward_and_fused_wgrad():
    from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection
    from d9d_b200.kernel._native import FUSED_WGRAD_ATTR
    from d9d_b200.kernel.moe import grouped_swiglu

    xp, pp, w, layout = _block_inputs(512, 256, 192, 8, 2, seed=3, empty=5)
    used = int(layout.seg_offsets[-1])
    cap, H = xp.shape
    out_buf = torch.zeros(cap + 256, H, device="cuda", dtype=torch.bfloat16)
    dx_buf = torch.zeros(cap + 256, H, device="cuda", dtype=torch.bfloat16)
    dy = torch.randn(cap, H, device="cuda").bfloat16()
    kw = dict(fp8=True, recipe="blockwise")

    leaves = [xp.clone().requires_grad_(), pp.clone().requires_grad_()] + [t.clone().requires_grad_() for t in w]
    y = grouped_swiglu(leaves[0], leaves[1], *leaves[2:], layout, out_buf, dx_buf, **kw)
    assert y.data_ptr() == out_buf.data_ptr()
    y.backward(dy)
    assert torch.equal(leaves[0].grad[:used], dx_buf[:used])
    whole = [t.grad.clone() for t in leaves]

    leaves2 = [xp.clone().requires_grad_(), pp.clone().requires_grad_()] + [t.clone().requires_grad_() for t in w]
    y2 = grouped_swiglu(leaves2[0], leaves2[1], *leaves2[2:], layout, **kw)
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.inputs):
        dx, dp = torch.autograd.grad(y2, leaves2[:2], dy, retain_graph=True)
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.weight):
        dws = torch.autograd.grad(y2, leaves2[2:], dy, allow_unused=True)
    assert torch.equal(dx[:used], whole[0][:used]) and torch.equal(dp[:used], whole[1][:used])
    for a, b in zip(dws, whole[2:]):
        assert torch.equal(a.float(), b.float())

    fused, plain = [torch.nn.Parameter(t.clone()) for t in w], [torch.nn.Parameter(t.clone()) for t in w]
    for p in fused + plain:
        p.grad_dtype = torch.float32
    for p in fused:
        p.grad = torch.zeros(p.shape, device="cuda", dtype=torch.float32)
        setattr(p, FUSED_WGRAD_ATTR, True)
    for params in (fused, plain):
        for _ in range(2):
            grouped_swiglu(xp, pp, *params, layout, **kw).backward(dy)
    for a, b in zip(fused, plain):
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-6, atol=0)


def test_blockwise_block_with_frozen_experts_quantises_no_weight_gradient_operands():
    from d9d_b200.kernel._native import native_ops
    from d9d_b200.kernel.moe import grouped_swiglu

    xp, pp, w, layout = _block_inputs(512, 256, 192, 8, 2, seed=5)
    ops = native_ops()
    calls = []
    real = ops.quantize_blockwise_t_tiles
    ops._cache["quantize_blockwise_t_tiles"] = lambda *a, **k: (calls.append(1), real(*a, **k))[1]
    try:
        x = xp.clone().requires_grad_()
        dy = torch.randn(xp.shape[0], w[2].shape[2], device="cuda").bfloat16()
        grouped_swiglu(x, pp, *w, layout, fp8=True, recipe="blockwise").backward(dy)
        assert x.grad is not None and not calls
        w[0].requires_grad_()
        grouped_swiglu(x, pp, *w, layout, fp8=True, recipe="blockwise").backward(dy)
        assert w[0].grad is not None and len(calls) == 2  # the gate gradient only: x and d(gate)
    finally:
        ops._cache["quantize_blockwise_t_tiles"] = real


def test_blockwise_experts_model_trains_like_bf16():
    """A small Qwen3-MoE (hidden 256, 8 experts of 128) trained 50 steps from one seed with bf16 and blockwise fp8 experts."""
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

    def train(recipe):
        torch.manual_seed(0)
        model = Qwen3MoEForCausalLM(params, PipelineStageInfo(0, 1), HiddenStatesAggregationMode.no, False)
        model.reset_parameters()
        model = model.bfloat16().cuda()
        model.model.rope_provider.reset_parameters()
        blocks = [m for m in model.modules() if isinstance(m, GroupedSwiGLU)]
        if recipe is not None:
            for b in blocks:
                b.enable_fp8(recipe)
        opt = torch.optim.AdamW(model.parameters(), lr=2e-3)
        gen = torch.Generator(device="cuda").manual_seed(1)
        losses = []
        for _ in range(50):
            ids = torch.randint(0, 512, (4, 128), device="cuda", generator=gen)
            ids[:, 1::2] = (ids[:, 0::2] * 7 + 3) % 512
            labels = torch.roll(ids, -1, 1)
            out = model(input_ids=ids, position_ids=torch.arange(128, device="cuda")[None].expand(4, -1), labels=labels)
            loss = out["logps"].mean()
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(float(loss))
        return losses, blocks

    ref, _ = train(None)
    got, blocks = train("blockwise")
    assert all(b.fp8 and b.fp8_recipe == "blockwise" for b in blocks)
    print("bf16 losses", [round(v, 4) for v in ref[::10]], "blockwise fp8 losses", [round(v, 4) for v in got[::10]])
    assert got[-1] < 0.7 * got[0]
    assert abs(got[-1] - ref[-1]) <= 0.05 * ref[0]

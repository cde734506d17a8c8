"""Numerics of every native sm_90a kernel against a plain PyTorch fp32 reference of the same op."""

import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


# ----------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize(
    "M,N,K",
    [(128, 256, 64), (256, 512, 128), (1000, 776, 520), (4096, 2048, 768), (333, 129 * 8, 72), (8192, 576, 768)],
)
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_gemm_nt(ops, M, N, K, out_dtype):
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    d = torch.empty(M, N, device="cuda", dtype=out_dtype)
    ops.gemm(a, b, d, False, False, False)
    ref = a.float() @ b.float().t()
    assert _rel_err(d, ref) < (1e-2 if out_dtype == torch.bfloat16 else 1e-4)


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (1000, 776, 520), (4096, 768, 2048)])
def test_gemm_dgrad_layout(ops, M, N, K):
    # d[M,N] = a[M,K] @ b[K,N]   (b is MN-major: N contiguous)
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
    ops.gemm(a, b, d, False, True, False)
    assert _rel_err(d, a.float() @ b.float()) < 1e-2


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (776, 520, 1000), (768, 2048, 4096)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_gemm_wgrad_layout(ops, M, N, K, accumulate):
    # d[M,N] (+)= a[K,M]^T @ b[K,N]   (both MN-major)
    a = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    d0 = torch.randn(M, N, device="cuda", dtype=torch.float32)
    d = d0.clone()
    ops.gemm(a, b, d, True, True, accumulate)
    ref = a.float().t() @ b.float() + (d0 if accumulate else 0)
    assert _rel_err(d, ref) < 1e-4


def test_gemm_mn_a_k_b(ops):
    M, N, K = 384, 320, 192
    a = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    d = torch.empty(M, N, device="cuda", dtype=torch.float32)
    ops.gemm(a, b, d, True, False, False)
    assert _rel_err(d, a.float().t() @ b.float().t()) < 1e-4


def test_gemm_bf16_accumulate(ops):
    M, N, K = 512, 384, 256
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    d0 = torch.randn(M, N, device="cuda", dtype=torch.bfloat16)
    d = d0.clone()
    ops.gemm(a, b, d, False, False, True)
    assert _rel_err(d, a.float() @ b.float().t() + d0.float()) < 1e-2


def _make_groups(counts, align=128):
    offs = [0]
    for c in counts:
        offs.append(offs[-1] + (c + align - 1) // align * align)
    return offs


@pytest.mark.parametrize("b_mn", [False, True])
def test_gemm_grouped_m(ops, b_mn):
    E, K, N = 5, 192, 320
    counts = [130, 0, 77, 256, 1]
    offs = _make_groups(counts)
    cap = offs[-1] + 256  # trailing unused tiles
    a = torch.zeros(cap, K, device="cuda", dtype=torch.bfloat16)
    tile_group = torch.full((cap // 128,), -1, dtype=torch.int32)
    for e, c in enumerate(counts):
        a[offs[e] : offs[e] + c] = torch.randn(c, K, device="cuda", dtype=torch.bfloat16)
        tile_group[offs[e] // 128 : offs[e + 1] // 128] = e
    tile_group = tile_group.cuda()
    w = torch.randn(E, K, N, device="cuda", dtype=torch.bfloat16) if b_mn else torch.randn(E, N, K, device="cuda", dtype=torch.bfloat16)
    d = torch.full((cap, N), 7.0, device="cuda", dtype=torch.bfloat16)
    ops.gemm_grouped_m(a, w, d, tile_group, b_mn)
    for e, c in enumerate(counts):
        we = w[e].float() if b_mn else w[e].float().t()
        ref = a[offs[e] : offs[e + 1]].float() @ we
        assert _rel_err(d[offs[e] : offs[e + 1]], ref) < 1e-2 or ref.numel() == 0
    assert (d[offs[-1] :] == 7.0).all()  # unused tiles untouched


@pytest.mark.parametrize("accumulate", [False, True])
def test_gemm_grouped_k(ops, accumulate):
    E, Md, Nd = 4, 192, 136
    counts = [130, 0, 77, 256]
    offs = _make_groups(counts)
    R = offs[-1]
    x = torch.zeros(R, Md, device="cuda", dtype=torch.bfloat16)
    dy = torch.zeros(R, Nd, device="cuda", dtype=torch.bfloat16)
    for e, c in enumerate(counts):
        x[offs[e] : offs[e] + c] = torch.randn(c, Md, device="cuda", dtype=torch.bfloat16)
        dy[offs[e] : offs[e] + c] = torch.randn(c, Nd, device="cuda", dtype=torch.bfloat16)
    go = torch.tensor(offs, dtype=torch.int32, device="cuda")
    d0 = torch.randn(E, Md, Nd, device="cuda", dtype=torch.float32)
    d = d0.clone()
    ops.gemm_grouped_k(x, dy, d, go, accumulate)
    for e in range(E):
        ref = x[offs[e] : offs[e + 1]].float().t() @ dy[offs[e] : offs[e + 1]].float() + (d0[e] if accumulate else 0)
        assert (d[e] - ref).abs().max().item() < 1e-2 * max(1.0, ref.abs().max().item())


# ----------------------------------------------------------------------------- fused linear CE
@pytest.mark.parametrize("T,V,K", [(256, 1000, 128), (1000, 5003 * 8 // 8 * 8, 256), (2048, 32000, 768)])
def test_linear_ce(ops, T, V, K):
    h = (torch.randn(T, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(V, K, device="cuda") * 0.1).bfloat16()
    tgt = torch.randint(0, V, (T,), device="cuda")
    tgt[::7] = -100
    nll, lse = ops.ce_forward(h, w, tgt, -100)
    logits = h.float() @ w.float().t()
    ref = torch.nn.functional.cross_entropy(logits, tgt, ignore_index=-100, reduction="none")
    assert torch.allclose(nll, ref, atol=2e-3, rtol=2e-3)
    assert torch.allclose(lse, torch.logsumexp(logits, -1), atol=2e-3, rtol=2e-3)
    g = torch.rand(T, device="cuda")
    out = torch.empty(T, V, device="cuda", dtype=torch.bfloat16)
    ops.ce_dlogits(h, w, tgt, lse, g, out, -100)
    p = torch.softmax(logits, -1)
    onehot = torch.zeros_like(p)
    valid = tgt != -100
    onehot[valid, tgt[valid]] = 1
    refg = (p - onehot) * (g * valid)[:, None]
    assert _rel_err(out, refg) < 2e-2


@pytest.mark.parametrize("softcap,with_bias", [(0.0, False), (8.0, False), (0.0, True), (8.0, True)])
def test_linear_ce_slice_options(ops, softcap, with_bias):
    """Bias / tanh soft-capping / class-id offset of a classifier slice inside the CE epilogues."""
    T, V, K, v0, v1 = 384, 1500, 128, 520, 1300
    h = (torch.randn(T, K, device="cuda") * 0.5).bfloat16()
    w = (torch.randn(V, K, device="cuda") * 0.2).bfloat16()
    bias = torch.randn(V, device="cuda") * 0.5 if with_bias else None
    tgt = torch.randint(0, V, (T,), device="cuda")
    tgt[::7] = -100
    z = h.float() @ w.float().t()
    if with_bias:
        z = z + bias
    dz = torch.ones_like(z)
    if softcap > 0:
        th = torch.tanh(z / softcap)
        z, dz = softcap * th, 1 - th * th
    zs = z[:, v0:v1]
    b = bias[v0:v1].contiguous() if with_bias else None
    nll, lse, tl = ops.ce_forward_ex(h, w[v0:v1], tgt, -100, b, softcap, v0)
    inside = (tgt >= v0) & (tgt < v1)
    ref_lse = torch.logsumexp(zs, -1)
    ref_tl = torch.where(inside, z.gather(1, tgt.clamp(0, V - 1)[:, None])[:, 0], torch.zeros_like(ref_lse))
    assert torch.allclose(lse, ref_lse, atol=3e-3, rtol=3e-3)
    assert torch.allclose(tl, ref_tl, atol=3e-3, rtol=3e-3)
    assert torch.allclose(nll, torch.where(tgt == -100, torch.zeros_like(lse), ref_lse - ref_tl), atol=5e-3, rtol=5e-3)
    full_lse = torch.logsumexp(z, -1)
    g = torch.rand(T, device="cuda")
    out = torch.empty(T, (v1 - v0 + 127) // 128 * 128, device="cuda", dtype=torch.bfloat16)[:, : v1 - v0]
    ops.ce_dlogits(h, w[v0:v1], tgt, full_lse, g, out, -100, b, softcap, v0)
    p = torch.exp(zs - full_lse[:, None])
    rows = torch.nonzero(inside)[:, 0]
    p[rows, tgt[rows] - v0] -= 1
    ref = p * (g * (tgt != -100))[:, None] * dz[:, v0:v1]
    assert _rel_err(out, ref) < 2e-2


@pytest.mark.parametrize("sizes", [(4000,), (3000, 24), (1000, 520, 8)])
@pytest.mark.parametrize("budget", [1 << 30, 512 * 1024 * 2])
@pytest.mark.parametrize("fused_wgrad", [False, True])
def test_linear_cross_entropy_split_blocks_autograd(monkeypatch, sizes, budget, fused_wgrad):
    """The public function over split classifier blocks with the vocabulary-chunked backward vs fp32 autograd."""
    from d9d_b200.kernel import _native
    from d9d_b200.kernel.cce import main as cce

    monkeypatch.setattr(cce, "_CHUNK_BYTES", budget)
    T, K = 512, 256
    e = (torch.randn(T, K, device="cuda") * 0.5).bfloat16().requires_grad_()
    ws = [(torch.randn(s, K, device="cuda") * 0.1).bfloat16().requires_grad_() for s in sizes]
    tgt = torch.randint(0, sum(sizes), (T,), device="cuda")
    tgt[::9] = -100
    tgt[3] = sum(sizes) - 1
    if fused_wgrad:
        for w in ws:
            w.grad_dtype = torch.float32
            w.grad = torch.full(w.shape, 0.5, device="cuda", dtype=torch.float32)
            setattr(w, _native.FUSED_WGRAD_ATTR, True)
    loss = cce.linear_cross_entropy(e, ws, tgt, reduction="sum")
    loss.backward()
    e2 = e.detach().float().requires_grad_()
    w2 = [w.detach().float().requires_grad_() for w in ws]
    nll, _ = cce.linear_cross_entropy_reference(e2, torch.cat(w2), tgt)
    nll.sum().backward()
    assert abs(loss.item() - nll.sum().item()) < 2e-3 * abs(nll.sum().item())
    assert _rel_err(e.grad, e2.grad) < 2e-2
    for w, r in zip(ws, w2):
        assert _rel_err(w.grad.float() - (0.5 if fused_wgrad else 0.0), r.grad) < 2e-2


def test_gemm_dgrad_layout_fp32_accumulate(ops):
    # d[M,N] (fp32) += a[M,K] @ b[K,N]: the accumulate epilogue of the chunked linear-CE input gradient
    M, N, K = 1024, 768, 2048
    a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    d0 = torch.randn(M, N, device="cuda", dtype=torch.float32)
    d = d0.clone()
    ops.gemm(a, b, d, False, True, True)
    assert _rel_err(d, a.float() @ b.float() + d0) < 1e-4


# ----------------------------------------------------------------------------- RMSNorm
@pytest.mark.parametrize("N", [64, 128, 256, 768, 1024, 2048, 4096, 7168])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("zc", [False, True])
def test_rms_norm(ops, N, dtype, zc):
    M = 517
    x = torch.randn(M, N, device="cuda", dtype=dtype)
    w = (torch.randn(N, device="cuda") * 0.1 + (0 if zc else 1)).to(dtype)
    out, inv = ops.rms_norm_fwd(x, w, 1e-6, zc)
    xf, wf = x.float(), w.float() + (1 if zc else 0)
    inv_ref = torch.rsqrt(xf.pow(2).mean(-1) + 1e-6)
    ref = xf * inv_ref[:, None] * wf
    tol = 2e-2 if dtype == torch.bfloat16 else 1e-5
    assert torch.allclose(out.float(), ref, atol=tol, rtol=tol)
    assert torch.allclose(inv, inv_ref, atol=1e-5, rtol=1e-5)
    dout = torch.randn_like(x)
    dx, dw = ops.rms_norm_bwd(dout, x, w, inv, zc)
    xr = xf.clone().requires_grad_(True)
    wr = w.float().clone().requires_grad_(True)
    y = xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-6) * (wr + (1 if zc else 0))
    y.backward(dout.float())
    assert _rel_err(dx, xr.grad) < (1e-2 if dtype == torch.bfloat16 else 1e-5)
    assert _rel_err(dw, wr.grad) < (1e-2 if dtype == torch.bfloat16 else 1e-4)


# ----------------------------------------------------------------------------- SiLU * mul
@pytest.mark.parametrize("n", [8, 1000, 12345, 1 << 20])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_silu_mul(ops, n, dtype):
    x = torch.randn(n, device="cuda", dtype=dtype)
    y = torch.randn(n, device="cuda", dtype=dtype)
    out = ops.silu_mul_fwd(x, y)
    ref = torch.nn.functional.silu(x.float()) * y.float()
    assert torch.allclose(out.float(), ref, atol=3e-2 if dtype == torch.bfloat16 else 1e-5, rtol=2e-2)
    g = torch.randn(n, device="cuda", dtype=dtype)
    dx, dy = ops.silu_mul_bwd(g, x, y)
    xr, yr = x.float().requires_grad_(True), y.float().requires_grad_(True)
    (torch.nn.functional.silu(xr) * yr).backward(g.float())
    tol = 1e-2 if dtype == torch.bfloat16 else 1e-5
    assert _rel_err(dx, xr.grad) < tol and _rel_err(dy, yr.grad) < tol


def test_silu_mul_probs(ops):
    R, C = 777, 576
    x = torch.randn(R, C, device="cuda", dtype=torch.bfloat16)
    y = torch.randn(R, C, device="cuda", dtype=torch.bfloat16)
    p = torch.rand(R, device="cuda")
    out = ops.silu_mul_probs_fwd(x, y, p)
    xr, yr, pr = x.float().requires_grad_(True), y.float().requires_grad_(True), p.clone().requires_grad_(True)
    ref = torch.nn.functional.silu(xr) * yr * pr[:, None]
    assert _rel_err(out, ref) < 1e-2
    g = torch.randn(R, C, device="cuda", dtype=torch.bfloat16)
    dx, dy, dp = ops.silu_mul_probs_bwd(g, x, y, p)
    ref.backward(g.float())
    assert _rel_err(dx, xr.grad) < 1e-2 and _rel_err(dy, yr.grad) < 1e-2 and _rel_err(dp, pr.grad) < 1e-3


# ----------------------------------------------------------------------------- RoPE
@pytest.mark.parametrize("D,rope_dim", [(128, 128), (64, 64), (128, 64), (256, 256)])
@pytest.mark.parametrize("style", [0, 1])
def test_rope(ops, D, rope_dim, style):
    T, H, maxpos = 300, 5, 512
    x = torch.randn(T, H, D, device="cuda", dtype=torch.bfloat16)
    inv_freq = 1.0 / (10000 ** (torch.arange(0, rope_dim, 2, device="cuda").float() / rope_dim))
    ang = torch.arange(maxpos, device="cuda").float()[:, None] * inv_freq[None]
    if style == 0:
        cos, sin = torch.cat([ang.cos(), ang.cos()], -1), torch.cat([ang.sin(), ang.sin()], -1)
    else:
        cos, sin = ang.cos().repeat_interleave(2, -1), ang.sin().repeat_interleave(2, -1)
    pos = torch.randint(0, maxpos, (T,), device="cuda")
    out = ops.rope_apply(x, cos.contiguous(), sin.contiguous(), pos, style, False)
    xf = x.float()
    xr, xpass = xf[..., :rope_dim], xf[..., rope_dim:]
    c, s = cos[pos][:, None, :], sin[pos][:, None, :]
    if style == 0:
        rot = torch.cat([-xr[..., rope_dim // 2 :], xr[..., : rope_dim // 2]], -1)
    else:
        rot = torch.stack([-xr[..., 1::2], xr[..., 0::2]], -1).flatten(-2)
    ref = torch.cat([xr * c + rot * s, xpass], -1)
    assert torch.allclose(out.float(), ref, atol=3e-2, rtol=2e-2)
    back = ops.rope_apply(out, cos.contiguous(), sin.contiguous(), pos, style, True)
    assert torch.allclose(back.float(), xf, atol=6e-2, rtol=3e-2)  # inverse rotation == transpose


# ----------------------------------------------------------------------------- MoE layout / permute
@pytest.mark.parametrize("T,k,E", [(1000, 4, 16), (4096, 8, 128), (37, 2, 8)])
def test_moe_layout_and_permute(ops, T, k, E):
    H = 256
    ids = torch.stack([torch.randperm(E, device="cuda")[:k] for _ in range(T)])
    ids[::13, 0] = -1  # dropped
    cap = (T * k + E * 127 + 127) // 128 * 128
    counts, seg, row_map, tile_group = ops.moe_build_layout(ids, E, 128, cap)
    flat = ids.flatten()
    ref_counts = torch.bincount(flat[flat >= 0], minlength=E)
    assert torch.equal(counts.long(), ref_counts)
    aligned = (ref_counts + 127) // 128 * 128
    ref_seg = torch.cat([torch.zeros(1, dtype=torch.long, device="cuda"), aligned.cumsum(0)])
    assert torch.equal(seg.long(), ref_seg)
    # stable sort order
    rm = row_map.long()
    for e in range(0, E, max(1, E // 8)):
        idx = (flat == e).nonzero().flatten()
        assert torch.equal(rm[idx], ref_seg[e] + torch.arange(len(idx), device="cuda"))
    assert (rm[flat < 0] == -1).all()
    tg = tile_group.long()
    for e in range(E):
        assert (tg[ref_seg[e] // 128 : ref_seg[e + 1] // 128] == e).all()
    assert (tg[ref_seg[-1] // 128 :] == -1).all()

    x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
    probs = torch.rand(T, k, device="cuda")
    xp, pp = ops.moe_permute(x, probs, row_map, counts, seg, cap)
    valid = rm >= 0
    tok = torch.arange(T, device="cuda").repeat_interleave(k)
    assert torch.equal(xp[rm[valid]], x[tok[valid]])
    assert torch.equal(pp[rm[valid]], probs.flatten()[valid])
    used = torch.zeros(cap, dtype=torch.bool, device="cuda")
    used[rm[valid]] = True
    pad = ~used
    pad[ref_seg[-1] :] = False
    assert (xp[pad] == 0).all() and (pp[pad] == 0).all()

    yp = torch.randn(cap, H, device="cuda", dtype=torch.bfloat16)
    y, _ = ops.moe_gather(yp, None, row_map, T, k)
    ref = torch.zeros(T, H, device="cuda")
    ref.index_add_(0, tok[valid], yp[rm[valid]].float())
    assert torch.allclose(y.float(), ref, atol=3e-2, rtol=2e-2)
    dpp = torch.randn(cap, device="cuda")
    y2, dprobs = ops.moe_gather(yp, dpp, row_map, T, k)
    assert torch.equal(y2, y)
    refp = torch.zeros(T * k, device="cuda")
    refp[valid] = dpp[rm[valid]]
    assert torch.equal(dprobs.flatten(), refp)


def test_grad_utils(ops):
    x = torch.randn(100003, device="cuda")
    out = torch.zeros(1, device="cuda")
    ops.sumsq_accumulate_(x, out)
    assert math.isclose(out.item(), x.pow(2).sum().item(), rel_tol=1e-4)
    xb = x.bfloat16()
    out.zero_()
    ops.sumsq_accumulate_(xb, out)
    assert math.isclose(out.item(), xb.float().pow(2).sum().item(), rel_tol=1e-4)
    sc = torch.tensor([0.5], device="cuda")
    ref = x * 0.5
    ops.scale_inplace_(x, sc)
    assert torch.allclose(x, ref)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("accumulate", [False, True])
def test_gemm_unaligned_output_uses_direct_epilogue(ops, dtype, accumulate):
    # an output whose base address is not 16-byte aligned cannot go through TMA: the direct-store epilogue must kick in
    M, N, K = 304, 200, 256
    a = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    flat = torch.randn(M * N + 1, device="cuda", dtype=dtype)
    d = flat[1:].view(M, N)
    d0 = d.clone()
    ops.gemm(a, b, d, True, True, accumulate)
    ref = a.float().t() @ b.float() + (d0.float() if accumulate else 0)
    assert _rel_err(d, ref) < (1e-2 if dtype == torch.bfloat16 else 1e-4)
    assert flat[0] == flat[0]  # untouched guard element is still a number


@pytest.mark.parametrize("M,N,K", [(128, 768, 16384), (512, 768, 8192), (2048, 768, 4096)])
def test_gemm_split_k_accumulate(ops, M, N, K):
    # few output tiles + long K: the fp32-accumulate epilogue splits K across CTAs (TMA reduce-add into the output)
    a = torch.randn(K, M, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(K, N, device="cuda", dtype=torch.bfloat16)
    d0 = torch.randn(M, N, device="cuda", dtype=torch.float32)
    d = d0.clone()
    ops.gemm(a, b, d, True, True, True)
    assert _rel_err(d, a.float().t() @ b.float() + d0) < 1e-4


@pytest.mark.parametrize("E,k", [(128, 8), (8, 2), (64, 6), (200, 4), (1024, 32)])
@pytest.mark.parametrize("renorm", [True, False])
@pytest.mark.parametrize("with_bias", [False, True])
def test_router_topk_matches_reference(ops, E, k, renorm, with_bias):
    from d9d_b200.kernel.router import route_topk, route_topk_reference

    torch.manual_seed(E + k)
    T = 777
    logits = (torch.randn(T, E, device="cuda") * 2).bfloat16()
    bias = torch.randn(E, device="cuda") * 0.05 if with_bias else None
    a = logits.clone().requires_grad_()
    b = logits.clone().float().requires_grad_()
    idx, probs = route_topk(a, k, renorm, bias)
    ridx, rprobs = route_topk_reference(b, k, renorm, bias)
    # compare as sets ordered by expert id (the order among the k selections is not part of the contract)
    order, rorder = idx.argsort(-1), ridx.argsort(-1)
    assert torch.equal(idx.gather(-1, order), ridx.gather(-1, rorder))
    torch.testing.assert_close(probs.gather(-1, order), rprobs.gather(-1, rorder), rtol=1e-4, atol=1e-6)
    w = torch.randn(T, k, device="cuda")
    (probs.gather(-1, order) * w).sum().backward()
    (rprobs.gather(-1, rorder) * w).sum().backward()
    torch.testing.assert_close(a.grad.float(), b.grad, rtol=2e-2, atol=2e-3 * float(b.grad.abs().max()))


@pytest.mark.parametrize("D,rope_dim", [(128, 128), (64, 64), (128, 64), (256, 256)])
@pytest.mark.parametrize("style", [0, 1])
@pytest.mark.parametrize("zero_centered", [False, True])
def test_fused_qk_norm_rope_matches_unfused_reference(ops, D, rope_dim, style, zero_centered):
    from d9d_b200.kernel.rope import rotate_reference
    from d9d_b200.kernel.rope.fused_qk import qk_norm_rope

    torch.manual_seed(D + style)
    B, S, Hq, Hk = 2, 75, 6, 2
    fused = torch.randn(B, S, (Hq + 2 * Hk) * D, device="cuda").bfloat16()  # q|k|v packed: exercises strided heads
    q = fused[..., : Hq * D].reshape(B, S, Hq, D)
    k = fused[..., Hq * D : (Hq + Hk) * D].reshape(B, S, Hk, D)
    wq = (torch.randn(D, device="cuda") * 0.1 + (0.0 if zero_centered else 1.0)).bfloat16()
    wk = (torch.randn(D, device="cuda") * 0.1 + (0.0 if zero_centered else 1.0)).bfloat16()
    ang = torch.rand(B, S, rope_dim // 2, device="cuda") * 6.28
    ang = torch.cat([ang, ang], -1) if style == 0 else ang.repeat_interleave(2, -1)
    cos, sin = ang.cos(), ang.sin()

    def reference(qf, kf, wqf, wkf):
        def norm(x, w):
            x = x.float()
            r = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + 1e-6)
            return x * r * (w.float() + (1.0 if zero_centered else 0.0))
        return (rotate_reference(norm(qf, wqf), cos, sin, style), rotate_reference(norm(kf, wkf), cos, sin, style))

    leaves = [t.clone().requires_grad_() for t in (q, k, wq, wk)]
    ref_leaves = [t.float().clone().requires_grad_() for t in (q, k, wq, wk)]
    qo, ko = qk_norm_rope(*leaves, cos, sin, 1e-6, zero_centered, style)
    rq, rk = reference(*ref_leaves)
    torch.testing.assert_close(qo.float(), rq, rtol=2e-2, atol=2e-2)
    torch.testing.assert_close(ko.float(), rk, rtol=2e-2, atol=2e-2)
    gq, gk = torch.randn_like(rq), torch.randn_like(rk)
    torch.autograd.backward([qo, ko], [gq.bfloat16(), gk.bfloat16()])
    torch.autograd.backward([rq, rk], [gq.bfloat16().float(), gk.bfloat16().float()])
    for a, b, name in zip(leaves, ref_leaves, ("dq", "dk", "dwq", "dwk")):
        scale = float(b.grad.abs().max())
        torch.testing.assert_close(a.grad.float(), b.grad, rtol=3e-2, atol=3e-2 * scale, msg=lambda m: f"{name}: {m}")  # noqa: B023

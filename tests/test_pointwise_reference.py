"""Self-test of the fp64 references / per-element bounds that the pointwise kernel tests rely on: each bound must accept a
correctly rounded result and a torch fp32 emulation of the kernel's order of operations, and reject the faults a broken
kernel makes.  CPU only.

In fp32 outputs a 4-ulp fault is within what the kernel may legitimately be off: ``1 / (1 + __expf(-x))`` is a few
ulps off, and so is an fp32 sum over a row or a column.  The SiLU and RMSNorm-backward bounds therefore reject it in bf16
and fp16 outputs only (the exact probes of the kernel suite cover fp32); the other bounds reject it in every dtype."""

import pytest
import torch

from tests.gemm_reference import assert_within, err_ratio
from tests.pointwise_reference import (
    f32,
    inv_rms_rel,
    moe_gather_ref,
    qk_norm_rope_bwd_ref,
    qk_norm_rope_fwd_ref,
    rms_norm_bwd_ref,
    rms_norm_fwd_ref,
    rope_ref,
    silu_mul_bwd_ref,
    silu_mul_fwd_ref,
    silu_mul_probs_bwd_ref,
    silu_mul_probs_fwd_ref,
    sumsq_ref,
)

DTYPES = [torch.bfloat16, torch.float16, torch.float32]
EPS = 1e-6


def _gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def bump_ulps(t: torch.Tensor, ref: torch.Tensor, ulps: int = 4) -> torch.Tensor:
    """t with its largest-magnitude element (by ``ref``) moved ``ulps`` units in the last place away from zero."""
    it = {2: torch.int16, 4: torch.int32}[t.element_size()]
    out = t.clone()
    i = int(ref.abs().argmax())
    out.view(it).view(-1)[i] += ulps  # sign-magnitude: adding to the bit pattern grows |value| for either sign
    return out


def _rejects(d, ref, bound):
    assert err_ratio(d, ref, bound) > 1.0


# ----------------------------------------------------------------------------- RMSNorm
def _rms_case(M, N, dtype, zc, seed=0):
    g = _gen(seed + N)
    x = (torch.randn(M, N, generator=g) * torch.rand(M, 1, generator=g) * 3 + 0.01).to(dtype)
    w = (torch.randn(N, generator=g) * 0.1 + (0.0 if zc else 1.0)).to(dtype)
    return x, w


def _rms_fwd_emulated(x, w, zc):
    """fp32, in the kernel's order: per-lane sums of 8, a tree over the lanes, rsqrt, (x * ir) * w."""
    M, N = x.shape
    xf = x.float()
    ss = xf.square().view(M, N // 8, 8).sum(-1)
    while ss.shape[1] > 1:
        if ss.shape[1] % 2:
            ss = torch.cat([ss, torch.zeros(M, 1)], 1)
        ss = ss[:, 0::2] + ss[:, 1::2]
    ir = torch.rsqrt(ss[:, 0] / N + f32(EPS))
    wf = w.float() + 1.0 if zc else w.float()
    return (xf * ir[:, None] * wf).to(x.dtype), ir


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N", [8, 72, 1032, 16384])
@pytest.mark.parametrize("zc", [False, True])
def test_rms_fwd_bound(dtype, N, zc):
    x, w = _rms_case(7, N, dtype, zc)
    ref, bound, ir_ref, ir_bound = rms_norm_fwd_ref(x, w, EPS, zc)
    assert_within(ref.to(dtype), ref, bound, "correctly rounded")
    out, ir = _rms_fwd_emulated(x, w, zc)
    assert_within(ir, ir_ref, ir_bound, "emulated inv_rms")
    ref_k, bound_k, _, _ = rms_norm_fwd_ref(x, w, EPS, zc, inv_rms=ir)
    assert_within(out, ref_k, bound_k, "emulated out")
    _rejects(bump_ulps(out, ref_k), ref_k, bound_k)
    # a row normalised with its neighbour's inv_rms: caught by the inv_rms check and by the output check
    _rejects(ir.roll(1), ir_ref, ir_bound)
    wrong = (x.float() * ir.roll(1)[:, None] * (w.float() + (1.0 if zc else 0.0))).to(dtype)
    _rejects(wrong, ref, bound)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N", [64, 136, 4104])
@pytest.mark.parametrize("zc", [False, True])
def test_rms_bwd_bound(dtype, N, zc):
    M = 37
    x, w = _rms_case(M, N, dtype, zc, seed=1)
    dy = torch.randn(M, N, generator=_gen(2)).to(dtype)
    _, ir = _rms_fwd_emulated(x, w, zc)
    dx_ref, dx_b, dw_ref, dw_b = rms_norm_bwd_ref(dy, x, w, ir, zc)
    assert_within(dx_ref.to(dtype), dx_ref, dx_b, "dx correctly rounded")
    assert_within(dw_ref.to(dtype), dw_ref, dw_b, "dw correctly rounded")
    # fp32 emulation: xh = x * ir, dot of dy * w * xh summed per row, dx = ir * (dy * w - xh * mean)
    xf, df, ir2 = x.float(), dy.float(), ir[:, None]
    wf = w.float() + 1.0 if zc else w.float()
    xh = xf * ir2
    mean = (df * wf * xh).sum(-1, keepdim=True) / N
    dx = (ir2 * (df * wf - xh * mean)).to(dtype)
    dw = (df * xh).sum(0).to(dtype)
    assert_within(dx, dx_ref, dx_b, "dx emulated")
    assert_within(dw, dw_ref, dw_b, "dw emulated")
    if dtype != torch.float32:
        _rejects(bump_ulps(dx, dx_ref), dx_ref, dx_b)
        _rejects(bump_ulps(dw, dw_ref), dw_ref, dw_b)
    # a row normalised with its neighbour's inv_rms; a dw that lost the last row
    irr = ir.roll(1)[:, None]
    _rejects((irr * (df * wf - xf * irr * ((df * wf * xf * irr).sum(-1, keepdim=True) / N))).to(dtype), dx_ref, dx_b)
    _rejects((df[:-1] * xh[:-1]).sum(0).to(dtype), dw_ref, dw_b)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rms_end_to_end_bound(dtype):
    """The fp64 inv_rms with its error term: fp32 autograd of the RMSNorm formula stays inside."""
    M, N = 33, 512
    x, w = _rms_case(M, N, dtype, False, seed=3)
    dy = torch.randn(M, N, generator=_gen(4)).to(dtype)
    ir64 = torch.rsqrt(x.double().square().mean(-1) + f32(EPS))
    dx_ref, dx_b, dw_ref, dw_b = rms_norm_bwd_ref(dy, x, w, ir64, False, ir_rel=inv_rms_rel(N))
    xr, wr = x.float().requires_grad_(), w.float().requires_grad_()
    (xr * torch.rsqrt(xr.square().mean(-1, keepdim=True) + EPS) * wr).backward(dy.float())
    assert_within(xr.grad.to(dtype), dx_ref, dx_b, "dx")
    assert_within(wr.grad.to(dtype), dw_ref, dw_b, "dw")


# ----------------------------------------------------------------------------- SiLU * mul (* probs)
@pytest.mark.parametrize("dtype", DTYPES)
def test_silu_mul_bound(dtype):
    g = _gen(5)
    x = (torch.randn(4099, generator=g) * 3).to(dtype)
    y, dout = torch.randn(4099, generator=g).to(dtype), torch.randn(4099, generator=g).to(dtype)
    ref, bound = silu_mul_fwd_ref(x, y)
    assert_within(ref.to(dtype), ref, bound, "correctly rounded")
    emu = (torch.nn.functional.silu(x.float()).to(dtype).float() * y.float()).to(dtype)  # silu rounded before the product
    assert_within(emu, ref, bound, "silu rounded first")
    dx_ref, dx_b, dy_ref, dy_b = silu_mul_bwd_ref(dout, x, y)
    xf, yf, gf = x.float(), y.float(), dout.float()
    sg = torch.sigmoid(xf)
    silu = xf * sg
    dx, dy = (gf * yf * (sg + silu * (1 - sg))).to(dtype), (gf * silu).to(dtype)
    assert_within(dx_ref.to(dtype), dx_ref, dx_b, "dx correctly rounded")
    assert_within(dx, dx_ref, dx_b, "dx emulated")
    assert_within(dy, dy_ref, dy_b, "dy emulated")
    if dtype != torch.float32:
        _rejects(bump_ulps(emu, ref), ref, bound)
        _rejects(bump_ulps(dx, dx_ref), dx_ref, dx_b)
        _rejects(bump_ulps(dy, dy_ref), dy_ref, dy_b)


def test_silu_mul_probs_bound():
    R, C = 19, 264
    g = _gen(6)
    x, y, dout = ((torch.randn(R, C, generator=g) * 3).bfloat16(), torch.randn(R, C, generator=g).bfloat16(),
                  torch.randn(R, C, generator=g).bfloat16())
    p = torch.rand(R, generator=g)
    ref, bound = silu_mul_probs_fwd_ref(x, y, p)
    xf, yf, gf = x.float(), y.float(), dout.float()
    sg = torch.sigmoid(xf)
    silu = xf * sg
    out = (silu * yf * p[:, None]).bfloat16()
    assert_within(out, ref, bound, "fwd")
    _rejects(bump_ulps(out, ref), ref, bound)
    dx_ref, dx_b, dy_ref, dy_b, dp_ref, dp_b = silu_mul_probs_bwd_ref(dout, x, y, p)
    gp = gf * p[:, None]
    dx, dy = (gp * yf * (sg + silu * (1 - sg))).bfloat16(), (gp * silu).bfloat16()
    dp = (gf * silu * yf).view(R, C // 8, 8).sum(-1).sum(-1)  # per lane, then across the warp
    assert_within(dx, dx_ref, dx_b, "dx")
    assert_within(dy, dy_ref, dy_b, "dy")
    assert_within(dp, dp_ref, dp_b, "dprobs")
    _rejects(bump_ulps(dx, dx_ref), dx_ref, dx_b)
    _rejects(dp.roll(1), dp_ref, dp_b)  # one row's dprobs from the wrong row (here: every row's)
    bad = dp.clone()
    bad[5] = dp[6]
    _rejects(bad, dp_ref, dp_b)


# ----------------------------------------------------------------------------- RoPE
def _angles(maxpos, rope_dim, style, seed):
    ang = torch.rand(maxpos, rope_dim // 2, generator=_gen(seed)) * 6.28
    ang = torch.cat([ang, ang], -1) if style == 0 else ang.repeat_interleave(2, -1)
    return ang.cos(), ang.sin()


def _rope_f32(x, c, s, style):
    rd = c.shape[-1]
    xf = x.float()
    xr = xf[..., :rd]
    if style == 0:
        rot = torch.cat([-xr[..., rd // 2:], xr[..., : rd // 2]], -1)
    else:
        rot = torch.stack([-xr[..., 1::2], xr[..., 0::2]], -1).flatten(-2)
    return torch.cat([xr * c + rot * s, xf[..., rd:]], -1).to(x.dtype)


@pytest.mark.parametrize("style", [0, 1])
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("D,rope_dim", [(64, 64), (128, 32), (256, 80)])
def test_rope_bound(style, inverse, D, rope_dim):
    T, H, maxpos = 23, 3, 64
    x = torch.randn(T, H, D, generator=_gen(7)).bfloat16()
    cos, sin = _angles(maxpos, rope_dim, style, 8)
    pos = torch.randint(0, maxpos, (T,), generator=_gen(9))
    ref, bound = rope_ref(x, cos, sin, pos, style, inverse)
    c, s = cos[pos][:, None], sin[pos][:, None]
    s = -s if inverse else s
    out = _rope_f32(x, c, s, style)
    assert_within(ref.bfloat16(), ref, bound, "correctly rounded")
    assert_within(out, ref, bound, "fp32")
    _rejects(bump_ulps(out, ref), ref, bound)
    _rejects(_rope_f32(x, c, -s, style), ref, bound)  # sign of the rotation flipped
    if rope_dim < D:  # pass-through dims rotated too (by one radian)
        rest = D - rope_dim
        wrong = out.clone()
        wrong[..., rope_dim:] = _rope_f32(x[..., rope_dim:], torch.full((rest,), 0.5403), torch.full((rest,), 0.8415), 1)
        _rejects(wrong, ref, bound)
    if style == 0:
        # HALF-style partner taken from the wrong lane: one lane's worth (D / 32 elements) too far
        vec = D // 32
        rd = rope_dim
        xf = x.float()
        xr = xf[..., :rd]
        part = torch.cat([-xr[..., rd // 2:], xr[..., : rd // 2]], -1).roll(vec, -1)
        wrong = torch.cat([xr * c + part * s, xf[..., rd:]], -1).bfloat16()
        _rejects(wrong, ref, bound)


# ----------------------------------------------------------------------------- fused q/k RMSNorm + RoPE
@pytest.mark.parametrize("style", [0, 1])
@pytest.mark.parametrize("D,rope_dim", [(64, 16), (128, 128), (256, 32)])
def test_qk_norm_rope_bound(style, D, rope_dim):
    T, Hq, Hk = 9, 5, 3
    g = _gen(10)
    q, k = (torch.randn(T, Hq, D, generator=g) * 2).bfloat16(), torch.randn(T, Hk, D, generator=g).bfloat16()
    wq, wk = (torch.randn(D, generator=g) * 0.1 + 1).bfloat16(), (torch.randn(D, generator=g) * 0.1 + 1).bfloat16()
    cos, sin = _angles(T, rope_dim, style, 11)
    qo_r, qo_b, ko_r, ko_b, ir_r, ir_b = qk_norm_rope_fwd_ref(q, k, wq, wk, cos, sin, EPS, False, style)
    x = torch.cat([q, k], 1).float()
    ir = torch.rsqrt(x.view(T, Hq + Hk, D // 8, 8).square().sum(-1).sum(-1) / D + f32(EPS))
    assert_within(ir, ir_r, ir_b, "inv_rms")
    _rejects(ir.roll(1, 1), ir_r, ir_b)
    qo_r, qo_b, ko_r, ko_b, _, _ = qk_norm_rope_fwd_ref(q, k, wq, wk, cos, sin, EPS, False, style, inv_rms=ir)
    c, s = cos[:, None], sin[:, None]
    qo = _rope_f32((q.float() * ir[:, :Hq, None] * wq.float()), c, s, style).bfloat16()
    ko = _rope_f32((k.float() * ir[:, Hq:, None] * wk.float()), c, s, style).bfloat16()
    assert_within(qo, qo_r, qo_b, "q out")
    assert_within(ko, ko_r, ko_b, "k out")
    _rejects(bump_ulps(ko, ko_r), ko_r, ko_b)
    _rejects(_rope_f32((q.float() * ir[:, :Hq, None].roll(1, 1) * wq.float()), c, s, style).bfloat16(), qo_r, qo_b)

    gq, gk = torch.randn(T, Hq, D, generator=g).bfloat16(), torch.randn(T, Hk, D, generator=g).bfloat16()
    dq_r, dq_b, dk_r, dk_b, dwq_r, dwq_b, dwk_r, dwk_b = qk_norm_rope_bwd_ref(gq, gk, q, k, wq, wk, cos, sin, ir, False, style)
    outs = []
    for gg, xx, ww, irx in ((gq, q, wq, ir[:, :Hq]), (gk, k, wk, ir[:, Hq:])):
        rd = c.shape[-1]  # rotate back by -theta in fp32
        gf = gg.float()
        gr = gf[..., :rd]
        rot = torch.cat([-gr[..., rd // 2:], gr[..., : rd // 2]], -1) if style == 0 else torch.stack([-gr[..., 1::2], gr[..., 0::2]], -1).flatten(-2)
        dy = torch.cat([gr * c - rot * s, gf[..., rd:]], -1)
        xh = xx.float() * irx[..., None]
        gw = dy * ww.float()
        mean = (gw * xh).sum(-1, keepdim=True) / D
        outs += [(irx[..., None] * (gw - xh * mean)).bfloat16(), (dy * xh).sum((0, 1))]
    dq, dwq, dk, dwk = outs
    assert_within(dq, dq_r, dq_b, "dq")
    assert_within(dk, dk_r, dk_b, "dk")
    assert_within(dwq, dwq_r, dwq_b, "dwq")
    assert_within(dwk, dwk_r, dwk_b, "dwk")
    _rejects(bump_ulps(dq, dq_r), dq_r, dq_b)
    _rejects(dwq - dwq_r.float() / T, dwq_r, dwq_b)  # a lost token's worth of the weight gradient, on average


# ----------------------------------------------------------------------------- MoE gather, sumsq
def test_moe_gather_bound():
    T, k, H, cap = 31, 4, 64, 200
    g = _gen(12)
    rm = torch.randperm(cap, generator=g)[: T * k].int()
    rm[::5] = -1
    yp = torch.randn(cap, H, generator=g).bfloat16()
    dpp = torch.randn(cap, generator=g)
    y_r, y_b, dp_r = moe_gather_ref(yp, rm, T, k, dpp)
    r = rm.long().view(T, k)
    rows = yp.float()[r.clamp_min(0)] * (r >= 0)[..., None]
    acc = torch.zeros(T, H)
    for j in range(k):  # sequential fp32 sum, as in the kernel
        acc = acc + rows[:, j]
    assert_within(acc.bfloat16(), y_r, y_b, "y")
    _rejects(rows[:, : k - 1].sum(1).bfloat16(), y_r, y_b)  # k-1 of the k rows
    assert torch.equal(dp_r.float(), torch.where(r >= 0, dpp[r.clamp_min(0)], 0.0))


def test_sumsq_bound():
    x = torch.randn(100003, generator=_gen(13))
    ref, bound = sumsq_ref(x, 3.0e4, adds=64)
    out = torch.tensor(3.0e4)
    for part in x.chunk(64):  # fp32 block sums, each added to the running total
        out = out + part.square().sum()
    assert abs(float(out) - ref) <= bound
    assert abs(float(x.square().sum()) - ref) > bound  # '=' instead of '+='

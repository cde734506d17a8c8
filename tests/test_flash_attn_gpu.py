"""Native wgmma flash attention (forward + backward) against the fp32 oracle of the same op.

Mirrors the reference's coverage of ``flash_attn_func`` / ``flash_attn_varlen_func`` (causal, GQA/MQA, sliding windows,
learnable sinks with ``dsink``, soft-cap, packed sequences; ``d9d/kernel/flash_attn/function.py``)."""

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _oracle(q, k, v, causal, window, sink, softcap, dout, dlse=None):
    from d9d_b200.kernel.flash_attn.function import attention_reference

    leaves = [t.detach().float().requires_grad_() for t in (q, k, v)]
    s = sink.detach().float().requires_grad_() if sink is not None else None
    out, lse = attention_reference(*leaves, None, causal, window, s, softcap)
    loss = (out.float() * dout.float()).sum()
    if dlse is not None:
        loss = loss + (torch.nan_to_num(lse, neginf=0.0) * dlse).sum()
    loss.backward()
    return out, lse, [t.grad for t in leaves], (s.grad if s is not None else None)


def _check(name, got, ref, tol=2.5e-2):
    got, ref = got.float(), ref.float()
    scale = float(ref.abs().max()) + 1e-6
    err = float((got - ref).abs().max()) / scale
    assert err < tol, f"{name}: max err {err:.4f} (relative to max |ref| {scale:.3g})"


CASES = [
    # B, Sq, Sk, Hq, Hk, D, causal, window, sink, softcap
    (2, 256, 256, 4, 2, 128, True, (None, None), False, 0.0),
    (2, 256, 256, 4, 2, 128, False, (None, None), False, 0.0),
    (1, 384, 384, 2, 2, 64, True, (None, None), False, 0.0),
    (2, 200, 200, 4, 1, 128, True, (None, None), False, 0.0),
    (1, 128, 512, 2, 1, 128, True, (None, None), False, 0.0),
    (1, 512, 128, 2, 1, 128, True, (None, None), False, 0.0),
    (1, 1000, 1000, 3, 3, 64, False, (None, None), False, 0.0),
    (1, 777, 777, 4, 2, 128, True, (100, None), False, 0.0),
    (1, 640, 640, 2, 2, 128, False, (64, 32), False, 0.0),
    (2, 320, 320, 4, 2, 128, True, (None, None), True, 0.0),
    (1, 512, 512, 2, 1, 128, True, (200, None), True, 0.0),
    (1, 300, 300, 2, 2, 64, True, (None, None), False, 20.0),
    (1, 2048, 2048, 8, 2, 128, True, (None, None), False, 0.0),
]


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,D,causal,window,use_sink,softcap", CASES)
def test_flash_attention_forward_backward(ops, B, Sq, Sk, Hq, Hk, D, causal, window, use_sink, softcap):
    from d9d_b200.kernel.flash_attn import flash_attn_func

    torch.manual_seed(Sq * 7 + D + Hq)
    q = torch.randn(B, Sq, Hq, D, device="cuda").bfloat16().requires_grad_()
    k = torch.randn(B, Sk, Hk, D, device="cuda").bfloat16().requires_grad_()
    v = torch.randn(B, Sk, Hk, D, device="cuda").bfloat16().requires_grad_()
    sink = torch.randn(Hq, device="cuda").requires_grad_() if use_sink else None
    dout = torch.randn(B, Sq, Hq, D, device="cuda").bfloat16()
    out, lse = flash_attn_func(q, k, v, causal=causal, window_size=window, learnable_sink=sink, softcap=softcap, return_lse=True)
    out.backward(dout)
    ref_out, ref_lse, (rdq, rdk, rdv), rdsink = _oracle(q, k, v, causal, window, sink, softcap, dout)
    _check("out", out, ref_out)
    finite = torch.isfinite(ref_lse)
    torch.testing.assert_close(lse[finite], ref_lse[finite], rtol=2e-3, atol=2e-3)
    _check("dq", q.grad, rdq)
    _check("dk", k.grad, rdk)
    _check("dv", v.grad, rdv)
    if use_sink:
        _check("dsink", sink.grad, rdsink)


def test_flash_attention_lse_gradient(ops):
    from d9d_b200.kernel.flash_attn import flash_attn_func

    torch.manual_seed(3)
    q = torch.randn(1, 256, 2, 128, device="cuda").bfloat16().requires_grad_()
    k = torch.randn(1, 256, 1, 128, device="cuda").bfloat16().requires_grad_()
    v = torch.randn(1, 256, 1, 128, device="cuda").bfloat16().requires_grad_()
    dout = torch.randn(1, 256, 2, 128, device="cuda").bfloat16()
    dlse = torch.randn(1, 2, 256, device="cuda")
    out, lse = flash_attn_func(q, k, v, causal=True, return_lse=True)
    torch.autograd.backward([out, lse], [dout, dlse])
    _, _, (rdq, rdk, rdv), _ = _oracle(q, k, v, True, (None, None), None, 0.0, dout, dlse)
    _check("dq", q.grad, rdq)
    _check("dk", k.grad, rdk)
    _check("dv", v.grad, rdv)


@pytest.mark.parametrize("causal,window", [(True, (None, None)), (False, (None, None)), (True, (64, None))])
def test_flash_attention_varlen_matches_per_sequence(ops, causal, window):
    from d9d_b200.kernel.flash_attn import flash_attn_func, flash_attn_varlen_func

    torch.manual_seed(11)
    lens = [130, 1, 257, 64, 300]
    Hq, Hk, D = 4, 2, 128
    total = sum(lens)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device="cuda", dtype=torch.int32)
    q = torch.randn(total, Hq, D, device="cuda").bfloat16().requires_grad_()
    k = torch.randn(total, Hk, D, device="cuda").bfloat16().requires_grad_()
    v = torch.randn(total, Hk, D, device="cuda").bfloat16().requires_grad_()
    dout = torch.randn(total, Hq, D, device="cuda").bfloat16()
    out, lse = flash_attn_varlen_func(q, k, v, cu, cu, max(lens), max(lens), causal=causal, window_size=window, return_lse=True)
    out.backward(dout)
    got = [t.grad.clone() for t in (q, k, v)]
    for t in (q, k, v):
        t.grad = None
    outs, lses = [], []
    start = 0
    for n in lens:
        sl = slice(start, start + n)
        o, l = flash_attn_func(q[sl][None], k[sl][None], v[sl][None], causal=causal, window_size=window, return_lse=True)
        outs.append(o[0])
        lses.append(l[0])
        start += n
    ref_out = torch.cat(outs)
    ref_out.backward(dout)
    _check("out", out, ref_out, tol=1e-3)
    torch.testing.assert_close(lse, torch.cat(lses, dim=-1), rtol=1e-4, atol=1e-4)
    for name, a, t in zip(("dq", "dk", "dv"), got, (q, k, v)):
        _check(name, a, t.grad, tol=1e-3)


def test_attention_entry_point_is_native_in_training(ops):
    """No library (cuDNN / SDPA) kernel on the training path: forward + backward = our launches only."""
    from d9d_b200.kernel._native import native_ops
    from d9d_b200.kernel.flash_attn.function import flash_attn_func

    q = torch.randn(1, 256, 4, 128, device="cuda").bfloat16().requires_grad_()
    k = torch.randn(1, 256, 2, 128, device="cuda").bfloat16().requires_grad_()
    v = torch.randn(1, 256, 2, 128, device="cuda").bfloat16().requires_grad_()
    before = native_ops().launches
    out, _ = flash_attn_func(q, k, v, causal=True)
    assert native_ops().launches == before + 1
    out.sum().backward()
    assert native_ops().launches == before + 4  # + delta, dK/dV, dQ kernels
    assert q.grad is not None and k.grad is not None and v.grad is not None

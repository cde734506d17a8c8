"""Native wgmma flash attention (forward, delta pre-pass, dK/dV and dQ kernels) against the fp64 reference and per-element
error bound of ``tests/attention_reference.py``: out, lse, dq, dk, dv and dsink of every case, at every (qk, v) head-dim
pair the kernels are built for: (64, 64), (128, 128) and (192, 128), the last as multi-head latent attention uses it.

Inputs are peaky (scores reach about +-20, so soft-caps of 5 to 10 bend them) and every row's scores rise from one key tile to
the next, so the online softmax rescales.  The matrix covers sequence lengths on the 128-row forward and 64-row backward tile
edges, and at (192, 128) on the 32-row streamed dK/dV tile edges; Sq > Sk causal (query tiles without a visible key); windows
(0, 0), causal, right-only, left >= Sk and left at 127 / 128 / 129, also with Sq != Sk; GQA groups 1, 2, 4, 8 and 16;
soft-cap with windows, sinks and packing; sinks of +-8 and one 100 above the row max; a nonzero dlse; an explicit
softmax_scale; B = 2 and 3; packed batches with cu_seqlens_q != cu_seqlens_k, empty sequences, rows outside every sequence
and 70,000 one-token sequences.

Sequence isolation: every row outside the sequence under test (neighbours, other batch elements, padding) is NaN; the rows
under test must stay within bound, and rows outside every sequence come back as out = dq = dk = dv = 0, lse = -inf.

Set D9D_ATTN_REPORT=<file> to write the worst err/bound per output tensor and head-dim pair as JSON.
"""

import json
import math
import os

import pytest
import torch

from tests.attention_reference import assert_lse_within, assert_within, batch_reference, fixed_reference, make_inputs

pytestmark = pytest.mark.gpu

P64, P128, P192 = (64, 64), (128, 128), (192, 128)
EQ, ALL = (P64, P128), (P64, P128, P192)

_worst: dict[str, dict[str, float]] = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("D9D_ATTN_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({"worst_err_over_bound": _worst}, f, indent=1)


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _per_pair(table):
    """(Dqk, Dv, *row) for every head-dim pair listed in the first column of each row."""
    return [(*dims, *row) for pairs, *row in table for dims in pairs]


def _seed_offset(Dqk, Dv):
    """Equal-dims cases add their head dim to the seed, (192, 128) cases add nothing."""
    return Dqk if Dqk == Dv else 0


def _check(got: dict, ref: dict, what: str, dims: tuple[int, int], rows: dict | None = None) -> None:
    """got / ref keyed by output name; ``rows`` optionally maps a name to a function selecting the rows to compare."""
    worst = _worst.setdefault("{}-{}".format(*dims), {})
    for name, (want, bound) in ref.items():
        if name not in got:
            continue
        g = got[name].detach()
        assert g.shape == want.shape, (what, name, g.shape, want.shape)
        if rows is not None:
            if name not in rows:
                continue
            g, want, bound = (rows[name](t) for t in (g, want, bound))
        if name == "lse":
            r = assert_lse_within(g, want, bound, f"{what} {name}")
        else:
            r = assert_within(g, want, bound, f"{what} {name}")
        worst[name] = max(worst.get(name, 0.0), r)


def _sink(pattern, Hq):
    if pattern is None:
        return None
    return torch.tensor([pattern[h % len(pattern)] for h in range(Hq)], device="cuda", dtype=torch.float32).requires_grad_()


def _api_window(wl, wr, seed):
    """(causal, window_size) for the kernel window (wl, wr); causal windows alternate between the two spellings."""
    causal = wr == 0 and seed % 2 == 0
    return causal, (wl if wl >= 0 else None, None if causal else (wr if wr >= 0 else None))


def _run_fixed(B, Sq, Sk, Hq, Hk, Dqk, Dv, wl, wr, softcap=0.0, sink=None, dlse=False, scale=None, seed=0, poison=None):
    from d9d_b200.kernel.flash_attn import flash_attn_func

    sc = scale if scale is not None else 1.0 / math.sqrt(Dqk)
    gen = torch.Generator().manual_seed(seed)
    q, k, v, dout = make_inputs(Sq, Sk, Hq, Hk, Dqk, Dv, scale=sc, B=B, gen=gen, device="cuda")
    dl = torch.randn(B, Hq, Sq, generator=gen).cuda() if dlse else None
    qi, ki, vi, doi = q.clone(), k.clone(), v.clone(), dout.clone()
    if poison is not None:  # every batch element but `poison` is NaN
        for t in (qi, ki, vi, doi):
            t[torch.arange(B) != poison] = float("nan")
    qi, ki, vi = (t.requires_grad_() for t in (qi, ki, vi))
    s = _sink(sink, Hq)
    causal, window = _api_window(wl, wr, seed)
    out, lse = flash_attn_func(qi, ki, vi, softmax_scale=scale, causal=causal, window_size=window, learnable_sink=s,
                               softcap=softcap, return_lse=True)
    torch.autograd.backward([out, lse] if dl is not None else [out], [dout if poison is None else doi] + ([dl] if dl is not None else []))
    got = {"out": out, "lse": lse, "dq": qi.grad, "dk": ki.grad, "dv": vi.grad}
    if s is not None and poison is None:
        got["dsink"] = s.grad
    ref = fixed_reference(q, k, v, scale=sc, wl=wl, wr=wr, softcap=softcap, sink=None if s is None else s.detach(),
                          out=out.detach(), dout=dout, dlse=dl)
    rows = None if poison is None else {n: (lambda t: t[poison]) for n in ("out", "lse", "dq", "dk", "dv")}
    _check(got, ref, f"B={B} Sq={Sq} Sk={Sk} Hq={Hq} Hk={Hk} D=({Dqk},{Dv}) w=({wl},{wr}) cap={softcap} sink={sink}", (Dqk, Dv),
           rows)
    return got


FIXED = [
    # head-dim pairs, B, Sq, Sk, Hq, Hk, wl, wr, softcap, sink, dlse, scale
    (ALL, 1, 1, 1, 2, 1, -1, -1, 0.0, None, False, None),
    ((P192,), 1, 31, 31, 2, 2, -1, 0, 0.0, None, False, None),
    ((P192,), 1, 33, 33, 4, 1, -1, -1, 0.0, None, True, None),
    (ALL, 1, 63, 63, 2, 2, -1, 0, 0.0, None, False, None),
    (ALL, 1, 64, 64, 4, 1, -1, -1, 0.0, None, True, None),
    (ALL, 1, 65, 65, 2, 1, -1, 0, 0.0, [8.0, -8.0], False, None),
    ((P192,), 1, 97, 97, 2, 2, -1, 0, 0.0, None, False, None),
    (ALL, 1, 127, 127, 2, 2, -1, 0, 0.0, None, False, None),
    (ALL, 1, 128, 128, 2, 2, -1, -1, 0.0, None, True, None),
    (EQ, 1, 129, 129, 8, 1, -1, 0, 0.0, None, False, None),
    ((P192,), 1, 129, 129, 4, 1, -1, 0, 0.0, None, False, None),
    (EQ, 1, 255, 255, 16, 1, -1, -1, 0.0, None, False, None),
    ((P192,), 1, 255, 255, 4, 1, -1, -1, 0.0, None, False, None),
    (ALL, 1, 256, 256, 2, 2, 128, 0, 0.0, None, False, None),
    (ALL, 1, 257, 257, 2, 2, 127, -1, 0.0, None, False, None),   # left-only window
    (ALL, 1, 257, 257, 2, 1, 129, 0, 0.0, None, True, None),
    (ALL, 1, 200, 200, 2, 2, 0, 0, 0.0, None, False, None),      # window (0, 0)
    (ALL, 1, 200, 200, 2, 2, -1, 5, 0.0, None, False, None),     # right-only window
    (EQ, 1, 100, 300, 2, 2, 400, -1, 0.0, None, False, None),
    (ALL, 1, 257, 129, 2, 1, -1, 0, 0.0, None, False, None),     # causal Sq > Sk
    (ALL, 1, 257, 129, 2, 1, -1, 0, 0.0, [8.0, -8.0], True, None),
    (ALL, 1, 129, 257, 2, 2, 64, 0, 0.0, None, False, None),
    (EQ, 1, 300, 200, 2, 2, 50, 10, 0.0, None, False, None),
    (EQ, 1, 257, 257, 2, 1, 128, 0, 5.0, None, False, None),
    ((P192,), 1, 257, 257, 4, 1, 128, 0, 5.0, None, False, None),
    (ALL, 1, 200, 200, 2, 2, -1, 0, 10.0, [8.0, -8.0], True, None),
    (EQ, 1, 129, 129, 2, 2, -1, 0, 0.0, [125.0, -8.0], False, None),
    (ALL, 1, 65, 65, 2, 2, 0, 0, 0.0, [125.0, 125.0], True, None),
    (EQ, 1, 200, 200, 4, 2, -1, 0, 0.0, None, False, 0.05),
    ((P192,), 1, 200, 200, 4, 1, -1, 0, 0.0, None, False, 0.05),
    (EQ, 3, 200, 200, 4, 2, -1, 0, 7.0, [8.0, -8.0], True, None),
    ((P192,), 3, 200, 200, 4, 1, -1, 0, 7.0, [8.0, -8.0], True, None),
    (ALL, 1, 8192, 8192, 1, 1, -1, 0, 0.0, None, False, None),
    # flagship-like shapes: B = 2, longer and uneven sequences, windows with Sq = Sk, a soft-cap of 20 and sinks near 0
    ((P128,), 2, 256, 256, 4, 2, -1, 0, 0.0, None, False, None),
    ((P128,), 2, 256, 256, 4, 2, -1, -1, 0.0, None, False, None),
    ((P64,), 1, 384, 384, 2, 2, -1, 0, 0.0, None, False, None),
    ((P128,), 2, 200, 200, 4, 1, -1, 0, 0.0, None, False, None),
    ((P128,), 1, 128, 512, 2, 1, -1, 0, 0.0, None, False, None),
    ((P128,), 1, 512, 128, 2, 1, -1, 0, 0.0, None, False, None),
    ((P64,), 1, 1000, 1000, 3, 3, -1, -1, 0.0, None, False, None),
    ((P128,), 1, 777, 777, 4, 2, 100, 0, 0.0, None, False, None),
    ((P128,), 1, 640, 640, 2, 2, 64, 32, 0.0, None, False, None),
    ((P128,), 2, 320, 320, 4, 2, -1, 0, 0.0, [1.0, -1.0], False, None),
    ((P128,), 1, 512, 512, 2, 1, 200, 0, 0.0, [1.0, -1.0], False, None),
    ((P64,), 1, 300, 300, 2, 2, -1, 0, 20.0, None, False, None),
    ((P128,), 1, 2048, 2048, 8, 2, -1, 0, 0.0, None, False, None),
]


@pytest.mark.parametrize("Dqk,Dv,B,Sq,Sk,Hq,Hk,wl,wr,softcap,sink,dlse,scale", _per_pair(FIXED))
def test_fixed_length(ops, B, Sq, Sk, Hq, Hk, Dqk, Dv, wl, wr, softcap, sink, dlse, scale):
    _run_fixed(B, Sq, Sk, Hq, Hk, Dqk, Dv, wl, wr, softcap, sink, dlse, scale, seed=Sq * 31 + Sk + Hq + _seed_offset(Dqk, Dv))


@pytest.mark.parametrize("Dqk,Dv,Hk", [(64, 64, 2), (128, 128, 2), (192, 128, 1)], ids=["64", "128", "192-128"])
@pytest.mark.parametrize("poison", [0, 1, 2])
def test_fixed_batch_isolation(ops, Dqk, Dv, Hk, poison):
    _run_fixed(3, 200, 200, 4, Hk, Dqk, Dv, 100, 0, 5.0, [8.0], True, None, seed=3, poison=poison)


def _run_varlen(lens_q, lens_k, Hq, Hk, Dqk, Dv, wl, wr, softcap=0.0, sink=None, dlse=False, lead=0, pad_q=0, pad_k=0, seed=0,
                poison=None):
    """Packed batch with `lead` rows before the first query sequence and pad_q / pad_k rows after the last.  poison = b: every
    row outside sequence b is NaN."""
    from d9d_b200.kernel.flash_attn import flash_attn_varlen_func

    sc = 1.0 / math.sqrt(Dqk)
    cu_q = [lead] + [lead + sum(lens_q[: i + 1]) for i in range(len(lens_q))]
    cu_k = [0] + [sum(lens_k[: i + 1]) for i in range(len(lens_k))]
    total_q, total_k = cu_q[-1] + pad_q, cu_k[-1] + pad_k
    gen = torch.Generator().manual_seed(seed)
    q, k, v, dout = make_inputs(total_q, total_k, Hq, Hk, Dqk, Dv, scale=sc, gen=gen, device="cuda")
    dl = torch.randn(Hq, total_q, generator=gen).cuda() if dlse else None
    qi, ki, vi, doi = q.clone(), k.clone(), v.clone(), dout.clone()
    inside_q = torch.zeros(total_q, dtype=torch.bool)
    inside_k = torch.zeros(total_k, dtype=torch.bool)
    inside_q[cu_q[0] : cu_q[-1]] = True
    inside_k[cu_k[0] : cu_k[-1]] = True
    if poison is not None:
        keep_q = torch.zeros(total_q, dtype=torch.bool)
        keep_k = torch.zeros(total_k, dtype=torch.bool)
        keep_q[cu_q[poison] : cu_q[poison + 1]] = True
        keep_k[cu_k[poison] : cu_k[poison + 1]] = True
        qi[~keep_q], doi[~keep_q] = float("nan"), float("nan")
        ki[~keep_k], vi[~keep_k] = float("nan"), float("nan")
    qi, ki, vi = (t.requires_grad_() for t in (qi, ki, vi))
    s = _sink(sink, Hq)
    causal, window = _api_window(wl, wr, seed)
    tq = torch.tensor(cu_q, dtype=torch.int32, device="cuda")
    tk = torch.tensor(cu_k, dtype=torch.int32, device="cuda")
    out, lse = flash_attn_varlen_func(qi, ki, vi, tq, tk, max(lens_q), max(lens_k), causal=causal, window_size=window,
                                      learnable_sink=s, softcap=softcap, return_lse=True)
    torch.autograd.backward([out, lse] if dl is not None else [out], [doi] + ([dl] if dl is not None else []))
    got = {"out": out, "lse": lse, "dq": qi.grad, "dk": ki.grad, "dv": vi.grad}
    if s is not None and poison is None:
        got["dsink"] = s.grad
    ref = batch_reference(q, k, v, cu_q, cu_k, scale=sc, wl=wl, wr=wr, softcap=softcap, sink=None if s is None else s.detach(),
                          out=out.detach(), dout=dout, dlse=dl)
    rows = None
    if poison is not None:  # the sequence under test plus every row outside all sequences
        rq = (keep_q | ~inside_q).cuda()
        rk = (keep_k | ~inside_k).cuda()
        rows = {"out": lambda t: t[rq], "dq": lambda t: t[rq], "lse": lambda t: t[:, rq], "dk": lambda t: t[rk],
                "dv": lambda t: t[rk]}
    _check(got, ref, f"varlen q={lens_q} k={lens_k} D=({Dqk},{Dv}) w=({wl},{wr}) cap={softcap} sink={sink} poison={poison}",
           (Dqk, Dv), rows)
    return got


VARLEN = [
    # head-dim pairs, lens_q, lens_k, Hq, Hk, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k
    (EQ, [1, 63, 129, 64], [1, 200, 129, 300], 4, 2, -1, 0, 7.0, [8.0, -8.0], True, 0, 0, 0),  # q: suffix of a longer k
    ((P192,), [1, 63, 129, 64], [1, 200, 129, 300], 4, 1, -1, 0, 7.0, [8.0, -8.0], True, 0, 0, 0),
    (ALL, [70, 129, 20], [150, 60, 257], 2, 1, 128, 0, 0.0, None, False, 0, 0, 0),
    (ALL, [0, 65, 0, 127, 3], [0, 0, 64, 128, 257], 2, 2, -1, 0, 5.0, [8.0], True, 3, 5, 7),  # empty q / k / both, padding
    (EQ, [63, 64, 65, 127, 128, 129, 255, 256, 257], [63, 64, 65, 127, 128, 129, 255, 256, 257], 4, 1, 127, -1, 0.0, [-8.0],
     False, 0, 0, 0),
    ((P192,), [31, 33, 63, 65, 127, 129, 255, 257], [31, 33, 63, 65, 127, 129, 255, 257], 4, 1, 127, -1, 0.0, [-8.0], False,
     0, 0, 0),
    (ALL, [100, 37], [100, 37], 2, 2, -1, -1, 10.0, None, True, 0, 61, 13),
]


@pytest.mark.parametrize("Dqk,Dv,lens_q,lens_k,Hq,Hk,wl,wr,softcap,sink,dlse,lead,pad_q,pad_k", _per_pair(VARLEN))
def test_varlen(ops, lens_q, lens_k, Hq, Hk, Dqk, Dv, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k):
    _run_varlen(lens_q, lens_k, Hq, Hk, Dqk, Dv, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k,
                seed=len(lens_q) + wl + _seed_offset(Dqk, Dv))


@pytest.mark.parametrize("Dqk,Dv,lens_q,lens_k,Hq,Hk,wl,wr,softcap,sink,dlse,lead,pad_q,pad_k", _per_pair(VARLEN))
def test_varlen_isolation(ops, lens_q, lens_k, Hq, Hk, Dqk, Dv, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k):
    for b in range(len(lens_q)):
        _run_varlen(lens_q, lens_k, Hq, Hk, Dqk, Dv, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k, seed=b, poison=b)


@pytest.mark.parametrize("D", [64, 128])
def test_varlen_70000_one_token_sequences(ops, D):
    """More sequences than a grid dimension other than x can hold (65,535)."""
    from d9d_b200.kernel.flash_attn import flash_attn_varlen_func

    n, Hq, Hk = 70_000, 2, 1
    sc = 1.0 / math.sqrt(D)
    gen = torch.Generator().manual_seed(7)
    q, k, v, dout = make_inputs(1, 1, Hq, Hk, D, scale=sc, B=n, gen=gen, device="cuda")
    dl = torch.randn(Hq, n, generator=gen).cuda()
    cu = torch.arange(n + 1, dtype=torch.int32, device="cuda")
    qi, ki, vi = (t.reshape(n, -1, D).clone().requires_grad_() for t in (q, k, v))
    s = _sink([8.0, -8.0], Hq)
    out, lse = flash_attn_varlen_func(qi, ki, vi, cu, cu, 1, 1, causal=True, learnable_sink=s, softcap=7.0, return_lse=True)
    torch.autograd.backward([out, lse], [dout.reshape(n, Hq, D), dl])
    ref = fixed_reference(q, k, v, scale=sc, wl=-1, wr=0, softcap=7.0, sink=s.detach(), out=out.detach().view(n, 1, Hq, D),
                          dout=dout, dlse=dl.t().reshape(n, Hq, 1))
    got = {"out": out.view(n, 1, Hq, D), "lse": lse.t().reshape(n, Hq, 1), "dq": qi.grad.view(n, 1, Hq, D),
           "dk": ki.grad.view(n, 1, Hk, D), "dv": vi.grad.view(n, 1, Hk, D), "dsink": s.grad}
    _check(got, ref, f"{n} one-token sequences D={D}", (D, D))


@pytest.mark.parametrize("varlen", [False, True])
@pytest.mark.parametrize("Dqk,Dv", [P128, P192])
def test_backward_is_deterministic(ops, Dqk, Dv, varlen):
    """No atomics in the backward: two runs on the same inputs are bitwise equal."""
    from d9d_b200.kernel._native import native_ops

    Hq, Hk, sc = 8, 2, Dqk**-0.5
    lens = [300, 1, 517, 64] if varlen else [1024]
    total = sum(lens)
    q, k, v, dout = make_inputs(total, total, Hq, Hk, Dqk, Dv, scale=sc, gen=torch.Generator().manual_seed(4), device="cuda")
    if varlen:
        cu = torch.tensor([0] + [sum(lens[: i + 1]) for i in range(len(lens))], dtype=torch.int32, device="cuda")
        args = (cu, cu, max(lens), max(lens))
    else:
        q, k, v, dout = (t[None] for t in (q, k, v, dout))
        args = (None, None, 0, 0)
    out, lse = native_ops().flash_attn_fwd(q, k, v, sc, -1, 0, 0.0, None, *args)
    assert out.shape == (*q.shape[:-1], Dv)
    runs = [native_ops().flash_attn_bwd(dout, q, k, v, out, lse, sc, -1, 0, 0.0, *args, None)[:3] for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert runs[0][0].shape == q.shape and runs[0][1].shape == k.shape and runs[0][2].shape == v.shape


@pytest.mark.parametrize("dqk,dv", [(192, 192), (128, 64), (64, 128), (256, 128), (192, 64)])
def test_unsupported_head_dims_raise_in_the_binding(ops, dqk, dv):
    """Pairs the kernels are not built for are refused before any launch."""
    from d9d_b200.kernel._native import native_ops
    from d9d_b200.kernel.flash_attn.native import native_supported

    q = torch.randn(1, 64, 2, dqk, device="cuda").bfloat16()
    k = torch.randn(1, 64, 2, dqk, device="cuda").bfloat16()
    v = torch.randn(1, 64, 2, dv, device="cuda").bfloat16()
    assert not native_supported(q, k, v)
    with pytest.raises(RuntimeError, match="head dims"):
        native_ops().flash_attn_fwd(q, k, v, 0.1, -1, 0, 0.0, None, None, None, 0, 0)
    out = torch.zeros(1, 64, 2, dv, device="cuda").bfloat16()
    lse = torch.zeros(1, 2, 64, device="cuda")
    with pytest.raises(RuntimeError, match="head dims"):
        native_ops().flash_attn_bwd(out, q, k, v, out, lse, 0.1, -1, 0, 0.0, None, None, 0, 0, None)
    torch.cuda.synchronize()


def test_mismatched_shapes_raise_in_the_binding(ops):
    from d9d_b200.kernel._native import native_ops

    q = torch.randn(1, 64, 2, 192, device="cuda").bfloat16()
    k = torch.randn(1, 64, 2, 192, device="cuda").bfloat16()
    v = torch.randn(1, 64, 2, 128, device="cuda").bfloat16()
    with pytest.raises(RuntimeError, match="k and v"):
        native_ops().flash_attn_fwd(q, k, v[:, :32], 0.1, -1, 0, 0.0, None, None, None, 0, 0)
    with pytest.raises(RuntimeError, match="q and k"):
        native_ops().flash_attn_fwd(q, k[..., :128].contiguous(), v, 0.1, -1, 0, 0.0, None, None, None, 0, 0)
    out, lse = native_ops().flash_attn_fwd(q, k, v, 0.1, -1, 0, 0.0, None, None, None, 0, 0)
    with pytest.raises(RuntimeError, match="dout / out"):
        native_ops().flash_attn_bwd(q, q, k, v, out, lse, 0.1, -1, 0, 0.0, None, None, 0, 0, None)


def _assert_close_to_max(name, got, ref, tol):
    """max |got - ref| <= tol max |ref|."""
    got, ref = got.float(), ref.float()
    scale = float(ref.abs().max()) + 1e-6
    err = float((got - ref).abs().max()) / scale
    assert err < tol, f"{name}: max err {err:.4f} (relative to max |ref| {scale:.3g})"


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
    _assert_close_to_max("out", out, ref_out, tol=1e-3)
    torch.testing.assert_close(lse, torch.cat(lses, dim=-1), rtol=1e-4, atol=1e-4)
    for name, a, t in zip(("dq", "dk", "dv"), got, (q, k, v)):
        _assert_close_to_max(name, a, t.grad, tol=1e-3)


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

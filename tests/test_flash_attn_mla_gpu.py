"""Native wgmma flash attention at the multi-head latent attention head dims, (Dqk, Dv) = (192, 128): forward, delta
pre-pass, dK/dV and dQ kernels against the fp64 reference and per-element error bound of ``tests/attention_reference_mla.py``
(out, lse, dq, dk, dv and dsink of every case).

The matrix covers sequence lengths on the 128-row forward tile edges and on the streamed backward tile edges (32 rows in
dK/dV, 64 in dQ at these dims); Sq > Sk causal; windows left-only, right-only and (0, 0); GQA groups 1 and 4; soft-cap,
sinks, a nonzero dlse and an explicit softmax_scale; B = 3; packed batches with cu_seqlens_q != cu_seqlens_k, empty
sequences and rows outside every sequence.  Rows outside the sequence under test are NaN in the isolation cases.

Set D9D_ATTN_REPORT=<file> to write the worst err/bound per output tensor as JSON.
"""

import json
import math
import os

import pytest
import torch

from tests.attention_reference_mla import assert_lse_within, assert_within, batch_reference, fixed_reference, make_inputs

pytestmark = pytest.mark.gpu

DQK, DV = 192, 128
_worst: dict[str, float] = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("D9D_ATTN_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump({"head_dims": [DQK, DV], "worst_err_over_bound": _worst}, f, indent=1)


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    return _ops.load()


def _check(got: dict, ref: dict, what: str, rows: dict | None = None) -> None:
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
        _worst[name] = max(_worst.get(name, 0.0), r)


def _sink(pattern, Hq):
    if pattern is None:
        return None
    return torch.tensor([pattern[h % len(pattern)] for h in range(Hq)], device="cuda", dtype=torch.float32).requires_grad_()


def _api_window(wl, wr, seed):
    causal = wr == 0 and seed % 2 == 0
    return causal, (wl if wl >= 0 else None, None if causal else (wr if wr >= 0 else None))


def _run_fixed(B, Sq, Sk, Hq, Hk, wl, wr, softcap=0.0, sink=None, dlse=False, scale=None, seed=0, poison=None):
    from d9d_b200.kernel.flash_attn import flash_attn_func

    sc = scale if scale is not None else 1.0 / math.sqrt(DQK)
    gen = torch.Generator().manual_seed(seed)
    q, k, v, dout = make_inputs(Sq, Sk, Hq, Hk, DQK, DV, scale=sc, B=B, gen=gen, device="cuda")
    dl = torch.randn(B, Hq, Sq, generator=gen).cuda() if dlse else None
    qi, ki, vi, doi = q.clone(), k.clone(), v.clone(), dout.clone()
    if poison is not None:
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
    _check(got, ref, f"B={B} Sq={Sq} Sk={Sk} Hq={Hq} Hk={Hk} w=({wl},{wr}) cap={softcap} sink={sink}", rows)
    return got


FIXED = [
    # B, Sq, Sk, Hq, Hk, wl, wr, softcap, sink, dlse, scale
    (1, 1, 1, 2, 1, -1, -1, 0.0, None, False, None),
    (1, 31, 31, 2, 2, -1, 0, 0.0, None, False, None),
    (1, 33, 33, 4, 1, -1, -1, 0.0, None, True, None),
    (1, 63, 63, 2, 2, -1, 0, 0.0, None, False, None),
    (1, 64, 64, 4, 1, -1, -1, 0.0, None, True, None),
    (1, 65, 65, 2, 1, -1, 0, 0.0, [8.0, -8.0], False, None),
    (1, 97, 97, 2, 2, -1, 0, 0.0, None, False, None),
    (1, 127, 127, 2, 2, -1, 0, 0.0, None, False, None),
    (1, 128, 128, 2, 2, -1, -1, 0.0, None, True, None),
    (1, 129, 129, 4, 1, -1, 0, 0.0, None, False, None),
    (1, 255, 255, 4, 1, -1, -1, 0.0, None, False, None),
    (1, 256, 256, 2, 2, 128, 0, 0.0, None, False, None),
    (1, 257, 257, 2, 2, 127, -1, 0.0, None, False, None),   # left-only window
    (1, 257, 257, 2, 1, 129, 0, 0.0, None, True, None),
    (1, 200, 200, 2, 2, 0, 0, 0.0, None, False, None),      # window (0, 0)
    (1, 200, 200, 2, 2, -1, 5, 0.0, None, False, None),     # right-only window
    (1, 257, 129, 2, 1, -1, 0, 0.0, None, False, None),     # causal Sq > Sk
    (1, 257, 129, 2, 1, -1, 0, 0.0, [8.0, -8.0], True, None),
    (1, 129, 257, 2, 2, 64, 0, 0.0, None, False, None),
    (1, 257, 257, 4, 1, 128, 0, 5.0, None, False, None),
    (1, 200, 200, 2, 2, -1, 0, 10.0, [8.0, -8.0], True, None),
    (1, 65, 65, 2, 2, 0, 0, 0.0, [125.0, 125.0], True, None),
    (1, 200, 200, 4, 1, -1, 0, 0.0, None, False, 0.05),
    (3, 200, 200, 4, 1, -1, 0, 7.0, [8.0, -8.0], True, None),
    (1, 8192, 8192, 1, 1, -1, 0, 0.0, None, False, None),
]


@pytest.mark.parametrize("B,Sq,Sk,Hq,Hk,wl,wr,softcap,sink,dlse,scale", FIXED)
def test_fixed_length_192_128(ops, B, Sq, Sk, Hq, Hk, wl, wr, softcap, sink, dlse, scale):
    _run_fixed(B, Sq, Sk, Hq, Hk, wl, wr, softcap, sink, dlse, scale, seed=Sq * 31 + Sk + Hq)


@pytest.mark.parametrize("poison", [0, 1, 2])
def test_fixed_batch_isolation_192_128(ops, poison):
    _run_fixed(3, 200, 200, 4, 1, 100, 0, 5.0, [8.0], True, None, seed=3, poison=poison)


def _run_varlen(lens_q, lens_k, Hq, Hk, wl, wr, softcap=0.0, sink=None, dlse=False, lead=0, pad_q=0, pad_k=0, seed=0,
                poison=None):
    from d9d_b200.kernel.flash_attn import flash_attn_varlen_func

    sc = 1.0 / math.sqrt(DQK)
    cu_q = [lead] + [lead + sum(lens_q[: i + 1]) for i in range(len(lens_q))]
    cu_k = [0] + [sum(lens_k[: i + 1]) for i in range(len(lens_k))]
    total_q, total_k = cu_q[-1] + pad_q, cu_k[-1] + pad_k
    gen = torch.Generator().manual_seed(seed)
    q, k, v, dout = make_inputs(total_q, total_k, Hq, Hk, DQK, DV, scale=sc, gen=gen, device="cuda")
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
    _check(got, ref, f"varlen q={lens_q} k={lens_k} w=({wl},{wr}) cap={softcap} sink={sink} poison={poison}", rows)
    return got


VARLEN = [
    # lens_q, lens_k, Hq, Hk, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k
    ([1, 63, 129, 64], [1, 200, 129, 300], 4, 1, -1, 0, 7.0, [8.0, -8.0], True, 0, 0, 0),  # q: suffix of a longer k
    ([70, 129, 20], [150, 60, 257], 2, 1, 128, 0, 0.0, None, False, 0, 0, 0),
    ([0, 65, 0, 127, 3], [0, 0, 64, 128, 257], 2, 2, -1, 0, 5.0, [8.0], True, 3, 5, 7),  # empty q / k / both, padding
    ([31, 33, 63, 65, 127, 129, 255, 257], [31, 33, 63, 65, 127, 129, 255, 257], 4, 1, 127, -1, 0.0, [-8.0], False, 0, 0, 0),
    ([100, 37], [100, 37], 2, 2, -1, -1, 10.0, None, True, 0, 61, 13),
]


@pytest.mark.parametrize("lens_q,lens_k,Hq,Hk,wl,wr,softcap,sink,dlse,lead,pad_q,pad_k", VARLEN)
def test_varlen_192_128(ops, lens_q, lens_k, Hq, Hk, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k):
    _run_varlen(lens_q, lens_k, Hq, Hk, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k, seed=len(lens_q) + wl)


@pytest.mark.parametrize("case", [0, 2, 4])
def test_varlen_isolation_192_128(ops, case):
    lens_q, lens_k, Hq, Hk, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k = VARLEN[case]
    for b in range(len(lens_q)):
        _run_varlen(lens_q, lens_k, Hq, Hk, wl, wr, softcap, sink, dlse, lead, pad_q, pad_k, seed=b, poison=b)


@pytest.mark.parametrize("varlen", [False, True])
def test_backward_is_deterministic_192_128(ops, varlen):
    from d9d_b200.kernel._native import native_ops

    Hq, Hk, sc = 8, 2, DQK**-0.5
    lens = [300, 1, 517, 64] if varlen else [1024]
    total = sum(lens)
    q, k, v, dout = make_inputs(total, total, Hq, Hk, DQK, DV, scale=sc, gen=torch.Generator().manual_seed(4), device="cuda")
    if varlen:
        cu = torch.tensor([0] + [sum(lens[: i + 1]) for i in range(len(lens))], dtype=torch.int32, device="cuda")
        args = (cu, cu, max(lens), max(lens))
    else:
        q, k, v, dout = (t[None] for t in (q, k, v, dout))
        args = (None, None, 0, 0)
    out, lse = native_ops().flash_attn_fwd(q, k, v, sc, -1, 0, 0.0, None, *args, 0)
    assert out.shape == (*q.shape[:-1], DV)
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
        native_ops().flash_attn_fwd(q, k, v, 0.1, -1, 0, 0.0, None, None, None, 0, 0, 0)
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
        native_ops().flash_attn_fwd(q, k, v[:, :32], 0.1, -1, 0, 0.0, None, None, None, 0, 0, 0)
    with pytest.raises(RuntimeError, match="q and k"):
        native_ops().flash_attn_fwd(q, k[..., :128].contiguous(), v, 0.1, -1, 0, 0.0, None, None, None, 0, 0, 0)
    out, lse = native_ops().flash_attn_fwd(q, k, v, 0.1, -1, 0, 0.0, None, None, None, 0, 0, 0)
    with pytest.raises(RuntimeError, match="dout / out"):
        native_ops().flash_attn_bwd(q, q, k, v, out, lse, 0.1, -1, 0, 0.0, None, None, 0, 0, None)

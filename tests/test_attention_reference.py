"""Self-test of the fp64 reference / error bound that the flash attention kernel tests rely on: an fp32 emulation of the
kernels' algorithm must pass it, and each fault a broken kernel could have must exceed it, at the shapes and inputs the
GPU tests use: equal head dims 64 and 128, and separate qk and v head dims (192, 128), where a kernel has more ways to
mix up the two widths."""

import math

import pytest
import torch

from tests.attention_reference import batch_reference, fixed_reference, lse_err_ratio, make_inputs, visible
from tests.gemm_reference import err_ratio

L2E = math.log2(math.e)


def _pitch(x: torch.Tensor, pitch: int) -> torch.Tensor:
    """[S, H, Dv] read as if its rows were ``pitch`` elements apart (past the end of the buffer: zeros)."""
    S, H, Dv = x.shape
    flat = torch.zeros(S * H * pitch, dtype=x.dtype)
    flat[: x.numel()] = x.reshape(-1)
    return flat.view(S, H, pitch)[..., :Dv]


def emulate(q, k, v, *, scale, wl=-1, wr=-1, softcap=0.0, sink=None, dout=None, dlse=None, fault=None):
    """fp32 emulation of one sequence through the kernels with q / k [S, H, Dqk] and v / dout [S, H, Dv]: 128-key tiles
    with an online softmax in the log2 domain, P rounded to bf16 for O += P V, the sink folded into the max at the end;
    backward with P recomputed from the lse, Delta from the bf16 O over the Dv columns, dS rounded to bf16, fp32
    accumulation of dQ / dK (Dqk columns) and dV (Dv columns).  ``fault`` injects one bug."""
    Sq, Hq, Dqk = q.shape
    Sk, Hk, Dv = k.shape[0], k.shape[1], v.shape[2]
    g = Hq // Hk
    hmap = torch.arange(Hq) % Hk if fault == "gqa_mod" else torch.arange(Hq) // g
    if fault == "v_pitch":
        v = _pitch(v, Dqk)
    if fault == "do_pitch" and dout is not None:
        dout = _pitch(dout, Dqk)
    qf = q.float().permute(1, 0, 2)
    kf, vf = k.float().permute(1, 0, 2)[hmap], v.float().permute(1, 0, 2)[hmap]
    keep = visible(Sq, Sk, wl + (fault == "left"), wr + (fault == "right"))
    if fault == "diagonal":
        keep &= torch.arange(Sk)[None] < torch.arange(Sq)[:, None] + (Sk - Sq)
    if fault == "last_key":
        keep[:, Sk - 1] = False
    s = qf[..., : Dqk - 64] @ kf[..., : Dqk - 64].transpose(1, 2) if fault == "no_rope" else qf @ kf.transpose(1, 2)
    if softcap:
        t = torch.tanh(s * (scale / softcap))
        x = softcap * t * L2E
    else:
        x = s * (scale * L2E)
    x = x.masked_fill(~keep, -math.inf)
    m = torch.full((Hq, Sq, 1), -math.inf)
    l = torch.zeros(Hq, Sq, 1)
    o = torch.zeros(Hq, Sq, Dv)
    for j in range(0, Sk, 128):
        if fault == "skip_tile" and j == 128:
            continue
        xs = x[:, :, j : j + 128]
        m_new = torch.maximum(m, xs.amax(-1, keepdim=True))
        alpha = torch.where(m_new == -math.inf, 1.0, torch.exp2(m - m_new))
        pt = torch.exp2(xs - torch.where(m_new == -math.inf, 0.0, m_new))
        l = l * alpha + pt.sum(-1, keepdim=True)
        if fault != "no_rescale":
            o = o * alpha
        o = o + pt.bfloat16().float() @ vf[:, j : j + 128]
        m = m_new
    o_scale = torch.ones_like(l)
    if sink is not None and fault != "sink_ignored":
        s2 = (sink.float() * L2E).view(Hq, 1, 1).expand_as(m)
        up = s2 > m
        o_scale = torch.where(up, torch.exp2(m - s2), 1.0)
        l = torch.where(up, l * o_scale + 1.0, l + torch.where(m == -math.inf, 0.0, torch.exp2(s2 - m)))
        m = torch.where(up, s2, m)
    m_safe = torch.where(m == -math.inf, 0.0, m)
    out = torch.where(l > 0, o * o_scale / l, 0.0).bfloat16()
    lse = torch.where(l > 0, (m_safe + torch.log2(l)) / L2E, -math.inf)
    res = {"out": out.permute(1, 0, 2), "lse": lse[..., 0]}
    if dout is None:
        return res
    do = dout.float().permute(1, 0, 2)
    n_delta = 64 if fault == "delta_64" else Dv
    delta = (do[..., :n_delta] * out.float()[..., :n_delta]).sum(-1, keepdim=True)
    if dlse is not None and fault != "dlse_ignored":
        delta = delta - dlse.float()[..., None]
    lse2 = torch.where(lse == -math.inf, math.inf, lse * L2E)
    p = torch.where(keep, torch.exp2(x - lse2), 0.0)
    dp = do @ vf.transpose(1, 2)
    ds = p * (dp - delta)
    if softcap and fault != "capd_dropped":
        ds = ds * (1 - t * t)
    pb, dsb = p.bfloat16().float(), ds.bfloat16().float()
    dk_scale = 1.0 if fault == "dk_unscaled" else scale
    dq = scale * (dsb @ kf)
    dk_h, dv_h = dsb.transpose(1, 2) @ qf, pb.transpose(1, 2) @ do
    dk = torch.zeros(Hk, Sk, Dqk).index_add_(0, hmap, dk_h) * dk_scale
    dv = torch.zeros(Hk, Sk, Dv).index_add_(0, hmap, dv_h)
    if fault == "dq_partial":
        dq[..., Dv:] = 0.0
    if fault == "dk_partial":
        dk[..., Dv:] = 0.0
    res.update(dq=dq.bfloat16().permute(1, 0, 2), dk=dk.bfloat16().permute(1, 0, 2), dv=dv.bfloat16().permute(1, 0, 2))
    if sink is not None:
        ps = torch.where(lse == -math.inf, 0.0, torch.exp(sink.float().view(Hq, 1, 1) - lse))
        res["dsink"] = -(ps * delta).sum((1, 2))
    return res


def _run(Sq, Sk, Hq, Hk, Dqk, Dv, *, wl=-1, wr=-1, softcap=0.0, sink=None, with_dlse=False, fault=None, seed=0):
    scale = 1.0 / math.sqrt(Dqk)
    gen = torch.Generator().manual_seed(seed)
    q, k, v, dout = make_inputs(Sq, Sk, Hq, Hk, Dqk, Dv, scale=scale, gen=gen)
    sink_t = None if sink is None else torch.tensor(sink, dtype=torch.float32)
    dlse = torch.randn(Hq, Sq, generator=gen) if with_dlse else None
    kw = dict(scale=scale, wl=wl, wr=wr, softcap=softcap, sink=sink_t)
    got = emulate(q, k, v, dout=dout, dlse=dlse, fault=fault, **kw)
    ref = batch_reference(q, k, v, [0, Sq], [0, Sk], out=got["out"], dout=dout, dlse=dlse, **kw)
    r = {}
    for name, (want, bound) in ref.items():
        assert got[name].shape == want.shape, (name, got[name].shape, want.shape)
        r[name] = lse_err_ratio(got[name], want, bound) if name == "lse" else err_ratio(got[name], want, bound)
    return r


MLA = (192, 128)  # (Dqk, Dv) of multi-head latent attention

ACCEPT = [
    # Sq, Sk, Hq, Hk, D, wl, wr, softcap, sink, dlse
    (257, 257, 4, 2, 64, -1, -1, 0.0, None, False),
    (257, 257, 2, 2, 128, -1, 0, 0.0, [8.0, -8.0], True),
    (129, 255, 4, 1, 128, 128, 0, 5.0, None, False),
    (255, 129, 2, 1, 64, -1, 0, 10.0, [8.0, 0.0], True),
    (200, 200, 2, 2, 64, 127, 3, 0.0, None, True),
    (65, 65, 2, 2, 128, 0, 0, 0.0, [100.0, -8.0], False),
]


@pytest.mark.parametrize("dims", [None, MLA], ids=["D", "192-128"])
@pytest.mark.parametrize("Sq,Sk,Hq,Hk,D,wl,wr,softcap,sink,dlse", ACCEPT)
def test_accepts_kernel_emulation(Sq, Sk, Hq, Hk, D, wl, wr, softcap, sink, dlse, dims):
    """Each case at its listed head dim D = Dqk = Dv, and at (192, 128)."""
    Dqk, Dv = dims or (D, D)
    r = _run(Sq, Sk, Hq, Hk, Dqk, Dv, wl=wl, wr=wr, softcap=softcap, sink=sink, with_dlse=dlse)
    assert all(x <= 1.0 for x in r.values()), r


FAULTS = [
    ("left", dict(wl=128, wr=-1)),
    ("right", dict(wl=-1, wr=5)),
    ("diagonal", dict(wr=0)),
    ("last_key", dict()),
    ("sink_ignored", dict(sink=[8.0, 8.0, -8.0, 8.0])),
    ("capd_dropped", dict(softcap=10.0)),
    ("dk_unscaled", dict()),
    ("dlse_ignored", dict(with_dlse=True)),
    ("skip_tile", dict()),
    ("no_rescale", dict()),
    ("gqa_mod", dict()),
]
UNEQUAL_DIMS_FAULTS = [
    ("no_rope", dict()),          # S without the last 64-column box of Q and K
    ("v_pitch", dict()),          # V read at the Dqk row pitch
    ("do_pitch", dict()),         # dO read at the Dqk row pitch
    ("delta_64", dict()),         # Delta summed over the first 64 of the Dv columns
    ("dk_partial", dict()),       # dK written for the first Dv columns only
    ("dq_partial", dict()),       # dQ written for the first Dv columns only
]
FAULT_CASES = ([(f, kw, (D, D)) for D in (64, 128) for f, kw in FAULTS]
               + [(f, kw, MLA) for f, kw in UNEQUAL_DIMS_FAULTS + FAULTS])


@pytest.mark.parametrize("fault,kw,dims", FAULT_CASES,
                         ids=[f"{f}-{dqk}" if dqk == dv else f"{f}-{dqk}-{dv}" for f, _, (dqk, dv) in FAULT_CASES])
def test_rejects_fault(fault, kw, dims):
    assert max(_run(257, 257, 4, 2, *dims, **kw).values()) <= 1.0  # the same case without the fault passes
    r = _run(257, 257, 4, 2, *dims, fault=fault, **kw)
    assert max(r.values()) > 1.0, r


def test_reference_shapes_follow_each_head_dim():
    """out / dv take the v head dim, dq / dk the qk head dim, packed and fixed-length alike."""
    gen = torch.Generator().manual_seed(1)
    q, k, v, dout = make_inputs(20, 24, 4, 2, *MLA, scale=0.1, B=2, gen=gen)
    assert v.shape == (2, 24, 2, 128) and dout.shape == (2, 20, 4, 128)
    out = torch.zeros(2, 20, 4, 128).bfloat16()
    f = fixed_reference(q, k, v, scale=0.1, wr=0, out=out, dout=dout)
    assert f["out"][0].shape == (2, 20, 4, 128) and f["dv"][0].shape == (2, 24, 2, 128)
    assert f["dq"][0].shape == (2, 20, 4, 192) and f["dk"][0].shape == (2, 24, 2, 192)


def test_fixed_batch_folds_into_heads():
    """fixed_reference (batch folded into the heads) equals batch_reference over the same packed sequences."""
    B, S, Hq, Hk, D = 3, 70, 4, 2, 64
    gen = torch.Generator().manual_seed(5)
    q, k, v, dout = make_inputs(S, S, Hq, Hk, D, scale=0.125, B=B, gen=gen)
    sink = torch.tensor([1.0, -2.0, 8.0, 0.5])
    dlse = torch.randn(B, Hq, S, generator=gen)
    kw = dict(scale=0.125, wl=20, wr=0, softcap=7.0, sink=sink)
    f = fixed_reference(q, k, v, out=q, dout=dout, dlse=dlse, **kw)
    cu = [b * S for b in range(B + 1)]
    pk = lambda t: t.reshape(B * S, *t.shape[2:])  # noqa: E731
    p = batch_reference(pk(q), pk(k), pk(v), cu, cu, out=pk(q), dout=pk(dout), dlse=dlse.permute(1, 0, 2).reshape(Hq, B * S), **kw)
    for name in ("out", "dq", "dk", "dv"):
        torch.testing.assert_close(pk(f[name][0]), p[name][0], rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(pk(f[name][1]), p[name][1], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(f["lse"][0].permute(1, 0, 2).reshape(Hq, B * S), p["lse"][0])
    torch.testing.assert_close(f["dsink"][0], p["dsink"][0], rtol=1e-12, atol=1e-12)


def test_packed_rows_outside_sequences_must_be_zero():
    Hq, Hk, D = 2, 1, 64
    gen = torch.Generator().manual_seed(2)
    q, k, v, dout = make_inputs(40, 40, Hq, Hk, D, scale=0.125, gen=gen)
    cu_q, cu_k = [3, 10, 10, 30], [0, 0, 25, 36]  # rows 0-2 and 30-39 of q and 36-39 of k lie outside every sequence
    ref = batch_reference(q, k, v, cu_q, cu_k, scale=0.125, out=q, dout=dout)
    assert bool((ref["lse"][0][:, :3] == -math.inf).all()) and bool((ref["lse"][0][:, 30:] == -math.inf).all())
    for name, rows in (("out", [0, 2, 30, 39]), ("dq", [0, 35]), ("dk", [36, 39]), ("dv", [37])):
        want, bound = ref[name]
        assert bool((bound[rows] == 0).all()) and bool((want[rows] == 0).all())
    # sequence 0 has queries but no key: out = dq = 0 (up to the underflow floor), lse = -inf
    for name in ("out", "dq"):
        assert bool((ref[name][0][3:10] == 0).all()) and bool((ref[name][1][3:10] <= 2.0**-100).all())
    assert bool((ref["lse"][0][:, 3:10] == -math.inf).all())

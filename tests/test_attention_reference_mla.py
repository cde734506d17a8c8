"""Self-test of the fp64 reference / error bound at unequal head dims (``tests/attention_reference_mla.py``), (Dqk, Dv) =
(192, 128) as in multi-head latent attention: at equal dims it matches ``tests/attention_reference.py`` bitwise; an fp32
emulation of the kernels' algorithm must pass it, and each fault a kernel with separate qk and v head
dims could have must exceed it."""

import math

import pytest
import torch

from tests.attention_reference import lse_err_ratio, visible
from tests.attention_reference_mla import batch_reference, fixed_reference, make_inputs
from tests.gemm_reference import err_ratio
from tests.test_attention_reference import ACCEPT, FAULTS

L2E = math.log2(math.e)
DQK, DV = 192, 128


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


def _run(Sq, Sk, Hq, Hk, *, wl=-1, wr=-1, softcap=0.0, sink=None, with_dlse=False, fault=None, seed=0):
    scale = 1.0 / math.sqrt(DQK)
    gen = torch.Generator().manual_seed(seed)
    q, k, v, dout = make_inputs(Sq, Sk, Hq, Hk, DQK, DV, scale=scale, gen=gen)
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


@pytest.mark.parametrize("Sq,Sk,Hq,Hk,D,wl,wr,softcap,sink,dlse", ACCEPT)
def test_accepts_kernel_emulation_at_192_128(Sq, Sk, Hq, Hk, D, wl, wr, softcap, sink, dlse):
    """The window, sink, soft-cap and dlse settings of the equal-dims self-test, at (192, 128)."""
    del D
    r = _run(Sq, Sk, Hq, Hk, wl=wl, wr=wr, softcap=softcap, sink=sink, with_dlse=dlse)
    assert all(x <= 1.0 for x in r.values()), r


MLA_FAULTS = [
    ("no_rope", dict()),          # S without the last 64-column box of Q and K
    ("v_pitch", dict()),          # V read at the Dqk row pitch
    ("do_pitch", dict()),         # dO read at the Dqk row pitch
    ("delta_64", dict()),         # Delta summed over the first 64 of the Dv columns
    ("dk_partial", dict()),       # dK written for the first Dv columns only
    ("dq_partial", dict()),       # dQ written for the first Dv columns only
]


@pytest.mark.parametrize("fault,kw", MLA_FAULTS + FAULTS, ids=[f for f, _ in MLA_FAULTS + FAULTS])
def test_rejects_fault_at_192_128(fault, kw):
    assert max(_run(257, 257, 4, 2, **kw).values()) <= 1.0  # the same case without the fault passes
    r = _run(257, 257, 4, 2, fault=fault, **kw)
    assert max(r.values()) > 1.0, r


def test_reference_shapes_follow_each_head_dim():
    """out / dv take the v head dim, dq / dk the qk head dim, packed and fixed-length alike."""
    gen = torch.Generator().manual_seed(1)
    q, k, v, dout = make_inputs(20, 24, 4, 2, DQK, DV, scale=0.1, B=2, gen=gen)
    assert v.shape == (2, 24, 2, DV) and dout.shape == (2, 20, 4, DV)
    out = torch.zeros(2, 20, 4, DV).bfloat16()
    f = fixed_reference(q, k, v, scale=0.1, wr=0, out=out, dout=dout)
    assert f["out"][0].shape == (2, 20, 4, DV) and f["dv"][0].shape == (2, 24, 2, DV)
    assert f["dq"][0].shape == (2, 20, 4, DQK) and f["dk"][0].shape == (2, 24, 2, DQK)


@pytest.mark.parametrize("packed", [False, True])
def test_equal_dims_match_the_equal_dims_reference_bitwise(packed):
    """At Dqk == Dv the separate-dims reference computes exactly what tests/attention_reference.py computes."""
    from tests import attention_reference as eq

    B, S, Hq, Hk, D = 2, 150, 4, 2, 64
    gen = torch.Generator().manual_seed(9)
    q, k, v, dout = eq.make_inputs(S, S, Hq, Hk, D, scale=0.125, B=B, gen=gen)
    sink = torch.tensor([1.0, -2.0, 8.0, 0.5])
    dlse = torch.randn(B, Hq, S, generator=gen)
    kw = dict(scale=0.125, wl=40, wr=0, softcap=7.0, sink=sink)
    if packed:
        cu = [0, 100, 100, B * S - 7]
        pk = lambda t: t.reshape(B * S, *t.shape[2:])  # noqa: E731
        args = (pk(q), pk(k), pk(v), cu, cu)
        kw.update(out=pk(q), dout=pk(dout), dlse=dlse.permute(1, 0, 2).reshape(Hq, B * S))
        want, got = eq.batch_reference(*args, **kw), batch_reference(*args, **kw)
    else:
        kw.update(out=q, dout=dout, dlse=dlse)
        want, got = eq.fixed_reference(q, k, v, **kw), fixed_reference(q, k, v, **kw)
    assert want.keys() == got.keys()
    for name in want:
        for a, b in zip(want[name], got[name]):
            assert torch.equal(a, b), name

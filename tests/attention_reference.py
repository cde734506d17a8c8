"""fp64 reference and per-element error bound for the wgmma flash attention kernels (forward, delta pre-pass, dK/dV and dQ).
Pure torch: works on CPU tensors (self-test) and CUDA tensors alike.

Visibility (``d9d_ops.h``): key k of a sequence sees query q iff q + off - wl <= k <= q + off + wr, off = Sk - Sq, where a
negative wl / wr is unbounded.  Scores x = scale q.k, or cap tanh(scale q.k / cap) with a soft-cap; an optional per-head
sink joins the softmax denominator.

q and k have Dqk columns, v and out Dv (multi-head latent attention runs at (192, 128)); dq and dk have Dqk columns, dv Dv.
Each sum over a head dim below runs over its own width.

Error sources of the kernels, all taken from the tensors actually passed to them:

* S = Q K^T accumulates over Dqk in fp32:  |dx_ij| <= scale c_k(Dqk) |q_i|.|k_j|;  fast tanh adds cap 2^-10.9,
  and the log2-domain arithmetic / ex2 a few fp32 ulps of |x| and of the row max.  eps_i is the largest of these over the
  visible keys of row i; P_ij = exp(x_ij - lse_i) is then off by at most exp(2 eps_i) relatively (forward).
* P (and dS) are rounded to bf16 before they enter the second GEMM, whose fp32 accumulation runs over Sk (forward, dQ) or
  g Sq (dK / dV, g = Hq / Hk).
* The backward recomputes P from the forward's lse, so the lse bound joins eps_i there; dP = dO V^T accumulates over
  Dv; Delta = dO.O - dlse, also over Dv, is taken from the bf16 O the backward is given.
* Every bf16 output is rounded once more (2^-8 relative).  Results below 2^-100 may flush to zero.
"""

from __future__ import annotations

import math

import torch

from tests.gemm_reference import U_BF16, assert_within, ck, err_ratio  # noqa: F401  (re-exported for the tests)

U_F32 = 2.0**-24
ULP_MATH = 2.0**-21    # relative error of ex2 / lg2 / rcp (approx) and of the fp32 roundings around them
TANH_REL = 2.0**-10.9  # relative error of tanh.approx.f32
TINY = 2.0**-100       # underflow: fp32 flush-to-zero below 2^-126


def visible(Sq: int, Sk: int, wl: int, wr: int, device=None) -> torch.Tensor:
    """[Sq, Sk] bool: key k visible to query q."""
    q = torch.arange(Sq, device=device)[:, None] + (Sk - Sq)
    k = torch.arange(Sk, device=device)[None, :]
    keep = torch.ones(Sq, Sk, dtype=torch.bool, device=device)
    if wl >= 0:
        keep &= k >= q - wl
    if wr >= 0:
        keep &= k <= q + wr
    return keep


def _heads(x: torch.Tensor, Hq: int) -> torch.Tensor:
    """[S, Hk, D] -> fp64 [Hq, S, D] with query head h reading kv head h // (Hq / Hk)."""
    g = Hq // x.shape[1]
    return x.double().permute(1, 0, 2).repeat_interleave(g, dim=0)


def _group_sum(x: torch.Tensor, Hk: int) -> torch.Tensor:
    """[Hq, S, D] -> [S, Hk, D], summing the query heads of each kv head."""
    Hq, S, D = x.shape
    return x.view(Hk, Hq // Hk, S, D).sum(1).permute(1, 0, 2)


def sequence_reference(q, k, v, *, scale: float, wl: int = -1, wr: int = -1, softcap: float = 0.0, sink=None, out=None,
                       dout=None, dlse=None, chunk: int = 1024) -> dict[str, tuple[torch.Tensor, torch.Tensor]]:
    """(reference, bound) per output for one sequence: q [Sq, Hq, Dqk], k [Sk, Hk, Dqk], v [Sk, Hk, Dv], sink [Hq] or None.

    Always ``out`` [Sq, Hq, Dv] and ``lse`` [Hq, Sq] (-inf where a row sees no key and there is no sink).  With ``dout``
    (and the bf16 ``out`` the backward is given, optional ``dlse`` [Hq, Sq]) also ``dq``, ``dk``, ``dv`` and, with a sink,
    ``dsink`` [Hq] (its fp32 sum over the whole batch is bounded by :func:`batch_reference`).  Rows are processed
    ``chunk`` queries at a time, so long sequences fit in memory."""
    Sq, Hq, Dqk = q.shape
    Sk, Hk, Dv = k.shape[0], k.shape[1], v.shape[2]
    dev = q.device
    kf, vf = _heads(k, Hq), _heads(v, Hq)
    kabs, vabs = kf.abs(), vf.abs()
    keep_all = visible(Sq, Sk, wl, wr, dev)
    sink64 = sink.double().view(Hq, 1) if sink is not None else None
    n_tiles = max(1, -(-Sk // 128))
    bwd = dout is not None
    res = {n: [] for n in ("out", "out_b", "lse", "lse_b", "dq", "dq_b")}
    if bwd:
        dk, dk_b = (torch.zeros(Hq, Sk, Dqk, dtype=torch.float64, device=dev) for _ in range(2))
        dv, dv_b = (torch.zeros(Hq, Sk, Dv, dtype=torch.float64, device=dev) for _ in range(2))
        dsink = torch.zeros(Hq, dtype=torch.float64, device=dev)
        dsink_b = torch.zeros(Hq, dtype=torch.float64, device=dev)
        dsink_abs = torch.zeros(Hq, dtype=torch.float64, device=dev)
    for i0 in range(0, Sq, chunk):
        i1 = min(Sq, i0 + chunk)
        keep = keep_all[i0:i1][None]                       # [1, n, Sk]
        qf = q[i0:i1].double().permute(1, 0, 2)            # [Hq, n, Dqk]
        s = scale * (qf @ kf.transpose(1, 2))
        s_err = scale * ck(Dqk) * (qf.abs() @ kabs.transpose(1, 2))
        if softcap:
            t = torch.tanh(s / softcap)
            x = softcap * t
            s_err = s_err + softcap * TANH_REL * t.abs()
        else:
            x = s
        x = x.masked_fill(~keep, -math.inf)
        m = x.amax(-1, keepdim=True) if Sk else torch.full((Hq, i1 - i0, 1), -math.inf, dtype=torch.float64, device=dev)
        if sink64 is not None:
            m = torch.maximum(m, sink64[:, :, None].expand_as(m))
        m_safe = torch.where(torch.isfinite(m), m, 0.0)
        e = torch.exp(x - m_safe)
        tot = e.sum(-1, keepdim=True)
        if sink64 is not None:
            tot = tot + torch.exp(sink64[:, :, None] - m_safe)
        lse = torch.where(tot > 0, m_safe + torch.log(tot), -math.inf)  # [Hq, n, 1]
        p = torch.where(tot > 0, e / tot.clamp_min(1e-300), 0.0)
        xv = torch.where(keep, x, 0.0)
        eps = torch.where(keep, s_err + ULP_MATH * (xv.abs() + m_safe.abs()), 0.0)
        eps = eps.amax(-1, keepdim=True) if Sk else torch.zeros_like(m)
        eta = torch.expm1(2 * eps) + ck(Sk) + ULP_MATH * (n_tiles + 2)  # relative error of P
        o = p @ vf
        a = p @ vabs
        res["out"].append(o)
        res["out_b"].append((1 + U_BF16) * ((eta + U_BF16 + ck(Sk)) * a) + U_BF16 * o.abs() + TINY)
        lse_b = eps + ck(Sk) + ULP_MATH * (n_tiles + 4 + lse.abs().nan_to_num(posinf=0, neginf=0))
        res["lse"].append(lse[..., 0])
        res["lse_b"].append(torch.where(torch.isfinite(lse), lse_b, 0.0)[..., 0])
        if not bwd:
            continue
        do = dout[i0:i1].double().permute(1, 0, 2)
        ob = out[i0:i1].double().permute(1, 0, 2)
        delta = (do * ob).sum(-1, keepdim=True)
        delta_err = ck(Dv) * (do.abs() * ob.abs()).sum(-1, keepdim=True) + 2 * U_F32 * delta.abs()
        if dlse is not None:
            dl = dlse[:, i0:i1].double()[..., None]
            delta = delta - dl
            delta_err = delta_err + 2 * U_F32 * (delta.abs() + dl.abs())
        dp = do @ vf.transpose(1, 2)
        dp_err = ck(Dv) * (do.abs() @ vabs.transpose(1, 2))
        dpd = dp - delta
        eta_b = torch.expm1(eps + torch.where(torch.isfinite(lse), lse_b, 0.0)) + ULP_MATH  # P recomputed from the lse
        cap_d = (1 - t * t) if softcap else 1.0
        cap_d_err = (2 * t.abs() * TANH_REL * t.abs()) if softcap else 0.0
        ds = p * dpd * cap_d
        ds_err = p * ((eta_b + 4 * U_F32) * dpd.abs() * cap_d + (1 + eta_b) * (dp_err + delta_err) * cap_d + dpd.abs() * cap_d_err)
        ds_rnd = ds_err + U_BF16 * (ds.abs() + ds_err)    # kernel's bf16 dS vs exact dS
        p_rnd = (eta_b + U_BF16 * (1 + eta_b)) * p         # kernel's bf16 P vs exact P
        dq = scale * (ds @ kf)
        res["dq"].append(dq)
        res["dq_b"].append((1 + U_BF16) * scale * ((ds_rnd + ck(Sk) * ds.abs()) @ kabs) * (1 + 2 * U_F32) + U_BF16 * dq.abs() + TINY)
        qabs, doabs = qf.abs(), do.abs()
        dk += scale * (ds.transpose(1, 2) @ qf)
        dk_b += scale * ((ds_rnd + ck(Sq * Hq // Hk) * ds.abs()).transpose(1, 2) @ qabs)
        dv += p.transpose(1, 2) @ do
        dv_b += (p_rnd + ck(Sq * Hq // Hk) * p).transpose(1, 2) @ doabs
        if sink64 is not None:
            ps = torch.where(torch.isfinite(lse), torch.exp(sink64[:, :, None] - lse), 0.0)  # [Hq, n, 1]
            dsink -= (ps * delta).sum((1, 2))
            lse_rel = torch.expm1(torch.where(torch.isfinite(lse), lse_b, 0.0)) + ULP_MATH
            dsink_b += (ps * (lse_rel * delta.abs() + (1 + lse_rel) * delta_err)).sum((1, 2))
            dsink_abs += (ps * delta.abs()).sum((1, 2))
    cat = {n: torch.cat(vals, dim=1) for n, vals in res.items() if vals}
    r = {
        "out": (cat["out"].permute(1, 0, 2), cat["out_b"].permute(1, 0, 2)),
        "lse": (cat["lse"], cat["lse_b"]),
    }
    if bwd:
        r["dq"] = (cat["dq"].permute(1, 0, 2), cat["dq_b"].permute(1, 0, 2))
        dk_r, dv_r = _group_sum(dk, Hk), _group_sum(dv, Hk)
        r["dk"] = (dk_r, (1 + U_BF16) * _group_sum(dk_b, Hk) + U_BF16 * dk_r.abs() + TINY)
        r["dv"] = (dv_r, (1 + U_BF16) * _group_sum(dv_b, Hk) + U_BF16 * dv_r.abs() + TINY)
        if sink64 is not None:
            r["dsink"] = (dsink, dsink_b)
            r["dsink_abs"] = (dsink_abs, dsink_abs)
    return r


def batch_reference(q, k, v, cu_q: list[int], cu_k: list[int], **kw) -> dict[str, tuple[torch.Tensor, torch.Tensor]]:
    """:func:`sequence_reference` over a packed batch: q [total_q, Hq, Dqk], k [total_k, Hk, Dqk], v [total_k, Hk, Dv],
    sequence b = rows [cu_q[b], cu_q[b+1]) / [cu_k[b], cu_k[b+1]).  lse is [Hq, total_q].  Rows outside every sequence must
    be exactly 0 (lse: -inf).  ``out`` / ``dlse`` (packed like q / lse) are sliced per sequence."""
    total_q, Hq, Dqk = q.shape
    total_k, Hk, Dv = k.shape[0], k.shape[1], v.shape[2]
    dev = q.device
    z = lambda *shape: torch.zeros(*shape, dtype=torch.float64, device=dev)  # noqa: E731
    bwd = kw.get("dout") is not None
    acc = {"out": [z(total_q, Hq, Dv), z(total_q, Hq, Dv)], "lse": [torch.full((Hq, total_q), -math.inf, dtype=torch.float64, device=dev),
                                                                     z(Hq, total_q)]}
    if bwd:
        acc.update(dq=[z(total_q, Hq, Dqk), z(total_q, Hq, Dqk)], dk=[z(total_k, Hk, Dqk), z(total_k, Hk, Dqk)],
                   dv=[z(total_k, Hk, Dv), z(total_k, Hk, Dv)])
        if kw.get("sink") is not None:
            acc.update(dsink=[z(Hq), z(Hq)], dsink_abs=[z(Hq), z(Hq)])
    for b in range(len(cu_q) - 1):
        qs, ks = slice(cu_q[b], cu_q[b + 1]), slice(cu_k[b], cu_k[b + 1])
        if qs.stop == qs.start:
            continue
        kws = dict(kw)
        for name in ("out", "dout"):
            if kws.get(name) is not None:
                kws[name] = kws[name][qs]
        if kws.get("dlse") is not None:
            kws["dlse"] = kws["dlse"][:, qs]
        r = sequence_reference(q[qs], k[ks], v[ks], **kws)
        for name, (ref, bound) in r.items():
            dst = acc[name]
            if name in ("lse",):
                dst[0][:, qs], dst[1][:, qs] = ref, bound
            elif name in ("out", "dq"):
                dst[0][qs], dst[1][qs] = ref, bound
            elif name in ("dk", "dv"):
                dst[0][ks], dst[1][ks] = ref, bound
            else:
                dst[0] += ref
                dst[1] += bound
    out = {name: tuple(v) for name, v in acc.items() if name != "dsink_abs"}
    if "dsink" in acc:  # fp32 sum over every row of the batch, then rounded to fp32
        ref, bound = out["dsink"]
        out["dsink"] = (ref, bound + ck(total_q) * acc["dsink_abs"][0] + 2 * U_F32 * ref.abs())
    return out


def fixed_reference(q, k, v, **kw) -> dict[str, tuple[torch.Tensor, torch.Tensor]]:
    """:func:`sequence_reference` over a fixed-length batch, q [B, Sq, Hq, Dqk], k [B, Sk, Hk, Dqk], v [B, Sk, Hk, Dv],
    lse / dlse [B, Hq, Sq]: the batch is folded into the heads (head b Hq + h reads kv head b Hk + h // g), so that many
    short sequences cost one call."""
    B, Sq, Hq = q.shape[:3]
    Sk, Hk = k.shape[1], k.shape[2]
    fold = lambda x, S, H: x.permute(1, 0, 2, 3).reshape(S, B * H, x.shape[-1])  # noqa: E731
    unfold = lambda x, S, H: x.reshape(S, B, H, x.shape[-1]).permute(1, 0, 2, 3)  # noqa: E731
    kws = dict(kw)
    if kws.get("sink") is not None:
        kws["sink"] = kws["sink"].repeat(B)
    for name in ("out", "dout"):
        if kws.get(name) is not None:
            kws[name] = fold(kws[name], Sq, Hq)
    if kws.get("dlse") is not None:
        kws["dlse"] = kws["dlse"].reshape(B * Hq, Sq)
    r = sequence_reference(fold(q, Sq, Hq), fold(k, Sk, Hk), fold(v, Sk, Hk), **kws)
    res = {"out": tuple(unfold(t, Sq, Hq) for t in r["out"]), "lse": tuple(t.reshape(B, Hq, Sq) for t in r["lse"])}
    if "dq" in r:
        res["dq"] = tuple(unfold(t, Sq, Hq) for t in r["dq"])
        res["dk"] = tuple(unfold(t, Sk, Hk) for t in r["dk"])
        res["dv"] = tuple(unfold(t, Sk, Hk) for t in r["dv"])
    if "dsink" in r:
        ref, bound = (t.view(B, Hq).sum(0) for t in r["dsink"])
        ab = r["dsink_abs"][0].view(B, Hq).sum(0)
        res["dsink"] = (ref, bound + ck(B * Sq) * ab + 2 * U_F32 * ref.abs())
    return res


def lse_err_ratio(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """err_ratio for an lse: where the reference is -inf the result must be -inf too."""
    inf = ref == -math.inf
    if bool((got[inf] != -math.inf).any()) or bool((got[~inf] == -math.inf).any()):
        return math.inf
    return err_ratio(got[~inf], ref[~inf], bound[~inf])


def assert_lse_within(got, ref, bound, what: str = "lse") -> float:
    r = lse_err_ratio(got, ref, bound)
    if not r <= 1.0:
        inf = ref == -math.inf
        if bool((got[inf] != -math.inf).any()) or bool((got[~inf] == -math.inf).any()):
            raise AssertionError(f"{what}: -inf pattern differs from the reference")
        assert_within(got[~inf], ref[~inf], bound[~inf], what)
    return r


def make_inputs(Sq: int, Sk: int, Hq: int, Hk: int, Dqk: int, Dv: int | None = None, *, scale: float, peak: float = 20.0,
                ramp: float = 8.0, B=None, gen: torch.Generator | None = None, device="cpu"):
    """bf16 (q, k, v, dout) as [S, H, D] (or [B, S, H, D]): q / k with Dqk columns, v / dout with Dv (default Dqk).  Scores
    reach about +-peak, so that soft-caps of 5 to 10 bend them and P is far from uniform, and every row's score rises by
    about ``ramp`` from the first key to the last, so the running max of the online softmax moves from one key tile to the
    next.  v / dout are the first Dv columns of the Dqk-wide draws, so a given seed yields the same q and k at every Dv."""
    Dv = Dqk if Dv is None else Dv
    lead = () if B is None else (B,)
    a = math.sqrt(peak / 3.0 / (scale * math.sqrt(Dqk)))
    q = torch.randn(*lead, Sq, Hq, Dqk, generator=gen) * a
    k = torch.randn(*lead, Sk, Hk, Dqk, generator=gen) * a
    v = torch.randn(*lead, Sk, Hk, Dqk, generator=gen)
    dout = torch.randn(*lead, Sq, Hq, Dqk, generator=gen)
    c = math.sqrt(ramp / scale)
    q[..., 0] += c
    k[..., 0] += c * (torch.arange(Sk) / max(Sk - 1, 1)).view(*((1,) * len(lead)), Sk, 1)
    q, k, v, dout = (t.bfloat16().to(device) for t in (q, k, v, dout))
    return q, k, v[..., :Dv].contiguous(), dout[..., :Dv].contiguous()

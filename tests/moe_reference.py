"""fp64 reference and per-element error bound for the bf16 MoE expert block ``grouped_swiglu`` and for the expert path
``moe_permute -> grouped_swiglu -> moe_unpermute``.  Pure torch: works on CPU tensors (self-test) and CUDA tensors alike.

The block over the 128-row aligned layout, per expert segment ``[seg[e], seg[e+1])`` (pad rows are zero):

    forward   G = x Wg,  U = x Wu,  h = silu(G) U p,  y = h Wd
    backward  dh = dy Wd^T,  dgate = dh U p silu'(G),  dup = dh silu(G) p,  dp = sum_f dh silu(G) U,
              dx = dgate Wg^T + dup Wu^T,  dWg = x^T dgate,  dWu = x^T dup,  dWd = h^T dy

The kernels round ``G``, ``U``, ``h``, ``y``, ``dh``, ``dgate``, ``dup`` and ``dx`` to bf16 (the up-projection's input
gradient is rounded before it is added to the gate's, ``EPI_BF16_ACC``) and the weight gradients to their gradient dtype.
The bound is a first-order propagation in absolute values, stage by stage: every stage adds its own rounding term (the
GEMMs' ``ck(K) |A||B|`` plus output rounding from ``tests.gemm_reference``, the SiLU·mul·prob kernels' terms from
``tests.pointwise_reference``) to the error it inherits.  Inherited errors are carried by the product rule
``|prod(a + da) - prod(a)| <= prod(|a| + e_a) - prod(|a|)``; SiLU and its derivative are Lipschitz with
``|silu(G + d) - silu(G)| <= (|silu'(G)| + |d| / 2) |d|`` and ``|silu'(G + d) - silu'(G)| <= |d| / 2``
(``|silu''| <= 1/2``), so no fudge factor is needed.
"""

from __future__ import annotations

import torch

from tests.gemm_reference import U_BF16, U_F32, ck, gemm_bound
from tests.pointwise_reference import U32, cn, rounding

OUTPUTS = ("y", "dx", "dprobs", "dWg", "dWu", "dWd")
BF16 = torch.bfloat16


def _mag(*terms: tuple[torch.Tensor, torch.Tensor | float]) -> torch.Tensor:
    """prod(|a| + e_a) over (a, e_a) pairs: the largest magnitude a product of perturbed factors can have."""
    out = None
    for a, e in terms:
        out = a.abs() + e if out is None else out * (a.abs() + e)
    return out


def _prod_err(*terms: tuple[torch.Tensor, torch.Tensor | float]) -> torch.Tensor:
    """prod(|a| + e_a) - prod(|a|) over (a, e_a) pairs: how far a product of perturbed factors can move."""
    return _mag(*terms) - _mag(*((a, 0.0) for a, _ in terms))


def _stage(prod: torch.Tensor, S: torch.Tensor, inherited: torch.Tensor, K: int, out_dtype: torch.dtype,
           d0: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """(reference, bound) of a GEMM whose operands carry errors: ``gemm_bound`` on the magnitudes the kernel saw
    (``S`` = |A| |B| with |A| inflated by its error), plus the ``inherited`` error ``e_A |B|`` and its output rounding."""
    ref, bound = gemm_bound(prod, S, K, out_dtype, d0)
    u = U_BF16 if out_dtype == BF16 else 2 * U_F32
    return ref, bound + (1 + u) * inherited


def _silu_terms(G: torch.Tensor, eG: torch.Tensor):
    """silu(G), silu'(G), sigma(G), their error bounds for an input that is off by at most ``eG``, and the
    ``__expf`` / fast-reciprocal relative error ``e_f`` of the kernels at the input they actually read."""
    sg = torch.sigmoid(G)
    s = G * sg
    ds = sg * (1 + G * (1 - sg))
    es = (ds.abs() + 0.5 * eG) * eG
    ef = 2.0**-20 + (G.abs() + eG) * 2.0**-23
    return s, ds, sg, es, 0.5 * eG, ef


def expert_block_ref(xp: torch.Tensor, pp: torch.Tensor, wg: torch.Tensor, wu: torch.Tensor, wd: torch.Tensor,
                     seg_offsets, dy: torch.Tensor | None = None, *, wgrad_dtype: torch.dtype = torch.float32,
                     g0: tuple | None = None) -> dict[str, tuple[torch.Tensor, torch.Tensor]]:
    """fp64 ``(reference, bound)`` of the block's outputs over the rows in use ``[0, seg_offsets[-1])``.

    ``xp [cap, H]`` bf16 (pad rows zero), ``pp [cap]`` fp32, ``wg, wu [E, H, F]`` / ``wd [E, F, H]`` bf16, ``dy [cap, H]``
    bf16.  Returns ``y``, and with ``dy`` also ``dx``, ``dprobs`` ([rows in use]) and ``dWg``, ``dWu``, ``dWd``
    ([E, ...], in ``wgrad_dtype``; with ``g0 = (gWg, gWu, gWd)`` the fused accumulate ``g0 + dW``).  An expert without
    rows has a zero bound: its gradient is exactly zero (or ``g0``).  The weights are widened one expert at a time, so
    DeepSeek-V3-sized experts fit."""
    seg = [int(v) for v in (seg_offsets.tolist() if torch.is_tensor(seg_offsets) else seg_offsets)]
    E, H, F = wg.shape
    rows = seg[-1]
    dev, f64 = xp.device, torch.float64
    out: dict[str, tuple[torch.Tensor, torch.Tensor]] = {}

    def zeros(*shape):
        return torch.zeros(*shape, dtype=f64, device=dev)

    y, yb = zeros(rows, H), zeros(rows, H)
    if dy is not None:
        dx, dxb, dp, dpb = zeros(rows, H), zeros(rows, H), zeros(rows), zeros(rows)
        dW = {n: [zeros(E, *s), zeros(E, *s)] for n, s in (("dWg", (H, F)), ("dWu", (H, F)), ("dWd", (F, H)))}
        if g0 is not None:
            for n, g in zip(("dWg", "dWu", "dWd"), g0):
                dW[n][0].copy_(g.double())
    for e in range(E):
        r0, r1 = seg[e], seg[e + 1]
        if r1 == r0:
            continue
        x, p = xp[r0:r1].double(), pp[r0:r1].double()[:, None]
        ax = x.abs()
        Wg, Wu, Wd = wg[e].double(), wu[e].double(), wd[e].double()
        aWg, aWu, aWd = Wg.abs(), Wu.abs(), Wd.abs()
        # gate / up projections: bf16 outputs of H-deep fp32 accumulations
        G, eG = gemm_bound(x @ Wg, ax @ aWg, H, BF16)
        Uv, eU = gemm_bound(x @ Wu, ax @ aWu, H, BF16)
        s, ds, sg, es, eds, ef = _silu_terms(G, eG)
        # h = silu(G) U p: inherited error, then the SiLU·mul·prob kernel's rounding (silu_mul_probs_fwd_ref)
        h = s * Uv * p
        hin = _prod_err((s, es), (Uv, eU), (p, 0.0))
        hmag = h.abs() + hin
        hb = hin + (ef + 3 * U32) * hmag + rounding(hmag, BF16)
        ref, b = _stage(h @ Wd, hmag @ aWd, hb @ aWd, F, BF16)
        y[r0:r1], yb[r0:r1] = ref, b
        if dy is None:
            continue
        g = dy[r0:r1].double()
        dh, edh = gemm_bound(g @ Wd.t(), g.abs() @ aWd.t(), F, BF16)
        # silu_mul_probs_bwd_ref with inherited errors in dh, G and U
        dgate = dh * Uv * p * ds
        dg_in = _prod_err((dh, edh), (Uv, eU), (p, 0.0), (ds, eds))
        dg_mag = dgate.abs() + dg_in
        dgb = (dg_in + (ef + 7 * U32) * _mag((dh, edh), (Uv, eU), (p, 0.0), (sg + s.abs(), 0.25 * eG + es))
               + rounding(dg_mag, BF16))
        dup = dh * s * p
        du_in = _prod_err((dh, edh), (s, es), (p, 0.0))
        du_mag = dup.abs() + du_in
        dub = du_in + (ef + 3 * U32) * du_mag + rounding(du_mag, BF16)
        t = dh * s * Uv
        t_in = _prod_err((dh, edh), (s, es), (Uv, eU))
        t_mag = t.abs() + t_in
        dp[r0:r1] = t.sum(-1)
        dpb[r0:r1] = (t_in + (ef + 3 * U32) * t_mag).sum(-1) + cn(F) * t_mag.sum(-1) + rounding(dp[r0:r1], torch.float32)
        # dx = bf16(bf16(dgate Wg^T) + bf16(dup Wu^T)): two F-deep GEMMs, the second accumulating in bf16
        P1, P2 = dgate @ Wg.t(), dup @ Wu.t()
        inh = dgb @ aWg.t() + dub @ aWu.t()
        dx[r0:r1] = P1 + P2
        dxb[r0:r1] = (ck(F) * (dg_mag @ aWg.t() + du_mag @ aWu.t()) + (1 + U_BF16) * inh
                      + U_BF16 * (P1.abs() + P2.abs() + (P1 + P2).abs() + 2 * inh))
        # weight gradients: reductions over the segment's rows
        K = r1 - r0
        for name, a, a_mag, a_b, bmat, b_mag, b_b in (("dWg", x, ax, None, dgate, dg_mag, dgb),
                                                      ("dWu", x, ax, None, dup, du_mag, dub),
                                                      ("dWd", h, hmag, hb, g, g.abs(), None)):
            inherited = a_mag.t() @ b_b if b_b is not None else a_b.t() @ b_mag
            d0 = dW[name][0][e] if g0 is not None else None
            ref, b = _stage(a.t() @ bmat, a_mag.t() @ b_mag, inherited, K, wgrad_dtype, d0)
            dW[name][0][e], dW[name][1][e] = ref, b
    out["y"] = (y, yb)
    if dy is not None:
        out["dx"], out["dprobs"] = (dx, dxb), (dp, dpb)
        out.update({n: tuple(v) for n, v in dW.items()})
    return out


def permute_ref(x: torch.Tensor, probs: torch.Tensor, row_map: torch.Tensor, capacity: int):
    """The exact copy ``moe_permute`` makes: ``xp [capacity, H]`` (bf16, pad rows zero) and ``pp [capacity]`` (fp32)."""
    rm = row_map.long().reshape(-1)
    keep = rm >= 0
    tok = torch.arange(x.shape[0], device=x.device).repeat_interleave(rm.numel() // max(x.shape[0], 1))
    xp = torch.zeros(capacity, x.shape[1], dtype=x.dtype, device=x.device)
    pp = torch.zeros(capacity, dtype=torch.float32, device=x.device)
    xp[rm[keep]] = x[tok[keep]]
    pp[rm[keep]] = probs.reshape(-1).float()[keep]
    return xp, pp


def _gather(v: torch.Tensor, vb: torch.Tensor, row_map: torch.Tensor, T: int, k: int):
    """fp32 sum of a token's k rows rounded to bf16 (``moe_gather``), rows carrying the errors ``vb``."""
    rm = row_map.long().reshape(T, k)
    keep = (rm >= 0)[..., None]
    rows = v[rm.clamp_min(0)] * keep
    inh = (vb[rm.clamp_min(0)] * keep).sum(1)
    ref = rows.sum(1)
    mag = rows.abs().sum(1) + inh
    return ref, inh + cn(k) * mag + rounding(ref.abs() + inh, BF16)


def expert_path_ref(x: torch.Tensor, probs: torch.Tensor, wg: torch.Tensor, wu: torch.Tensor, wd: torch.Tensor,
                    row_map: torch.Tensor, seg_offsets, capacity: int, dy: torch.Tensor | None = None, *,
                    wgrad_dtype: torch.dtype = torch.float32) -> dict[str, tuple[torch.Tensor, torch.Tensor]]:
    """``moe_permute -> grouped_swiglu -> moe_unpermute`` from ``x [T, H]`` bf16 and ``probs [T, k]``; dropped slots
    (``row_map < 0``) contribute nothing.  ``dy [T, H]`` bf16 is the gradient of the token outputs; ``dx`` sums the
    token's k rows like the forward, ``dprobs [T, k]`` is a copy of the block's per-row value (0 when dropped)."""
    T, k = probs.shape
    xp, pp = permute_ref(x, probs, row_map, capacity)
    dyp = None
    if dy is not None:
        dyp = torch.zeros(capacity, dy.shape[1], dtype=dy.dtype, device=dy.device)
        rm = row_map.long().reshape(-1)
        keep = rm >= 0
        dyp[rm[keep]] = dy.repeat_interleave(k, 0)[keep]
    blk = expert_block_ref(xp, pp, wg, wu, wd, seg_offsets, dyp, wgrad_dtype=wgrad_dtype)
    rows = blk["y"][0].shape[0]
    pad = capacity - rows

    def full(v):
        return torch.cat([v, v.new_zeros(pad, *v.shape[1:])])

    out = {"y": _gather(full(blk["y"][0]), full(blk["y"][1]), row_map, T, k)}
    if dy is not None:
        out["dx"] = _gather(full(blk["dx"][0]), full(blk["dx"][1]), row_map, T, k)
        rm = row_map.long().reshape(T, k)
        keep = rm >= 0
        out["dprobs"] = tuple(torch.where(keep, full(v)[rm.clamp_min(0)], 0.0) for v in blk["dprobs"])
        out.update({n: blk[n] for n in ("dWg", "dWu", "dWd")})
    return out

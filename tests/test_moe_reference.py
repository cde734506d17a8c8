"""The expert block's fp64 reference and bound (``tests/moe_reference.py``) on the CPU.

An fp32 emulation of the kernels' algorithm (bf16 operands, fp32 products and sums, bf16 rounding of every
intermediate the kernels store, the bf16 accumulate of the input gradient) must pass the bound; each injected fault of
the kind a kernel or autograd change could make must exceed it.  The layouts have empty, 1-row, 127 / 128 / 129-row
segments and dropped (token, slot) pairs."""

from __future__ import annotations

import pytest
import torch

from d9d_b200.kernel.moe import build_moe_layout
from tests.gemm_reference import err_ratio
from tests.moe_reference import OUTPUTS, expert_block_ref, expert_path_ref, permute_ref

BF = torch.bfloat16
SKEWED = (0, 1, 127, 128, 129, 0, 3, 5)  # tokens per expert


def _ids(counts, drop: int = 0, seed: int = 0) -> torch.Tensor:
    """[T, 1] expert ids with the given tokens per expert (shuffled) and ``drop`` dropped pairs (id -1)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.cat([torch.full((c,), e) for e, c in enumerate(counts)] + [torch.full((drop,), -1)])
    return ids[torch.randperm(ids.numel(), generator=g)][:, None]


def _problem(H=64, F=48, counts=SKEWED, drop=7, seed=0, wgrad_dtype=torch.float32, g0=False):
    g = torch.Generator().manual_seed(seed)
    E = len(counts)
    ids = _ids(counts, drop, seed)
    layout = build_moe_layout(ids, E)
    T = ids.shape[0]
    x = torch.randn(T, H, generator=g).to(BF)
    probs = torch.rand(T, 1, generator=g) * 0.8 + 0.1
    xp, pp = permute_ref(x, probs, layout.row_map, layout.capacity)
    w = [(torch.randn(E, a, b, generator=g) / a**0.5).to(BF) for a, b in ((H, F), (H, F), (F, H))]
    dy = torch.randn(layout.capacity, H, generator=g).to(BF)
    g0s = tuple(torch.randn(t.shape, generator=g).to(wgrad_dtype) for t in w) if g0 else None
    return xp, pp, w, layout, dy, g0s


def emulate(xp, pp, w, seg, dy, *, fault=None, wgrad_dtype=torch.float32, g0=None, counts=None):
    """The native block's algorithm in fp32 on bf16 values, segment by segment, with an optional injected fault."""
    wg, wu, wd = w
    E, H, F = wg.shape
    rows = seg[-1]
    y, dx, dp = torch.zeros(rows, H), torch.zeros(rows, H), torch.zeros(rows)
    dW = [torch.zeros(t.shape, dtype=wgrad_dtype) if g0 is None else g.clone() for t, g in zip(w, g0 or (None,) * 3)]
    target = next(e for e in range(E) if seg[e] > 0 and seg[e + 1] > seg[e])  # first non-empty expert after row 0

    def mm(a, b):
        return a.float() @ b.float()

    for e in range(E):
        r0, r1 = seg[e], seg[e + 1]
        if r1 == r0:
            continue
        x = xp[r0 - 1 : r1 - 1] if fault == "segment_one_row_early" and e == target else xp[r0:r1]
        p = pp[r0:r1, None]
        G, U = mm(x, wg[e]).to(BF).float(), mm(x, wu[e]).to(BF).float()
        sg = 1 / (1 + torch.exp(-G))
        s = G * sg
        h = (G * sg * U * p).to(BF)
        y[r0:r1] = mm(h, wd[e]).to(BF).float()
        dh = mm(dy[r0:r1], wd[e].t()).to(BF).float()
        gp = {"prob_missing": dh, "prob_twice": dh * p * p}.get(fault, dh * p)
        dsilu = sg if fault == "silu_prime_without_x_term" else sg + s * (1 - sg)
        dgate, dup = (gp * U * dsilu).to(BF), (gp * s).to(BF)
        dp[r0:r1] = (dh * h.float()).sum(-1) if fault == "dprobs_sums_h" else (dh * s * U).sum(-1)
        wa, wb = (wu[e], wg[e]) if fault == "gate_up_swapped_in_dgrad" else (wg[e], wu[e])
        P1, P2 = mm(dgate, wa.t()).to(BF).float(), mm(dup, wb.t()).to(BF).float()
        dx[r0:r1] = {"dx_without_up": P1, "dx_up_overwrites": P2, "dx_up_twice": (P1 + P2).to(BF).float() + P2}.get(
            fault, P1 + P2).to(BF).float()
        xw, dgw, duw, hw, dyw = x, dgate, dup, h, dy[r0:r1]
        if fault == "wgrad_skips_last_row":
            last = counts[e] - 1  # the segment's last token row
            keep = torch.arange(r1 - r0) != last
            xw, dgw, duw, hw, dyw = (t[keep] for t in (xw, dgw, duw, hw, dyw))
        for i, (a, b) in enumerate(((xw, dgw), (xw, duw), (hw, dyw))):
            prod = mm(a.t(), b)
            if g0 is not None and fault != "fused_wgrad_overwrites":
                dW[i][e] = (dW[i][e].float() + prod).to(wgrad_dtype)
            else:
                dW[i][e] = prod.to(wgrad_dtype)
    return dict(zip(OUTPUTS, (y, dx, dp, *dW)))


def _ratios(got: dict, ref: dict) -> dict[str, float]:
    return {n: err_ratio(got[n], *ref[n]) for n in OUTPUTS}


@pytest.mark.parametrize("wgrad_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("fused", [False, True])
def test_emulation_passes_the_bound(wgrad_dtype, fused):
    xp, pp, w, layout, dy, g0 = _problem(wgrad_dtype=wgrad_dtype, g0=fused)
    seg = layout.seg_offsets.tolist()
    assert layout.counts.tolist() == list(SKEWED) and (layout.row_map < 0).sum() == 7
    ref = expert_block_ref(xp, pp, *w, seg, dy, wgrad_dtype=wgrad_dtype, g0=g0)
    got = emulate(xp, pp, w, seg, dy, wgrad_dtype=wgrad_dtype, g0=g0)
    r = _ratios(got, ref)
    print(f"\nemulation err/bound ({wgrad_dtype}, fused={fused}): " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    assert all(v <= 1.0 for v in r.values()), r
    # empty experts: zero (or the untouched prior gradient) with a zero bound
    for n in ("dWg", "dWu", "dWd"):
        for e in (0, 5):
            assert float(ref[n][1][e].abs().max()) == 0.0


def test_bound_is_not_vacuous():
    """The bound stays within a few bf16 roundings of the values it bounds, where they are not cancelling."""
    xp, pp, w, layout, dy, _ = _problem(counts=(200, 300), drop=0)
    ref = expert_block_ref(xp, pp, *w, layout.seg_offsets, dy)
    for n in OUTPUTS:
        v, b = ref[n]
        big = v.abs() > v.abs().max() * 0.1
        rel = float((b[big] / v[big].abs()).median())
        assert rel < 0.1, (n, rel)


FAULTS = {  # fault -> the output that must exceed the bound
    "prob_missing": "dx",
    "prob_twice": "dWg",
    "silu_prime_without_x_term": "dx",
    "dprobs_sums_h": "dprobs",
    "dx_without_up": "dx",
    "dx_up_overwrites": "dx",
    "dx_up_twice": "dx",
    "gate_up_swapped_in_dgrad": "dx",
    "wgrad_skips_last_row": "dWd",
    "segment_one_row_early": "y",
    "fused_wgrad_overwrites": "dWu",
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_injected_fault_exceeds_the_bound(fault):
    """At the skewed layout (H = 64, F = 48, 8 experts, fp32 weight gradients; fused accumulation for the fused fault)."""
    fused = fault == "fused_wgrad_overwrites"
    xp, pp, w, layout, dy, g0 = _problem(g0=fused)
    seg = layout.seg_offsets.tolist()
    ref = expert_block_ref(xp, pp, *w, seg, dy, g0=g0)
    got = emulate(xp, pp, w, seg, dy, fault=fault, g0=g0, counts=layout.counts.tolist())
    r = _ratios(got, ref)
    assert r[FAULTS[fault]] > 1.0, (fault, r)
    if fault == "prob_missing":
        assert r["dWu"] > 1.0 and r["dWg"] > 1.0


def test_expert_path_reference_against_emulation():
    """permute -> block -> unpermute with dropped slots, k = 2: the emulated chain passes the chained bound."""
    g = torch.Generator().manual_seed(3)
    T, k, E, H, F = 300, 2, 6, 64, 48
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)])
    ids[torch.rand(T, k, generator=g) < 0.1] = -1
    layout = build_moe_layout(ids, E)
    x = torch.randn(T, H, generator=g).to(BF)
    probs = torch.rand(T, k, generator=g)
    w = [(torch.randn(E, a, b, generator=g) / a**0.5).to(BF) for a, b in ((H, F), (H, F), (F, H))]
    dy = torch.randn(T, H, generator=g).to(BF)
    ref = expert_path_ref(x, probs, *w, layout.row_map, layout.seg_offsets, layout.capacity, dy)

    xp, pp = permute_ref(x, probs, layout.row_map, layout.capacity)
    rm = layout.row_map.long()
    dyp = torch.zeros(layout.capacity, H, dtype=BF)
    dyp[rm[rm >= 0]] = dy.repeat_interleave(k, 0)[rm >= 0]
    blk = emulate(xp, pp, w, layout.seg_offsets.tolist(), dyp)

    def gather(v):
        full = torch.cat([v, v.new_zeros(layout.capacity - v.shape[0], *v.shape[1:])])
        rows = full[rm.clamp_min(0)].reshape(T, k, -1) * (rm >= 0).reshape(T, k, 1)
        return rows.float().sum(1).to(BF)

    got = {"y": gather(blk["y"]), "dx": gather(blk["dx"]),
           "dprobs": torch.where(rm >= 0, torch.cat([blk["dprobs"], torch.zeros(layout.capacity)])[rm.clamp_min(0)],
                                 0.0).reshape(T, k)}
    got.update({n: blk[n] for n in ("dWg", "dWu", "dWd")})
    for n in OUTPUTS:
        assert err_ratio(got[n], *ref[n]) <= 1.0, n
    assert bool((ref["dprobs"][0][ids < 0] == 0).all())
    # a slot summed twice (or a dropped slot read) exceeds it
    bad = got["y"].float() + gather(blk["y"]).float() * (torch.arange(T) == 5)[:, None]
    assert err_ratio(bad, *ref["y"]) > 1.0

"""The bf16 MoE expert block ``grouped_swiglu`` (one autograd node: six grouped wgmma GEMMs, the SiLU·mul·prob kernels,
caller buffers, split backward, fused weight-gradient accumulation) and the expert-parallel exchange kernels ``ep_push`` /
``ep_pull_sum`` on one GPU.

The block is checked per element against the fp64 reference and bound of ``tests/moe_reference.py`` (y, dx, dprobs and
the three weight gradients on the rows in use) at the flagship shape, a skewed layout off the tile edges, one expert
holding every token's first slot, dropped pairs, ~8192 rows per expert and a DeepSeek-V3 expert shape.  Every case puts
NaN in the rows past the last segment (the stale receive region of the expert-parallel path): nothing may leak.  The
worst err / bound per case and output is printed at the end of the module.

``ep_push`` / ``ep_pull_sum`` read and write through a device table of base pointers: W canary-filled buffers on one
device stand in for W peers."""

from __future__ import annotations

import re

import pytest
import torch

from tests.gemm_reference import assert_within
from tests.moe_reference import OUTPUTS, expert_block_ref, expert_path_ref, permute_ref

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF = torch.bfloat16
WORST: dict[tuple[str, str], float] = {}
SKEWED = (0, 1, 127, 128, 129, 0, 3000, 5)  # tokens per expert, E = 8


@pytest.fixture(scope="module")
def ops():
    from d9d_b200 import ops as _ops

    yield _ops.load()
    if WORST:
        print("\nworst err/bound per case and output:")
        for case in dict.fromkeys(c for c, _ in WORST):
            print(f"  {case}: " + ", ".join(f"{n} {WORST[(c, n)]:.3g}" for c, n in WORST if c == case))


def _check(case: str, got: dict, ref: dict, names=OUTPUTS) -> None:
    for n in names:
        r = assert_within(got[n], *ref[n], f"{case} {n}")
        WORST[(case, n)] = max(WORST.get((case, n), 0.0), r)


# ----------------------------------------------------------------------------- problems
def _skewed_ids(counts, drop: int, gen: torch.Generator) -> torch.Tensor:
    ids = torch.cat([torch.full((c,), e) for e, c in enumerate(counts)] + [torch.full((drop,), -1)])
    return ids[torch.randperm(ids.numel(), generator=gen)][:, None]


def _ids(kind: str, T: int, k: int, E: int, gen: torch.Generator) -> torch.Tensor:
    if kind == "skewed":
        return _skewed_ids(SKEWED, 11, gen)
    ids = torch.stack([torch.randperm(E, generator=gen)[:k] for _ in range(T)])
    if kind == "one_expert":  # every token's first slot is expert 0
        ids = torch.stack([torch.cat([torch.zeros(1, dtype=torch.long), 1 + torch.randperm(E - 1, generator=gen)[: k - 1]])
                           for _ in range(T)])
    elif kind == "dropped":
        ids[torch.rand(T, k, generator=gen) < 0.2] = -1
    return ids


CASES = {  # name: (routing, T, k, E, H, F, weight-gradient dtype)
    "flagship": ("uniform", 2048, 8, 128, 768, 576, torch.float32),
    "skewed": ("skewed", 0, 1, 8, 136, 200, torch.bfloat16),
    "one_expert": ("one_expert", 1000, 4, 8, 256, 192, torch.float32),
    "dropped": ("dropped", 1000, 4, 16, 256, 192, torch.bfloat16),
    "long_wgrad": ("uniform", 8192, 2, 2, 256, 192, torch.float32),  # 8192 rows per expert
    "deepseek_v3": ("uniform", 256, 8, 32, 7168, 2048, torch.float32),
}


class Problem:
    """Routing, permuted inputs (pad rows zero, NaN past the last segment) and weights on the GPU."""

    def __init__(self, kind, T, k, E, H, F, seed=0, unused_expert=None):
        from d9d_b200.kernel.moe import build_moe_layout

        gen = torch.Generator().manual_seed(seed)
        self.ids = _ids(kind, T, k, E, gen)
        if unused_expert is not None:  # its pairs are dropped: the expert gets no rows
            self.ids[self.ids == unused_expert] = -1
        self.T, self.k = self.ids.shape
        self.layout = build_moe_layout(self.ids.to(DEV), E)
        self.seg = self.layout.seg_offsets.tolist()
        self.used, self.cap = self.seg[-1], self.layout.capacity
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.x = torch.randn(self.T, H, device=DEV, generator=g).to(BF)
        self.probs = torch.rand(self.T, self.k, device=DEV, generator=g) * 0.9 + 0.05
        self.w = [(torch.randn(E, a, b, device=DEV, generator=g) / a**0.5).to(BF) for a, b in ((H, F), (H, F), (F, H))]
        self.xp, self.pp = permute_ref(self.x, self.probs, self.layout.row_map, self.cap)
        self.xp[self.used :] = float("nan")
        self.pp[self.used :] = float("nan")
        self.dy = torch.randn(self.cap, H, device=DEV, generator=g).to(BF)
        self.dy[self.used :] = float("nan")


def _params(w, grad_dtype):
    out = []
    for t in w:
        p = torch.nn.Parameter(t.clone())
        p.grad_dtype = grad_dtype
        out.append(p)
    return out


def _run_block(pb: Problem, grad_dtype=torch.float32, *, weights=None):
    """y, dx, dprobs and the weight gradients of one forward + backward of ``grouped_swiglu``."""
    from d9d_b200.kernel.moe import grouped_swiglu

    xp, pp = pb.xp.clone().requires_grad_(), pb.pp.clone().requires_grad_()
    ws = weights if weights is not None else _params(pb.w, grad_dtype)
    y = grouped_swiglu(xp, pp, *ws, pb.layout)
    yc = y.detach().clone()
    y.backward(pb.dy)
    u = pb.used
    return {"y": yc[:u], "dx": xp.grad[:u], "dprobs": pp.grad[:u],
            **{n: w.grad for n, w in zip(("dWg", "dWu", "dWd"), ws)}}


def _bitwise_equal(a: dict, b: dict, names=OUTPUTS) -> None:
    for n in names:
        assert (a[n] is None) == (b[n] is None), n
        if a[n] is not None:
            assert torch.equal(a[n], b[n]), n


# ----------------------------------------------------------------------------- the block against fp64
@pytest.mark.parametrize("case", list(CASES))
def test_block_against_fp64(ops, case):
    kind, T, k, E, H, F, gdt = CASES[case]
    pb = Problem(kind, T, k, E, H, F)
    tiles = pb.layout.tile_group.tolist()
    assert -1 not in tiles[: pb.used // 128] and set(tiles[pb.used // 128 :]) <= {-1}
    if case == "flagship":
        assert 250 <= len(tiles) and tiles[-1] == -1  # ~255 row tiles, unused ones at the end
    got = _run_block(pb, gdt)
    for n in OUTPUTS:
        assert bool(torch.isfinite(got[n]).all()), f"{case}: {n} is not finite"
    _check(case, got, expert_block_ref(pb.xp, pb.pp, *pb.w, pb.seg, pb.dy, wgrad_dtype=gdt))
    for n in ("dWg", "dWu", "dWd"):  # an expert without rows gets an exact zero gradient
        for e, c in enumerate(pb.layout.counts.tolist()):
            if c == 0:
                assert not bool(got[n][e].any()), (n, e)
    _bitwise_equal(got, _run_block(pb, gdt))  # two runs are bitwise equal


# ----------------------------------------------------------------------------- fused wgrad, frozen weights
@pytest.mark.parametrize("grad_dtype", [torch.float32, torch.bfloat16])
def test_fused_wgrad_accumulates_over_two_microbatches(ops, grad_dtype):
    from d9d_b200.kernel._native import FUSED_WGRAD_ATTR

    E, H, F = 8, 136, 200
    mbs = [Problem("dropped", 700, 2, E, H, F, seed=s, unused_expert=3) for s in (1, 2)]  # two routings
    g = torch.Generator(device=DEV).manual_seed(9)
    g0 = [torch.randn(t.shape, device=DEV, generator=g).to(grad_dtype) for t in mbs[0].w]
    ws = _params(mbs[0].w, grad_dtype)
    for p, gi in zip(ws, g0):
        p.grad = gi.clone()
        setattr(p, FUSED_WGRAD_ATTR, True)
    grads0 = [p.grad for p in ws]
    for pb in mbs:
        _run_block(pb, weights=ws)
    assert all(p.grad is gi for p, gi in zip(ws, grads0))  # accumulated in place
    ref1 = expert_block_ref(mbs[0].xp, mbs[0].pp, *mbs[0].w, mbs[0].seg, mbs[0].dy, wgrad_dtype=grad_dtype, g0=g0)
    acc = tuple(ref1[n][0] for n in ("dWg", "dWu", "dWd"))
    ref2 = expert_block_ref(mbs[1].xp, mbs[1].pp, *mbs[0].w, mbs[1].seg, mbs[1].dy, wgrad_dtype=grad_dtype, g0=acc)
    u = 2.0**-8 if grad_dtype == BF else 2.0**-23
    ref = {n: (ref2[n][0], ref2[n][1] + (1 + u) * ref1[n][1]) for n in ("dWg", "dWu", "dWd")}
    _check(f"fused_wgrad_{str(grad_dtype)[6:]}", dict(zip(("dWg", "dWu", "dWd"), (p.grad for p in ws))), ref,
           ("dWg", "dWu", "dWd"))
    for p, gi in zip(ws, g0):
        assert torch.equal(p.grad[3], gi[3]), "an expert without rows changed its gradient"


def _grouped_k_launches(prof) -> int:
    return sum(1 for ev in prof.events()
               if re.search(r"gemm_kernel<2, ", ev.name) or re.search(r"gemm_kernelILi2E", ev.name))


@pytest.mark.parametrize("frozen", ["all", "gate"])
def test_frozen_weights_launch_no_weight_gradient_gemm(ops, frozen):
    from torch.profiler import ProfilerActivity, profile

    pb = Problem("skewed", 0, 1, 8, 136, 200)
    trainable = _run_block(pb)
    ws = _params(pb.w, torch.float32)
    for p in (ws if frozen == "all" else ws[:1]):
        p.requires_grad_(False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        got = _run_block(pb, weights=ws)
        torch.cuda.synchronize()
    assert _grouped_k_launches(prof) == (0 if frozen == "all" else 2)
    _bitwise_equal(got, trainable, ("y", "dx", "dprobs"))
    assert all(p.grad is None for p in ws if not p.requires_grad)
    _bitwise_equal(got, trainable, [n for n, p in zip(("dWg", "dWu", "dWd"), ws) if p.requires_grad])


# ----------------------------------------------------------------------------- split backward, caller buffers
def test_split_backward_is_bitwise_the_joint_backward(ops):
    from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection
    from d9d_b200.kernel.moe import grouped_swiglu

    pb = Problem("skewed", 0, 1, 8, 136, 200, seed=3)
    whole = _run_block(pb)
    canary = torch.full((pb.cap + 64, pb.xp.shape[1]), -7168.0, device=DEV, dtype=BF)
    before = canary.clone()
    xp, pp = pb.xp.clone().requires_grad_(), pb.pp.clone().requires_grad_()
    ws = _params(pb.w, torch.float32)
    y = grouped_swiglu(xp, pp, *ws, pb.layout, None, canary)
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.inputs):
        dx, dp = torch.autograd.grad(y, (xp, pp), pb.dy, retain_graph=True)
    assert torch.equal(canary, before), "the inputs pass of a split backward wrote into the caller's dx buffer"
    with GLOBAL_GRAD_CONTEXT.with_directions(GradDirection.weight):
        dws = torch.autograd.grad(y, ws, pb.dy)
    u = pb.used
    split = {"y": y.detach()[:u], "dx": dx[:u], "dprobs": dp[:u], **dict(zip(("dWg", "dWu", "dWd"), dws))}
    _bitwise_equal(split, whole)
    assert torch.equal(canary, before)


def test_caller_buffers_aliased_like_the_expert_parallel_handler(ops):
    """``out`` and ``dx_out`` are one staging tensor and ``dy`` is a view of it, as the NVLink handler passes them."""
    from d9d_b200.kernel.moe import grouped_swiglu

    pb = Problem("skewed", 0, 1, 8, 136, 200, seed=4)
    plain = _run_block(pb)
    cap, H = pb.cap, pb.xp.shape[1]
    staging = torch.full((cap + 96, H), -7168.0, device=DEV, dtype=BF)
    xp, pp = pb.xp.clone().requires_grad_(), pb.pp.clone().requires_grad_()
    ws = _params(pb.w, torch.float32)
    y = grouped_swiglu(xp, pp, *ws, pb.layout, staging, staging)
    assert y.data_ptr() == staging.data_ptr()
    u = pb.used
    y_got = y[:u].clone()
    # the combine backward's ep_push stores dy into the staging region through a raw pointer: no autograd version bump
    with torch.autograd._unsafe_preserve_version_counter(staging):
        staging[:cap].copy_(pb.dy)
    dy = staging[:cap]
    y.backward(dy)
    assert torch.equal(staging[:u], plain["dx"]), "the input gradient is not in the staging region"
    got = {"y": y_got, "dx": xp.grad[:u], "dprobs": pp.grad[:u], **dict(zip(("dWg", "dWu", "dWd"), (w.grad for w in ws)))}
    _bitwise_equal(got, plain)
    assert bool((staging[cap:] == -7168.0).all()), "rows past the capacity were written"


# ----------------------------------------------------------------------------- the composed path, the expert path
def test_composed_path_against_fp64(ops):
    """Three ``grouped_linear`` calls and ``silu_mul_probs`` (what LoRA-wrapped projections run), with and without the
    fused-wgrad owner of ``grouped_linear``, and the fused block on the same problem, all against one reference."""
    from d9d_b200.kernel._native import FUSED_WGRAD_ATTR
    from d9d_b200.kernel.moe import grouped_linear
    from d9d_b200.kernel.swiglu import silu_mul_probs

    pb = Problem("skewed", 0, 1, 8, 136, 200, seed=5)
    _check("composed_fused_block", _run_block(pb),
           expert_block_ref(pb.xp, pb.pp, *pb.w, pb.seg, pb.dy, wgrad_dtype=torch.float32))
    gen = torch.Generator(device=DEV).manual_seed(7)
    for fused_owner in (False, True):
        ws = _params(pb.w, torch.float32)
        g0 = None
        if fused_owner:
            g0 = [torch.randn(p.shape, device=DEV, generator=gen) for p in ws]
            for p, gi in zip(ws, g0):
                p.grad = gi.clone()
                setattr(p, FUSED_WGRAD_ATTR, True)
        xp, pp = pb.xp.clone().requires_grad_(), pb.pp.clone().requires_grad_()
        h = silu_mul_probs(grouped_linear(xp, ws[0], pb.layout), grouped_linear(xp, ws[1], pb.layout), pp)
        y = grouped_linear(h, ws[2], pb.layout)
        y.backward(pb.dy)
        u = pb.used
        got = {"y": y.detach()[:u], "dx": xp.grad[:u], "dprobs": pp.grad[:u],
               **dict(zip(("dWg", "dWu", "dWd"), (w.grad for w in ws)))}
        ref = expert_block_ref(pb.xp, pb.pp, *pb.w, pb.seg, pb.dy, wgrad_dtype=torch.float32, g0=g0)
        _check("composed_fused_owner" if fused_owner else "composed", got, ref)


@pytest.mark.parametrize("case", ["flagship", "skewed"])
def test_expert_path_against_fp64(ops, case):
    """moe_permute -> grouped_swiglu -> moe_unpermute with x and probs as leaves (dropped slots in the skewed case)."""
    from d9d_b200.kernel.moe import grouped_swiglu, moe_permute, moe_unpermute

    kind, T, k, E, H, F, _ = CASES[case]
    pb = Problem(kind, T, k, E, H, F, seed=6)
    x, probs = pb.x.clone().requires_grad_(), pb.probs.clone().requires_grad_()
    ws = _params(pb.w, torch.float32)
    xp, pp = moe_permute(x, probs, pb.layout)
    y = moe_unpermute(grouped_swiglu(xp, pp, *ws, pb.layout), pb.layout)
    dy = torch.randn(pb.T, H, device=DEV, generator=torch.Generator(device=DEV).manual_seed(8)).to(BF)
    y.backward(dy)
    got = {"y": y.detach(), "dx": x.grad, "dprobs": probs.grad, **dict(zip(("dWg", "dWu", "dWd"), (w.grad for w in ws)))}
    ref = expert_path_ref(pb.x, pb.probs, *pb.w, pb.layout.row_map, pb.seg, pb.cap, dy)
    _check(f"expert_path_{case}", got, ref)
    if case == "skewed":
        assert bool((probs.grad[pb.ids.to(DEV) < 0] == 0).all())


# ----------------------------------------------------------------------------- ep_push / ep_pull_sum on one GPU
W = 3
EP_H = [8, 256, 264, 768, 7168]
EP_K = [1, 8, 32]
EP_T = [0, 1, 1000, 20_000]
EP_BUDGET = 1 << 26  # T * k * H elements of routed rows per grid point: the largest pairs are skipped


class Peers:
    """W byte buffers filled with random canary bytes: rows at ``off_x`` ([rows, H] bf16), probabilities at ``off_p``
    ([rows] fp32, 4-byte but not 16-byte aligned), and the device table of their base pointers."""

    def __init__(self, rows: int, H: int, gen: torch.Generator):
        self.rows, self.H = rows, H
        self.off_x = 48
        self.off_p = (self.off_x + rows * H * 2 + 64) // 16 * 16 + 4
        size = self.off_p + rows * 4 + 40
        self.bufs = [torch.randint(0, 256, (size,), dtype=torch.uint8, device=DEV, generator=gen) for _ in range(W)]
        self.table = torch.tensor([b.data_ptr() for b in self.bufs], dtype=torch.int64, device=DEV)

    def x(self, r: int) -> torch.Tensor:
        return self.bufs[r][self.off_x : self.off_x + self.rows * self.H * 2].view(BF).view(self.rows, self.H)

    def p(self, r: int) -> torch.Tensor:
        return self.bufs[r][self.off_p : self.off_p + self.rows * 4].view(torch.float32)


def _plan(T: int, k: int, gen: torch.Generator):
    """A destination (rank, row) per (token, slot) pair, unique per rank, about 10 % dropped (row -1)."""
    n = T * k
    rank = torch.randint(0, W, (n,), generator=gen, dtype=torch.int32)
    row = torch.full((n,), -1, dtype=torch.int32)
    keep = torch.rand(n, generator=gen) >= 0.1
    rows = max(1, n)
    for r in range(W):
        sel = (rank == r) & keep
        row[sel] = torch.randperm(rows, generator=gen)[: int(sel.sum())].int()
    return rank, row, rows


def _ep_grid():
    return [(H, k, T) for H in EP_H for k in EP_K for T in EP_T if T * k * H <= EP_BUDGET]


@pytest.mark.parametrize("H,k,T", _ep_grid())
def test_ep_push_and_pull_sum(ops, H, k, T):
    gen = torch.Generator().manual_seed(H * 131 + k * 7 + T)
    ggen = torch.Generator(device=DEV).manual_seed(H + k + T)
    rank, row, rows = _plan(T, k, gen)
    rank_d, row_d = rank.to(DEV), row.to(DEV)
    peers = Peers(rows, H, ggen)
    x = torch.randn(T, H, device=DEV, generator=ggen).to(BF)
    probs = torch.rand(T * k, device=DEV, generator=ggen)

    # push with probabilities, then without: rows land bitwise at (rank, row), nothing else changes
    for with_p in (True, False):
        before = [b.clone() for b in peers.bufs]
        ops.ep_push(x, probs if with_p else None, rank_d, row_d, peers.table.data_ptr(), peers.off_x, peers.off_p, k)
        torch.cuda.synchronize()
        for r in range(W):
            exp = before[r].clone()
            sel = ((rank == r) & (row >= 0)).to(DEV)
            dst = row_d[sel].long()
            exp[peers.off_x : peers.off_x + rows * H * 2].view(BF).view(rows, H)[dst] = x.repeat_interleave(k, 0)[sel]
            if with_p:
                exp[peers.off_p : peers.off_p + rows * 4].view(torch.float32)[dst] = probs[sel]
            assert torch.equal(peers.bufs[r], exp), f"rank {r} (probs={with_p})"

    # pull-sum: the owners' rows hold finite values; y is the in-order fp32 sum of the kept slots rounded to bf16
    for r in range(W):
        peers.x(r).copy_(torch.randn(rows, H, device=DEV, generator=ggen).to(BF))
        peers.p(r).copy_(torch.randn(rows, device=DEV, generator=ggen))
    y, dprobs = ops.ep_pull_sum(peers.table.data_ptr(), peers.off_x, peers.off_p, rank_d, row_d, T, k, H, True)
    y2, none = ops.ep_pull_sum(peers.table.data_ptr(), peers.off_x, peers.off_p, rank_d, row_d, T, k, H, False)
    src_x = torch.stack([peers.x(r) for r in range(W)]).cpu()
    src_p = torch.stack([peers.p(r) for r in range(W)]).cpu()
    rk, rw = rank.long().reshape(T, k), row.long().reshape(T, k)
    acc = torch.zeros(T, H, dtype=torch.float32)
    for j in range(k):
        kept = rw[:, j] >= 0
        acc[kept] += src_x[rk[kept, j], rw[kept, j]].float()
    dp_model = torch.where(rw >= 0, src_p[rk, rw.clamp_min(0)], torch.zeros(()))
    assert y.shape == (T, H) and y.dtype == BF
    assert torch.equal(y.cpu().view(torch.int16), acc.to(BF).view(torch.int16))
    assert torch.equal(y2, y)
    assert dprobs.shape == (T, k) and torch.equal(dprobs.cpu().view(torch.int32), dp_model.view(torch.int32))
    assert none.numel() == 0


def test_ep_refuses_bad_operands(ops):
    """Only conditions the host checks; every call is refused before a kernel is launched."""
    gen = torch.Generator().manual_seed(0)
    T, k, H = 16, 2, 64
    rank, row, rows = _plan(T, k, gen)
    rank, row = rank.to(DEV), row.to(DEV)
    peers = Peers(rows, H, torch.Generator(device=DEV).manual_seed(0))
    before = [b.clone() for b in peers.bufs]
    x = torch.randn(T, H, device=DEV).to(BF)
    probs = torch.rand(T * k, device=DEV)
    tbl, ox, op = peers.table.data_ptr(), peers.off_x, peers.off_p
    push_bad = [
        (torch.randn(T, 12, device=DEV).to(BF), probs, rank, row, ox, op),  # H % 8
        (x, probs, rank, row, ox + 8, op),  # off_x not 16-byte aligned
        (x, probs, rank, row, ox, op + 2),  # off_p not 4-byte aligned
        (x.float(), probs, rank, row, ox, op),  # dtype of x
        (x, probs, rank.long(), row, ox, op),  # dtype of dest_rank
        (x, probs, rank, row[:-1], ox, op),  # one destination per pair
        (x, probs[:-1], rank, row, ox, op),  # one probability per pair
        (x, probs.double(), rank, row, ox, op),  # probability dtype
    ]
    for xx, pr, rk, rw, a, b in push_bad:
        with pytest.raises(RuntimeError):
            ops.ep_push(xx, pr, rk, rw, tbl, a, b, k)
    pull_bad = [
        (ox, op, rank, row, T, k, 12),  # H % 8
        (ox + 8, op, rank, row, T, k, H),  # off_y not 16-byte aligned
        (ox, op + 2, rank, row, T, k, H),  # off_dp not 4-byte aligned
        (ox, op, rank, row, T, k + 1, H),  # one destination per pair
        (ox, op, rank.long(), row, T, k, H),  # dtype of dest_rank
    ]
    for a, b, rk, rw, t, kk, h in pull_bad:
        with pytest.raises(RuntimeError):
            ops.ep_pull_sum(tbl, a, b, rk, rw, t, kk, h, True)
    T33 = 4
    rank33 = torch.zeros(T33 * 33, dtype=torch.int32, device=DEV)
    row33 = torch.full((T33 * 33,), -1, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError):  # k > 32
        ops.ep_pull_sum(tbl, ox, op, rank33, row33, T33, 33, H, True)
    torch.cuda.synchronize()
    for b, b0 in zip(peers.bufs, before):
        assert torch.equal(b, b0)

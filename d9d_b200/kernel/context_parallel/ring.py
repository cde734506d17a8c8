"""Ring attention with an exact backward pass.

Every rank keeps its queries and, over ``world`` steps, sees every rank's K/V block once: while it computes attention of
its queries against the block it holds it already exchanges blocks with its ring neighbours.  Per-block results
``(out_b, lse_b)`` are merged on the fly (``lse = logaddexp(lse, lse_b)``, outputs re-weighted by ``exp(lse_b - lse)``),
which is algebraically the softmax over the whole sequence.  The backward pass runs the same ring once more: with the
saved global ``lse`` each block's probabilities are recomputed exactly, ``dQ`` accumulates locally and the ``dK / dV``
accumulators travel with their K/V block until they are back at its owner.

Masking is by *global token positions* (a ``[world, S_local]`` table of which tokens every rank holds), so any sharding
layout works; block pairs that are entirely masked (frequent with the zig-zag layout) are skipped, entirely visible ones
run unmasked.  The table lives on the host: which blocks to skip is decided without touching the device.

Block attention has two implementations:

* ``plan`` (CUDA default when the native flash kernels support the tensors): every rank's tokens are split into *runs* of
  consecutive global positions (one run for the contiguous layout, two for zig-zag); a (query run, key run) pair is then
  either fully visible, causal with aligned diagonals, or invisible, so a block is a handful of calls of the native
  wgmma flash-attention forward / backward kernels (``ops/csrc/flash_attn.cu``) on row slices - per-call ``(out, lse)``
  are merged exactly like whole blocks are, and the backward kernels take the *global* ``out`` / ``lse`` rows.  No score
  matrix is materialised.
* ``mask`` (CPU, layouts whose run pairs overlap partially, tensors the kernels do not take): PyTorch matmuls over a
  boolean position mask, queries scored in chunks.
"""

from __future__ import annotations

from typing import Any

import torch
import torch.distributed as dist
from torch.autograd import Function

_NEG_INF = float("-inf")


def _exchange(tensors: list[torch.Tensor], group: dist.ProcessGroup) -> tuple[list[torch.Tensor], list[dist.Work]]:
    """Start sending ``tensors`` to the next rank of the ring and receiving the previous rank's into fresh buffers."""
    world, rank = group.size(), group.rank()
    nxt, prv = (rank + 1) % world, (rank - 1) % world
    received = [torch.empty_like(t, memory_format=torch.contiguous_format) for t in tensors]  # irecv needs dense buffers
    ops = [dist.P2POp(dist.isend, t.contiguous(), group=group, group_peer=nxt) for t in tensors]
    ops += [dist.P2POp(dist.irecv, r, group=group, group_peer=prv) for r in received]
    return received, dist.batch_isend_irecv(ops)


def _wait(works: list[dist.Work]) -> None:
    for w in works:
        w.wait()


class _Masks:
    """Visibility of (my queries, rank ``src``'s keys) derived from the host-side position table; device masks of the
    partially visible pairs are built once and cached by the caller."""

    def __init__(self, positions: torch.Tensor, rank: int, causal: bool, device: torch.device, cache: dict | None):
        self._pos, self._rank, self._causal, self._device = positions, rank, causal, device
        self._cache = cache if cache is not None else {}

    def get(self, src: int) -> torch.Tensor | None | bool:
        """``None``: everything visible, ``False``: nothing visible, tensor: boolean ``[Sq, Sk]`` mask."""
        if not self._causal:
            return None
        pos_q, pos_k = self._pos[self._rank], self._pos[src]
        if int(pos_k.min()) > int(pos_q.max()):
            return False  # block lies entirely in the future
        if int(pos_k.max()) <= int(pos_q.min()):
            return None  # block lies entirely in the past
        key = (self._rank, src, str(self._device))
        mask = self._cache.get(key)
        if mask is None:
            mask = self._cache[key] = (pos_k[None, :] <= pos_q[:, None]).to(self._device)
        return mask


def _expand_heads(t: torch.Tensor, groups: int) -> torch.Tensor:
    return t if groups == 1 else t.repeat_interleave(groups, dim=2)


_QUERY_CHUNK = 2048  # queries scored at a time against one K/V block: bounds the fp32 score tile to [B, H, 2048, S_block]


def _query_chunks(length: int) -> list[slice]:
    return [slice(lo, min(lo + _QUERY_CHUNK, length)) for lo in range(0, length, _QUERY_CHUNK)]


def _block_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, mask: torch.Tensor | None
                   ) -> tuple[torch.Tensor, torch.Tensor]:
    """``(out [B,Sq,H,Dv] fp32, lse [B,H,Sq] fp32)`` of attention against one K/V block."""
    groups = q.shape[2] // k.shape[2]
    kf, vf = _expand_heads(k, groups).float(), _expand_heads(v, groups).float()
    outs, lses = [], []
    for rows in _query_chunks(q.shape[1]):
        scores = torch.einsum("bqhd,bkhd->bhqk", q[:, rows].float(), kf) * scale
        if mask is not None:
            scores = scores.masked_fill(~mask[rows], _NEG_INF)
        lse = torch.logsumexp(scores, dim=-1)
        probs = torch.exp(scores - lse.unsqueeze(-1).nan_to_num(neginf=0.0))  # rows without visible keys: exp(-inf) = 0
        outs.append(torch.einsum("bhqk,bkhd->bqhd", probs, vf))
        lses.append(lse)
    return torch.cat(outs, dim=1), torch.cat(lses, dim=2)


def _merge(out: torch.Tensor | None, lse: torch.Tensor | None, out_b: torch.Tensor, lse_b: torch.Tensor
           ) -> tuple[torch.Tensor, torch.Tensor]:
    if out is None or lse is None:
        return out_b, lse_b
    new_lse = torch.logaddexp(lse, lse_b)
    safe = new_lse.nan_to_num(neginf=0.0)  # both -inf -> weights exp(-inf - 0) = 0
    w_old = torch.exp(lse - safe).transpose(1, 2).unsqueeze(-1)  # [B,Sq,H,1]
    w_new = torch.exp(lse_b - safe).transpose(1, 2).unsqueeze(-1)
    return out * w_old + out_b * w_new, new_lse


def _block_backward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, grad_out: torch.Tensor, lse: torch.Tensor,
                    delta: torch.Tensor, scale: float, mask: torch.Tensor | None
                    ) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Gradients of one block given the *global* ``lse`` and ``delta = rowsum(dO * O)``: ``(dq, dk, dv)`` in fp32."""
    groups = q.shape[2] // k.shape[2]
    kf, vf = _expand_heads(k, groups).float(), _expand_heads(v, groups).float()
    dk, dv = torch.zeros_like(kf), torch.zeros_like(vf)
    dqs = []
    for rows in _query_chunks(q.shape[1]):
        qf, gf = q[:, rows].float(), grad_out[:, rows].float()
        scores = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
        if mask is not None:
            scores = scores.masked_fill(~mask[rows], _NEG_INF)
        probs = torch.exp(scores - lse[:, :, rows].unsqueeze(-1).nan_to_num(neginf=0.0))
        dv += torch.einsum("bhqk,bqhd->bkhd", probs, gf)
        dprobs = torch.einsum("bqhd,bkhd->bhqk", gf, vf)
        dscores = probs * (dprobs - delta[:, :, rows].unsqueeze(-1)) * scale
        dqs.append(torch.einsum("bhqk,bkhd->bqhd", dscores, kf))
        dk += torch.einsum("bhqk,bqhd->bkhd", dscores, qf)
    dq = torch.cat(dqs, dim=1)
    if groups > 1:
        b, sk, _, d = dk.shape
        dk = dk.view(b, sk, k.shape[2], groups, d).sum(3)
        dv = dv.view(b, sk, v.shape[2], groups, dv.shape[-1]).sum(3)
    return dq, dk, dv


# ------------------------------------------------------------------------------------------------------------------
# "plan" implementation: a block as calls of a flash-attention kernel on runs of consecutive positions
# ------------------------------------------------------------------------------------------------------------------
_FULL, _CAUSAL = 0, 1


def _position_runs(row: torch.Tensor) -> list[tuple[int, int, int]]:
    """Maximal runs of consecutive global positions in a rank's (host) position row: ``(first index, length, first position)``."""
    vals = row.tolist()
    runs, start = [], 0
    for i in range(1, len(vals) + 1):
        if i == len(vals) or vals[i] != vals[i - 1] + 1:
            runs.append((start, i - start, vals[start]))
            start = i
    return runs


class _BlockPlan:
    """Calls that make up attention of my queries against rank ``src``'s keys: ``(q_slice | None, k_slice | None, mode)`` with
    ``None`` = the whole block (no copy); ``calls(src)`` is ``None`` when a run pair overlaps partially (use the mask path)."""

    def __init__(self, positions: torch.Tensor, rank: int, causal: bool):
        self._runs = [_position_runs(positions[r]) for r in range(positions.shape[0])]
        self._rank, self._causal = rank, causal
        self._memo: dict[int, list[tuple[slice | None, slice | None, int]] | None] = {}

    def calls(self, src: int) -> list[tuple[slice | None, slice | None, int]] | None:
        if src not in self._memo:
            self._memo[src] = self._build(src)
        return self._memo[src]

    def _build(self, src: int) -> list[tuple[slice | None, slice | None, int]] | None:
        if not self._causal:
            return [(None, None, _FULL)]
        q_runs, k_runs = self._runs[self._rank], self._runs[src]
        rows: list[list[int | None]] = []
        for _qi, ql, qp in q_runs:
            row: list[int | None] = []
            for _ki, kl, kp in k_runs:
                if kp + kl - 1 <= qp:
                    row.append(_FULL)
                elif kp > qp + ql - 1:
                    row.append(None)
                elif kp == qp and kl == ql:
                    row.append(_CAUSAL)
                else:
                    return None  # partial overlap: not expressible as full / aligned-causal calls
            rows.append(row)
        if all(m == _FULL for row in rows for m in row):
            return [(None, None, _FULL)]

        def q_slice(i: int) -> slice | None:
            return None if len(q_runs) == 1 else slice(q_runs[i][0], q_runs[i][0] + q_runs[i][1])

        def k_slice(j: int) -> slice | None:
            return None if len(k_runs) == 1 else slice(k_runs[j][0], k_runs[j][0] + k_runs[j][1])

        out: list[tuple[slice | None, slice | None, int]] = []
        open_rows = list(range(len(q_runs)))
        # a query run that sees the whole block unmasked: one call over all keys (their order is irrelevant without a mask)
        for i in list(open_rows):
            if all(m == _FULL for m in rows[i]):
                out.append((q_slice(i), None, _FULL))
                open_rows.remove(i)
        # a key run that every remaining query run sees unmasked (and nothing else is visible to them): one call over those queries
        if len(open_rows) == len(q_runs):
            for j in range(len(k_runs)):
                if all(rows[i][j] == _FULL for i in open_rows) and all(rows[i][jj] is None for i in open_rows for jj in range(len(k_runs)) if jj != j):
                    return [*out, (None, k_slice(j), _FULL)]
        for i in open_rows:
            for j, m in enumerate(rows[i]):
                if m is not None:
                    out.append((q_slice(i), k_slice(j), m))
        return out


def _take(t: torch.Tensor, rows: slice | None) -> torch.Tensor:
    return t if rows is None else t[:, rows].contiguous()


def _attend_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, mode: int) -> tuple[torch.Tensor, torch.Tensor]:
    """``(out [B,Sq,H,Dv], lse [B,H,Sq] fp32)`` of one call: the native kernel on CUDA, the fp32 oracle elsewhere."""
    if q.is_cuda:
        from d9d_b200.kernel._native import native_ops

        out, lse = native_ops().flash_attn_fwd(q.contiguous(), k.contiguous(), v.contiguous(), scale, -1, 0 if mode == _CAUSAL else -1,
                                               0.0, None, None, None, 0, 0)
        return out, lse
    from d9d_b200.kernel.flash_attn.function import attention_reference

    return attention_reference(q, k, v, scale, causal=mode == _CAUSAL)


def _attend_backward(grad_out, q, k, v, out, lse, delta, scale: float, mode: int):
    """``(dq, dk, dv)`` of one call given the rows of the *global* output / lse (and, off the GPU, delta)."""
    if q.is_cuda:
        from d9d_b200.kernel._native import native_ops

        dq, dk, dv, _ = native_ops().flash_attn_bwd(grad_out.contiguous(), q.contiguous(), k.contiguous(), v.contiguous(), out.contiguous(),
                                                    lse.contiguous(), scale, -1, 0 if mode == _CAUSAL else -1, 0.0, None, None, 0, 0, None)
        return dq, dk, dv
    mask = None
    if mode == _CAUSAL:
        mask = torch.ones(q.shape[1], k.shape[1], dtype=torch.bool, device=q.device).tril()
    return _block_backward(q, k, v, grad_out, lse, delta, scale, mask)


def _plan_forward(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, calls) -> tuple[torch.Tensor, torch.Tensor]:
    """Block result ``(out fp32 [B,Sq,H,Dv], lse fp32 [B,H,Sq])``; query rows that see nothing in this block get ``lse = -inf``."""
    if len(calls) == 1 and calls[0][0] is None:
        out, lse = _attend_forward(q, _take(k, calls[0][1]), _take(v, calls[0][1]), scale, calls[0][2])
        return out.float(), lse.float()
    b, sq, h = q.shape[:3]
    out = q.new_zeros((b, sq, h, v.shape[-1]), dtype=torch.float32)
    lse = q.new_full((b, h, sq), _NEG_INF, dtype=torch.float32)
    q_cache: dict[tuple[int, int] | None, torch.Tensor] = {}
    for qs, ks, mode in calls:
        key = None if qs is None else (qs.start, qs.stop)
        if key not in q_cache:
            q_cache[key] = _take(q, qs)
        o_c, l_c = _attend_forward(q_cache[key], _take(k, ks), _take(v, ks), scale, mode)
        rows = slice(None) if qs is None else qs
        o_m, l_m = _merge(out[:, rows], lse[:, :, rows], o_c.float(), l_c.float())
        out[:, rows], lse[:, :, rows] = o_m, l_m
    return out, lse


def _plan_backward(q, k, v, grad_out, out, lse, delta, scale: float, calls) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """``(dq, dk, dv)`` (fp32, block shaped) of one block: sums of the per-call gradients."""
    dq = torch.zeros_like(q, dtype=torch.float32)
    dk = torch.zeros_like(k, dtype=torch.float32)
    dv = torch.zeros_like(v, dtype=torch.float32)
    for qs, ks, mode in calls:
        qr = slice(None) if qs is None else qs
        kr = slice(None) if ks is None else ks
        dq_c, dk_c, dv_c = _attend_backward(_take(grad_out, qs), _take(q, qs), _take(k, ks), _take(v, ks), _take(out, qs),
                                            lse[:, :, qr], delta[:, :, qr], scale, mode)
        dq[:, qr] += dq_c.float()
        dk[:, kr] += dk_c.float()
        dv[:, kr] += dv_c.float()
    return dq, dk, dv


def _use_plan(block_impl: str, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor) -> bool:
    if block_impl == "plan":
        return True
    if block_impl == "mask" or not q.is_cuda:
        return False
    from d9d_b200.kernel.flash_attn.native import native_supported

    return native_supported(q, k, v)


class _RingAttention(Function):
    @staticmethod
    def forward(ctx: Any, q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, masks: _Masks, group: dist.ProcessGroup,
                scale: float, plan: _BlockPlan | None = None) -> torch.Tensor:
        world, rank = group.size(), group.rank()
        out: torch.Tensor | None = None
        lse: torch.Tensor | None = None
        block = [k.detach(), v.detach()]
        for step in range(world):
            if step + 1 < world:
                incoming, works = _exchange(block, group)  # overlaps with the attention below
            src = (rank - step) % world
            mask = masks.get(src)
            if mask is not False:
                calls = plan.calls(src) if plan is not None else None
                if calls is not None:
                    out_b, lse_b = _plan_forward(q.detach(), block[0], block[1], scale, calls)
                else:
                    out_b, lse_b = _block_forward(q.detach(), block[0], block[1], scale, mask)
                out, lse = _merge(out, lse, out_b, lse_b)
            if step + 1 < world:
                _wait(works)
                block = incoming
        if out is None or lse is None:  # cannot happen with a causal mask over real positions, but keep shapes right
            out = q.new_zeros((*q.shape[:3], v.shape[-1]), dtype=torch.float32)
            lse = q.new_full((q.shape[0], q.shape[2], q.shape[1]), _NEG_INF, dtype=torch.float32)
        result = out.to(q.dtype)
        ctx.save_for_backward(q, k, v, result, lse)
        ctx.group, ctx.scale, ctx.masks, ctx.plan = group, scale, masks, plan
        return result

    @staticmethod
    def backward(ctx: Any, grad_out: torch.Tensor):  # type: ignore[override]
        q, k, v, out, lse = ctx.saved_tensors
        group, world, rank = ctx.group, ctx.group.size(), ctx.group.rank()
        delta = (grad_out.float() * out.float()).sum(-1).transpose(1, 2)  # [B,H,Sq]
        dq = torch.zeros_like(q, dtype=torch.float32)
        # the K/V block travels together with the gradient accumulated for it so far
        block = [k, v, torch.zeros_like(k, dtype=torch.float32), torch.zeros_like(v, dtype=torch.float32)]
        for step in range(world):
            src = (rank - step) % world
            mask = ctx.masks.get(src)
            if mask is not False:
                calls = ctx.plan.calls(src) if ctx.plan is not None else None
                if calls is not None:
                    dq_b, dk_b, dv_b = _plan_backward(q, block[0], block[1], grad_out, out, lse, delta, ctx.scale, calls)
                else:
                    dq_b, dk_b, dv_b = _block_backward(q, block[0], block[1], grad_out, lse, delta, ctx.scale, mask)
                dq += dq_b
                block[2] = block[2] + dk_b
                block[3] = block[3] + dv_b
            if world == 1:
                break
            # after the last step one more hop brings every block's gradient home
            last = step + 1 == world
            incoming, works = _exchange(block[2:] if last else block, group)
            _wait(works)
            block = [*block[:2], *incoming] if last else incoming
        return dq.to(q.dtype), block[2].to(k.dtype), block[3].to(v.dtype), None, None, None, None


def ring_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, group: dist.ProcessGroup, positions: torch.Tensor,
                   softmax_scale: float | None = None, causal: bool = True, mask_cache: dict | None = None,
                   block_impl: str = "auto") -> torch.Tensor:
    """Attention of the local queries over the keys / values of *all* ranks of ``group``.  Differentiable.

    ``q [B, S_local, H, D]``, ``k / v [B, S_local, Hk, D(v)]`` (``H % Hk == 0``).  ``positions``: host int64
    ``[world, S_local]`` - row ``r`` holds the global positions of rank ``r``'s tokens
    (``torch.stack([local_sequence_indices(S, world, r, layout) for r in range(world)])``).  ``mask_cache``: optional dict
    reused across calls so that device masks are built once.  ``block_impl``: ``"auto"`` (flash kernels on runs of consecutive
    positions when the tensors qualify, see the module docstring), ``"plan"`` or ``"mask"``.
    """
    if q.shape[2] % k.shape[2] != 0:
        raise ValueError("the number of query heads must be a multiple of the number of key/value heads")
    if positions.shape != (group.size(), q.shape[1]):
        raise ValueError(f"positions must be [world, S_local] = {(group.size(), q.shape[1])}, got {tuple(positions.shape)}")
    scale = softmax_scale if softmax_scale is not None else q.shape[-1] ** -0.5
    host_positions = positions.cpu()
    masks = _Masks(host_positions, group.rank(), bool(causal), q.device, mask_cache)
    plan = _BlockPlan(host_positions, group.rank(), bool(causal)) if _use_plan(block_impl, q, k, v) else None
    return _RingAttention.apply(q, k, v, masks, group, float(scale), plan)

"""Fused linear + cross-entropy that never materialises ``[tokens, vocab]`` logits.

Replaces the reference's dependency on the cut-cross-entropy Triton kernels (``d9d/kernel/cce/cce.py:47-298``,
``main.py:119-225``) with epilogues of the hand-written wgmma GEMM:

* forward : logits tiles stay in registers; the epilogue reduces them to online-softmax partials and the target logit
  (bias and tanh soft-capping are applied in the same epilogue);
* backward: the vocabulary is walked in *column chunks*.  For a chunk ``C[v0:v1]`` of the classifier the logits are
  recomputed and the epilogue writes ``g * (softmax - onehot) * dsoftcap`` as bf16 into one reusable
  ``[tokens, v1 - v0]`` buffer, which feeds two more wgmma GEMMs: ``dE += dL @ C[v0:v1]`` (fp32 accumulation in the
  epilogue) and ``dC[v0:v1] = dL^T @ E`` (full reduction depth = all tokens, so every row of ``dC`` is written exactly
  once - straight into the pre-allocated gradient buffer when the gradient infrastructure provides one).
  Chunking over *columns* instead of tokens is what keeps the extra memory small (default 256 MiB instead of the
  5 GB bf16 ``dlogits`` a 16k x 151k problem would need) without paying a read-modify-write pass over ``dC`` per chunk.
* the classifier may be given as several row blocks (``SplitLanguageModellingHead`` keeps one weight per vocabulary
  split): every block is consumed in place - no ``torch.cat`` of the weights, no split of the gradient.
* label smoothing ``eps`` and the z-loss ``zeta`` regularise the per-token loss (see ``linear_cross_entropy``).  They run
  on their own epilogue instances (the forward also sums each row's logits when ``eps > 0``; the backward writes the
  regularised gradient); with both at 0 the plain kernels run.
"""

from __future__ import annotations

import math
import os

from collections.abc import Sequence
from typing import Any

import torch
from torch import nn
from torch.autograd import Function

from d9d_b200.core.autograd import GLOBAL_GRAD_CONTEXT, GradDirection

from .._native import fused_wgrad_buffer, fused_wgrad_owner, grad_dtype_of, native_ops, on_gpu

IGNORE_INDEX = -100
# Upper bound for the backward's scratch memory (bf16 dlogits chunk + fp32 dE accumulator).
_CHUNK_BYTES = int(os.environ.get("D9D_CCE_CHUNK_BYTES", 256 << 20))
_V_TILE = 128  # rows of dC produced by one GEMM m-tile
# escape hatch: concatenate the classifier blocks first (one extra copy of the weights, gradient split by autograd)
_CAT_SPLITS = os.environ.get("D9D_CCE_CAT_SPLITS", "0") == "1"


def linear_cross_entropy_reference(e, c, targets, bias=None, ignore_index=IGNORE_INDEX, softcap=None, label_smoothing=0.0,
                                   z_loss_coef=0.0):
    """Materialised-logits oracle: ``(loss[T], lse[T])`` with ``loss = cross_entropy(z, y, label_smoothing) + z_loss_coef
    * lse^2`` (0 at ignored targets); with both coefficients 0 the loss is the NLL."""
    logits = e.float() @ c.float().t()
    if bias is not None:
        logits = logits + bias.float()
    if softcap is not None:
        logits = torch.tanh(logits / softcap) * softcap
    lse = torch.logsumexp(logits, dim=-1)
    if label_smoothing == 0 and z_loss_coef == 0:
        nll = torch.nn.functional.cross_entropy(logits, targets, ignore_index=ignore_index, reduction="none")
        return nll, lse
    loss = torch.nn.functional.cross_entropy(logits, targets, ignore_index=ignore_index, reduction="none",
                                             label_smoothing=label_smoothing)
    loss = torch.where(targets == ignore_index, torch.zeros_like(loss), loss + z_loss_coef * lse * lse)
    return loss, lse


class _EmulatedOps:
    """PyTorch fp32 stand-ins with the exact semantics of the native ops used by ``_LinearCEFunction`` - lets the CPU
    suite exercise the chunk plan / offsets / accumulation flags of the real code path."""

    launches = 0

    @staticmethod
    def _logits(h, w, bias, softcap):
        z = h.float() @ w.float().t()
        if bias is not None:
            z = z + bias
        dz = torch.ones_like(z)
        if softcap > 0:
            th = torch.tanh(z / softcap)
            z, dz = softcap * th, 1 - th * th
        return z, dz

    def ce_forward_ex(self, h, w, target, ignore_index, bias=None, softcap=0.0, col_offset=0):
        z, _ = self._logits(h, w, bias, softcap)
        lse = torch.logsumexp(z, -1)
        local = target - col_offset
        inside = (target != ignore_index) & (local >= 0) & (local < w.shape[0])
        tgt_logit = torch.where(inside, z.gather(1, local.clamp(0, w.shape[0] - 1)[:, None])[:, 0], torch.zeros_like(lse))
        nll = torch.where(target == ignore_index, torch.zeros_like(lse), lse - tgt_logit)
        return nll, lse, tgt_logit

    def ce_forward_reg(self, h, w, target, ignore_index, bias=None, softcap=0.0, col_offset=0):
        nll, lse, tgt_logit = self.ce_forward_ex(h, w, target, ignore_index, bias, softcap, col_offset)
        return nll, lse, tgt_logit, self._logits(h, w, bias, softcap)[0].sum(-1)

    def ce_dlogits(self, h, w, target, lse, grad, out, ignore_index, bias=None, softcap=0.0, col_offset=0):
        self.ce_dlogits_reg(h, w, target, lse, grad, out, ignore_index, 0.0, 0.0, 1, bias, softcap, col_offset)

    def ce_dlogits_reg(self, h, w, target, lse, grad, out, ignore_index, z_loss_coef, label_smoothing, num_classes,
                       bias=None, softcap=0.0, col_offset=0):
        z, dz = self._logits(h, w, bias, softcap)
        p = torch.exp(z - lse[:, None]) * (1 + 2 * z_loss_coef * lse[:, None]) - label_smoothing / num_classes
        local = target - col_offset
        inside = (target != ignore_index) & (local >= 0) & (local < w.shape[0])
        rows = torch.nonzero(inside)[:, 0]
        p[rows, local[rows]] -= 1 - label_smoothing
        g = torch.where(target == ignore_index, torch.zeros_like(grad), grad)
        out.copy_((p * g[:, None] * dz).to(out.dtype))

    @staticmethod
    def gemm(a, b, d, a_mn, b_mn, accumulate):
        r = (a.float().t() if a_mn else a.float()) @ (b.float() if b_mn else b.float().t())
        d.copy_((d.float() + r if accumulate else r).to(d.dtype))


def plan_vocab_chunks(split_sizes: Sequence[int], tokens: int, hidden: int, budget_bytes: int, sm_count: int = 132,
                      ) -> tuple[list[tuple[int, int, int]], int, bool]:
    """Column chunks ``(split, row_begin, row_end)`` of the classifier for the backward pass.

    The scratch memory is ``tokens x width`` bf16 (dlogits) plus, when more than one chunk is needed, a
    ``tokens x hidden`` fp32 accumulator for ``dE``.  Within the budget the width is chosen so that the ``dC`` GEMM of a
    chunk (``width / 128`` m-tiles x ``ceil(hidden / 256)`` n-tiles, reduction over all tokens) fills whole waves of
    ``sm_count`` persistent CTAs.  Returns ``(chunks, buffer_width, needs_fp32_accumulator)``.
    """

    def up(x: int, m: int) -> int:
        return (x + m - 1) // m * m

    tokens = max(tokens, 1)
    largest = max(split_sizes)
    if len(split_sizes) == 1 and tokens * up(largest, 8) * 2 <= budget_bytes:
        return [(0, 0, largest)], up(largest, 8), False  # one piece: dE is stored directly, no accumulator
    avail = max(budget_bytes - tokens * hidden * 4, budget_bytes // 2)  # the dlogits chunk keeps at least half the budget
    max_width = max(2 * _V_TILE, (avail // (2 * tokens)) // _V_TILE * _V_TILE)
    max_width = min(max_width, up(largest, _V_TILE))
    n_tiles = max(1, math.ceil(hidden / 256))
    best_w, best_eff = max_width, -1.0
    top = max_width // _V_TILE
    for m_tiles in range(top, max(1, top * 3 // 4) - 1, -1):  # wider first: ties keep the wider chunk
        tiles = m_tiles * n_tiles
        eff = tiles / (math.ceil(tiles / sm_count) * sm_count)
        if eff > best_eff + 1e-9:
            best_eff, best_w = eff, m_tiles * _V_TILE
    chunks: list[tuple[int, int, int]] = []
    for i, size in enumerate(split_sizes):
        n = max(1, math.ceil(size / best_w))
        # equal chunks within a split (whole dC tiles) instead of full ones plus a sliver
        width = min(best_w, up(math.ceil(size / n), _V_TILE))
        for r0 in range(0, size, width):
            chunks.append((i, r0, min(r0 + width, size)))
    return chunks, best_w, len(chunks) > 1


def _sm_count(device: torch.device) -> int:
    if device.type == "cuda":
        return torch.cuda.get_device_properties(device).multi_processor_count
    return 132


class _LinearCEFunction(Function):
    """``(loss[T], lse[T], nll[T] | None)``: the per-token loss of ``e @ cat(weights)^T + bias`` (see
    ``linear_cross_entropy``), its log-sum-exp and, when the loss is regularised, the plain NLL (else ``None``: the loss
    is the NLL).

    Inputs after ``n_splits``: the ``n_splits`` classifier blocks, then per block the leaf parameter that owns a
    pre-allocated gradient buffer (``fused_wgrad_owner``; the block itself is then passed detached) or ``None``.
    """

    @staticmethod
    def forward(ctx: Any, e: torch.Tensor, targets: torch.Tensor, bias: torch.Tensor | None, ignore_index: int, softcap: float,
                emulate: bool, label_smoothing: float, z_loss_coef: float, n_splits: int, *blocks: torch.Tensor | None):
        weights, owners = blocks[:n_splits], blocks[n_splits:]
        ops = _EmulatedOps() if emulate else native_ops()
        bias32 = None if bias is None else bias.detach().float().contiguous()
        v0 = 0
        parts = []
        for w in weights:
            b = None if bias32 is None else bias32[v0 : v0 + w.shape[0]]
            if label_smoothing > 0:  # (nll, lse, tgt_logit, zsum): the smoothing term needs the row's logit sum
                parts.append(ops.ce_forward_reg(e, w, targets, ignore_index, b, softcap, v0))
            else:
                parts.append(ops.ce_forward_ex(e, w, targets, ignore_index, b, softcap, v0))
            v0 += w.shape[0]
        if n_splits == 1:
            nll, lse = parts[0][:2]
        else:
            lse = torch.logsumexp(torch.stack([p[1] for p in parts]), dim=0)
            tgt_logit = torch.stack([p[2] for p in parts]).sum(0)
            nll = torch.where(targets == ignore_index, torch.zeros_like(lse), lse - tgt_logit)
        regularised = label_smoothing > 0 or z_loss_coef > 0
        loss = nll
        if regularised:
            reg = z_loss_coef * lse * lse
            if label_smoothing > 0:
                zsum = parts[0][3] if n_splits == 1 else torch.stack([p[3] for p in parts]).sum(0)
                reg = reg + label_smoothing * (lse - zsum / v0)
            loss = torch.where(targets == ignore_index, torch.zeros_like(lse), (1 - label_smoothing) * nll + reg)
        ctx.save_for_backward(e, targets, lse, bias32, *weights)
        ctx.owners = owners
        ctx.ignore_index, ctx.softcap, ctx.emulate, ctx.n_splits = ignore_index, softcap, emulate, n_splits
        ctx.label_smoothing, ctx.z_loss_coef, ctx.regularised = label_smoothing, z_loss_coef, regularised
        ctx.bias_dtype = None if bias is None else bias.dtype
        ctx.mark_non_differentiable(lse)
        if not regularised:
            return nll, lse, None
        ctx.mark_non_differentiable(nll)
        return loss, lse, nll

    @staticmethod
    def backward(ctx: Any, grad_loss: torch.Tensor, _grad_lse: torch.Tensor, _grad_nll: torch.Tensor | None):  # type: ignore[override]
        e, targets, lse, bias32, *weights = ctx.saved_tensors
        n = ctx.n_splits
        ops = _EmulatedOps() if ctx.emulate else native_ops()
        T, K = e.shape
        w_base = 9  # position of the first classifier block among the forward inputs
        dir_w = GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.weight)
        need_e = ctx.needs_input_grad[0] and GLOBAL_GRAD_CONTEXT.check_direction(GradDirection.inputs)
        need_b = bias32 is not None and ctx.needs_input_grad[2] and dir_w
        fused = [ctx.owners[i] is not None and ctx.needs_input_grad[w_base + n + i] and dir_w for i in range(n)]
        plain = [ctx.owners[i] is None and ctx.needs_input_grad[w_base + i] and dir_w for i in range(n)]
        g = grad_loss.float().contiguous()

        chunks, width, multi = plan_vocab_chunks([w.shape[0] for w in weights], T, K, _CHUNK_BYTES, _sm_count(e.device))
        buf = torch.empty(T, width, device=e.device, dtype=torch.bfloat16)
        de_acc = None
        if need_e:
            de_acc = torch.empty(T, K, device=e.device, dtype=torch.float32 if multi else e.dtype)
        dcs: list[torch.Tensor | None] = [
            torch.empty(w.shape, device=w.device, dtype=grad_dtype_of(w)) if plain[i] else None for i, w in enumerate(weights)
        ]
        dbias = torch.empty(bias32.shape, device=e.device, dtype=torch.float32) if need_b else None
        starts = [0]
        for w in weights:
            starts.append(starts[-1] + w.shape[0])

        first = True
        for i, r0, r1 in chunks:
            if not (need_e or need_b or fused[i] or plain[i]):
                continue
            w = weights[i][r0:r1]
            dl = buf[:, : r1 - r0]
            col0 = starts[i] + r0
            b = None if bias32 is None else bias32[col0 : col0 + (r1 - r0)]
            if ctx.regularised:
                ops.ce_dlogits_reg(e, w, targets, lse, g, dl, ctx.ignore_index, ctx.z_loss_coef, ctx.label_smoothing,
                                   starts[-1], b, ctx.softcap, col0)
            else:
                ops.ce_dlogits(e, w, targets, lse, g, dl, ctx.ignore_index, b, ctx.softcap, col0)
            if need_e:
                ops.gemm(dl, w, de_acc, False, True, not first)  # dE (+)= dL[T, v] @ C[v, K]
            if fused[i]:
                ops.gemm(dl, e, fused_wgrad_buffer(ctx.owners[i])[r0:r1], True, True, True)  # grad[v0:v1] += dL^T @ E
            elif plain[i]:
                ops.gemm(dl, e, dcs[i][r0:r1], True, True, False)  # dC[v0:v1] = dL^T @ E
            if need_b:
                dbias[col0 : col0 + (r1 - r0)] = dl.float().sum(0)
            first = False
        de = None
        if need_e:
            de = de_acc if de_acc.dtype == e.dtype else de_acc.to(e.dtype)
        db = None if dbias is None else dbias.to(ctx.bias_dtype)
        return (de, None, db, None, None, None, None, None, None, *dcs, *([None] * n))


class _LossSums(Function):
    """Identity on the per-token loss whose backward adds ``(sum nll, sum lse^2, count)`` over the non-ignored tokens to
    ``sums``: a forward recomputed for its backward (activation checkpointing) counts once."""

    @staticmethod
    def forward(ctx: Any, loss: torch.Tensor, nll: torch.Tensor, lse: torch.Tensor, valid: torch.Tensor, sums: torch.Tensor):
        ctx.save_for_backward(nll, lse, valid)
        ctx.sums = sums
        return loss.view_as(loss)

    @staticmethod
    def backward(ctx: Any, grad: torch.Tensor):  # type: ignore[override]
        nll, lse, valid = ctx.saved_tensors
        with torch.no_grad():
            zero = torch.zeros((), dtype=torch.float32, device=nll.device)
            ctx.sums.add_(torch.stack([torch.where(valid, nll.float(), zero).sum(),
                                       torch.where(valid, lse.float().square(), zero).sum(), valid.sum().float()]))
        return grad, None, None, None, None


def _native_eligible(e2: torch.Tensor, weights: Sequence[torch.Tensor]) -> bool:
    return e2.dtype == torch.bfloat16 and e2.shape[-1] % 8 == 0 and all(w.shape[1] == e2.shape[1] for w in weights)


def linear_cross_entropy(
    e: torch.Tensor,
    c: torch.Tensor | Sequence[torch.Tensor],
    targets: torch.Tensor,
    bias: torch.Tensor | None = None,
    ignore_index: int = IGNORE_INDEX,
    softcap: float | None = None,
    reduction: str = "mean",
    shift: bool | int = 0,
    return_lse: bool = False,
    _emulate: bool = False,
    label_smoothing: float = 0.0,
    z_loss_coef: float = 0.0,
    *,
    loss_sums: torch.Tensor | None = None,
    **_unused: Any,
) -> torch.Tensor | tuple[torch.Tensor, torch.Tensor]:
    """``cross_entropy(e @ c^T (+ bias), targets, label_smoothing) + z_loss_coef * lse^2`` with
    ``reduction in {none, mean, sum}``.

    ``e``: ``[..., K]`` embeddings; ``c``: ``[V, K]`` classifier or a sequence of row blocks of it (consumed in place);
    ``targets``: ``[...]`` int64.  ``shift=n`` drops the last ``n`` embeddings / first ``n`` targets along the sequence
    dim (causal LM shift).  ``softcap`` applies ``softcap * tanh(logits / softcap)``.  CCE's gradient-filtering options
    of the reference are accepted and ignored (gradients are exact).

    Per token, with ``z`` the logits after bias and soft-cap over all ``V`` classes, ``lse = logsumexp(z)``, ``eps =
    label_smoothing`` and ``zeta = z_loss_coef``: ``loss = (1 - eps) (lse - z_y) + eps (lse - mean_j z_j) + zeta lse^2``,
    0 at ignored targets (``F.cross_entropy(z, y, label_smoothing=eps) + zeta lse^2``).  ``mean`` divides by the number
    of non-ignored targets.  With both coefficients 0 this is the plain NLL, computed by the same kernels as without them.
    ``loss_sums`` (fp32 ``[3]``, optional) accumulates ``(sum nll, sum lse^2, count)`` over the non-ignored tokens,
    with the unsmoothed NLL, in backward (a recomputed forward counts once).
    """
    if not (0.0 <= label_smoothing <= 1.0):
        raise ValueError(f"label_smoothing must lie in [0, 1], got {label_smoothing}")
    if not (0.0 <= z_loss_coef < math.inf):
        raise ValueError(f"z_loss_coef must be finite and >= 0, got {z_loss_coef}")
    label_smoothing, z_loss_coef = float(label_smoothing), float(z_loss_coef)
    if loss_sums is not None and (loss_sums.dtype != torch.float32 or loss_sums.shape != (3,) or loss_sums.device != e.device):
        raise ValueError("loss_sums must be an fp32 [3] tensor on the embeddings' device")
    if isinstance(shift, bool):
        shift = int(shift)
    if shift:
        e = e[..., :-shift, :]
        targets = targets[..., shift:]
    blocks = [c] if isinstance(c, torch.Tensor) else list(c)
    if len(blocks) > 1 and _CAT_SPLITS:
        blocks = [torch.cat(blocks, dim=0)]
    lead_shape = targets.shape
    e2 = e.reshape(-1, e.shape[-1])
    t1 = targets.reshape(-1)
    if (on_gpu(e) or _emulate) and e2.numel() > 0:
        if not _emulate and not _native_eligible(e2, blocks):
            raise RuntimeError(
                f"d9d_b200.linear_cross_entropy: the native kernel needs bf16 embeddings with hidden % 8 == 0 (got {e2.dtype}, "
                f"{tuple(e2.shape)}); use linear_cross_entropy_reference explicitly for other inputs"
            )
        ws: list[torch.Tensor] = []
        owners: list[torch.Tensor | None] = []
        for w in blocks:
            owner = None if _emulate else fused_wgrad_owner(w)
            wl = w if w.dtype == e2.dtype else w.to(e2.dtype)
            ws.append((wl.detach() if owner is not None else wl).contiguous())
            owners.append(owner)
        nll, lse, plain_nll = _LinearCEFunction.apply(e2.contiguous(), t1.contiguous(), bias, ignore_index,
                                                      float(softcap or 0.0), _emulate, label_smoothing, z_loss_coef, len(ws),
                                                      *ws, *owners)
    else:
        full = blocks[0] if len(blocks) == 1 else torch.cat(blocks, dim=0)
        nll, lse = linear_cross_entropy_reference(e2, full, t1, bias, ignore_index, softcap, label_smoothing, z_loss_coef)
        plain_nll = None
        if loss_sums is not None and (label_smoothing > 0 or z_loss_coef > 0):
            with torch.no_grad():
                plain_nll = linear_cross_entropy_reference(e2, full, t1, bias, ignore_index, softcap)[0]
    if loss_sums is not None:
        plain_nll = nll if plain_nll is None else plain_nll
        nll = _LossSums.apply(nll, plain_nll.detach(), lse.detach(), t1 != ignore_index, loss_sums)
    if reduction == "none":
        loss = nll.view(lead_shape)
    elif reduction == "sum":
        loss = nll.sum()
    elif reduction == "mean":
        loss = nll.sum() / (t1 != ignore_index).sum().clamp_min(1)
    else:
        raise ValueError(f"unknown reduction {reduction!r}")
    if return_lse:
        return loss, lse.view(lead_shape)
    return loss


class LinearCrossEntropy(nn.Module):
    """Module wrapper with stored options (reference ``d9d/kernel/cce/main.py:228-282``)."""

    def __init__(self, ignore_index: int = IGNORE_INDEX, softcap: float | None = None, reduction: str = "mean",
                 shift: bool | int = 0, label_smoothing: float = 0.0, z_loss_coef: float = 0.0, **kwargs: Any):
        super().__init__()
        self.ignore_index, self.softcap, self.reduction, self.shift = ignore_index, softcap, reduction, shift
        self.label_smoothing, self.z_loss_coef = label_smoothing, z_loss_coef
        self.kwargs = kwargs

    def forward(self, e: torch.Tensor, c: torch.Tensor, targets: torch.Tensor, bias: torch.Tensor | None = None):
        return linear_cross_entropy(e, c, targets, bias=bias, ignore_index=self.ignore_index, softcap=self.softcap,
                                    reduction=self.reduction, shift=self.shift, label_smoothing=self.label_smoothing,
                                    z_loss_coef=self.z_loss_coef)

from __future__ import annotations

import dataclasses
import os
from collections.abc import Iterable
from typing import Any

import torch
import torch.distributed as dist
from torch import nn
from torch.distributed.tensor import DTensor

from d9d_b200.internals.nvlink import SymmetricArena
from d9d_b200.kernel._native import EXTERNAL_GRAD_OWNER_ATTR, FUSED_WGRAD_ATTR, native_ops

_ALIGN = 8  # elements: 16-byte vectors of bf16 parameters / 32-byte pairs of fp32 gradient vectors


def _local(p: torch.Tensor) -> torch.Tensor:
    """The rank-local storage of a parameter (DTensor parameters keep it in ``_local_tensor``)."""
    return p._local_tensor if isinstance(p, DTensor) else p.data  # noqa: SLF001


class NvlinkShardedAdamW(torch.optim.Optimizer):
    """Data-parallel AdamW (stochastic rounding, bf16 parameters) whose gradient reduction, update and parameter
    broadcast are two kernels over NVLink / NVSwitch peer memory instead of an NCCL all-reduce plus a replicated
    optimizer step (kernels: ``ops/csrc/nvlink_optim.cu``).

    * all parameters live in one *symmetric* bf16 arena, all gradients in a symmetric fp32 arena
      (``param.data`` / ``param.grad`` become views; wgrad GEMMs accumulate into the arena in their epilogue);
    * the arenas are cut into equal chunks owned round-robin (chunk ``c`` belongs to rank ``c % world``); a rank keeps
      AdamW moments for its chunks only (optimizer state memory and optimizer work are divided by the replica count);
    * during backward, whenever the last accumulation of a *wave* of chunks has landed, every rank reduces the chunks it
      owns by reading its peers' gradient buffers over NVLink on a side stream (plain P2P loads by default - measured
      faster than ``multimem.ld_reduce`` at 2 and 8 GPUs; ``D9D_NVLINK_MULTIMEM=1`` selects the in-switch reduction) and
      accumulates the sum of squares for clipping;
    * ``step()``: scalar all-reduce of the norm -> device-side barrier -> AdamW on the owned chunks with the new bf16
      parameters stored into every replica's parameter arena -> zero the gradient arena -> barrier.  No NCCL call moves
      gradient or parameter data and the host never waits.

    Mathematically this equals the reference's "all-reduce gradients, then every replica runs the same optimizer"
    (``d9d/internals/grad_sync`` + ``d9d/optim/stochastic/adamw.py``); gradients are SUMmed, ``grad_scale`` (a device
    scalar, e.g. ``1 / sum(loss weights)``) and the clip coefficient are applied inside the update kernel.
    """

    def __init__(self, params: Iterable[nn.Parameter], group: dist.ProcessGroup, lr: float, betas: tuple[float, float] = (0.9, 0.999),
                 eps: float = 1e-8, weight_decay: float = 1e-2, state_dtype: torch.dtype = torch.bfloat16,
                 max_norm: float | None = None, seed: int = 0, chunk_numel: int = 1 << 24, overlap_waves: int = 8):
        groups_in = list(params)
        if groups_in and isinstance(groups_in[0], dict):  # torch-style parameter groups (e.g. no weight decay for norms)
            groups_in = [{**g, "params": [p for p in g["params"] if p.requires_grad]} for g in groups_in]
            groups_in = [g for g in groups_in if g["params"]]
            params = [p for g in groups_in for p in g["params"]]
        else:
            params = [p for p in groups_in if p.requires_grad]
            groups_in = params
        if not params:
            raise ValueError("NvlinkShardedAdamW needs at least one trainable parameter")
        if any(_local(p).dtype != torch.bfloat16 for p in params):
            raise ValueError("NvlinkShardedAdamW supports bf16 parameters only")
        super().__init__(groups_in, {"lr": lr, "betas": betas, "eps": eps, "weight_decay": weight_decay})
        self._group = group
        self._world = group.size()
        self._rank = group.rank()
        self._max_norm = max_norm
        self._seed = seed
        self._step_count = 0
        device = _local(params[0]).device

        # Ownership is interleaved: the arena is cut into equal chunks and chunk c belongs to rank c % world, so every
        # rank has something to reduce as soon as *any* region of the gradients is final (backward finishes the arena
        # back to front).  A rank's moments for chunk c live in local slot c // world.  With several parameter groups every
        # group starts on a whole row of chunks, so a chunk never mixes hyper-parameters.
        params = [p for g in self.param_groups for p in g["params"]]
        layout = plan_arena_layout([[_local(p).numel() for p in g["params"]] for g in self.param_groups], self._world, int(chunk_numel))
        offsets, total = layout.offsets, layout.total
        self._real_numel = layout.real_numel  # end of the last parameter (before padding to whole rows of chunks)
        self._chunk = layout.chunk
        self._numel = total
        self._rows = layout.rows  # chunks per rank
        self._row_group = layout.row_group  # parameter group of every row of chunks
        self._shard = self._rows * self._chunk

        self.param_arena = SymmetricArena(total, torch.bfloat16, device, group)
        self.grad_arena = SymmetricArena(total, torch.float32, device, group)
        self.param_arena.buffer.zero_()
        self.grad_arena.buffer.zero_()
        with torch.no_grad():
            for p, off in zip(params, offsets, strict=True):
                local = _local(p)
                view = self.param_arena.buffer[off : off + local.numel()].view(local.shape)
                view.copy_(local)
                gview = self.grad_arena.buffer[off : off + local.numel()].view(local.shape)
                p.grad_dtype = torch.float32
                if isinstance(p, DTensor):  # the parameter now lives in the symmetric arena; the DTensor wrapper stays valid
                    p._local_tensor.set_(view)  # noqa: SLF001
                    p.grad = DTensor.from_local(gview, p.device_mesh, p.placements, run_check=False)
                else:
                    p.data = view
                    p.grad = gview
                setattr(p, FUSED_WGRAD_ATTR, True)
                setattr(p, EXTERNAL_GRAD_OWNER_ATTR, self)
        self._param_ranges = [(off, off + _local(p).numel()) for p, off in zip(params, offsets, strict=True)]
        self._params_flat = params
        self.exp_avg = torch.zeros(self._shard, dtype=state_dtype, device=device)
        self.exp_avg_sq = torch.zeros(self._shard, dtype=state_dtype, device=device)
        self._sumsq = torch.zeros(1, dtype=torch.float32, device=device)
        self._scale = torch.ones(1, dtype=torch.float32, device=device)
        self.grad_scale: torch.Tensor | None = None  # optional device scalar multiplied into every gradient
        self.last_grad_norm: torch.Tensor | None = None
        # ---- overlap of the gradient reduction with the tail of backward (enabled by set_required_accumulations)
        self._num_waves = max(1, min(int(overlap_waves), self._rows))
        self._required: int | None = None
        self._hooks: list = []
        self._side: torch.cuda.Stream | None = None
        self._next_wave = 0
        self._reduced_rows = 0  # rows [rows - reduced_rows, rows) of this step are already reduced
        self._acc_counts: list[int] = []
        self._wave_pending: list[int] = []
        self._waves_of_param: list[list[int]] = []
        torch.cuda.synchronize(device)
        self.param_arena.barrier()

    # ------------------------------------------------------------------ chunk / wave geometry
    def _owned_range(self, row: int) -> tuple[int, int]:
        begin = (row * self._world + self._rank) * self._chunk
        return begin, begin + self._chunk

    def _wave_rows(self, wave: int) -> range:
        """Wave 0 covers the *last* rows of the arena (their gradients are final first)."""
        per = -(-self._rows // self._num_waves)
        hi = self._rows - wave * per
        return range(max(hi - per, 0), max(hi, 0))

    def set_required_accumulations(self, num_backward_calls: int | None) -> None:
        """Enable (``n`` backward passes make a gradient final) or disable (``None``) the overlap of the cross-replica
        reduction with backward.  With it, whenever all gradients of a wave of chunks are final the owner reduces them
        on a side stream (after a device-side barrier among the replicas) while backward continues."""
        for h in self._hooks:
            h.remove()
        self._hooks = []
        self._required = num_backward_calls
        if num_backward_calls is None:
            return
        row_span = self._chunk * self._world
        per = -(-self._rows // self._num_waves)
        self._waves_of_param = []
        for lo, hi in self._param_ranges:
            rows = range(lo // row_span, (max(hi, lo + 1) - 1) // row_span + 1)
            self._waves_of_param.append(sorted({(self._rows - 1 - r) // per for r in rows}))
        self._reset_readiness()
        index = {id(p): i for i, p in enumerate(self._params_flat)}
        self._hooks = [p.register_post_accumulate_grad_hook(lambda q, _i=index: self._on_grad_final(_i[id(q)])) for p in self._params_flat]

    def _reset_readiness(self) -> None:
        self._acc_counts = [0] * len(self._params_flat)
        self._wave_pending = [0] * self._num_waves
        for waves in self._waves_of_param:
            for w in waves:
                self._wave_pending[w] += 1
        self._next_wave = 0
        self._reduced_rows = 0

    def _on_grad_final(self, idx: int) -> None:
        self._acc_counts[idx] += 1
        if self._acc_counts[idx] != self._required:
            return
        for w in self._waves_of_param[idx]:
            self._wave_pending[w] -= 1
        while self._next_wave < self._num_waves and self._wave_pending[self._next_wave] == 0:
            self._launch_wave(self._next_wave)
            self._next_wave += 1

    def _reduce_rows(self, rows: range) -> None:
        ops = native_ops()
        mc = self.grad_arena.multicast_ptr if self.uses_multicast else 0
        for row in rows:
            begin, end = self._owned_range(row)
            ops.nvl_reduce_shard_(self.grad_arena.buffer, self.grad_arena.peer_ptrs_dev, mc, begin, end, self._world, self._rank, self._sumsq)

    def _launch_wave(self, wave: int) -> None:
        """Reduce the owned chunks of ``wave`` on the side stream; everything enqueued on the current stream so far
        (i.e. the kernels that produced these gradients) is ordered before it."""
        rows = self._wave_rows(wave)
        if self._side is None:
            self._side = torch.cuda.Stream(device=self._sumsq.device)
        ready = torch.cuda.Event()
        ready.record()
        self._side.wait_event(ready)
        with torch.cuda.stream(self._side):
            if self._reduced_rows == 0:
                self._sumsq.zero_()
            self.grad_arena.barrier()  # every replica finished the gradients of this wave
            self._reduce_rows(rows)
        self._reduced_rows += len(rows)

    @property
    def uses_multicast(self) -> bool:
        """NVSwitch multicast (``multimem``) path or explicit peer loads/stores (default).

        ``multimem.ld_reduce`` / ``multimem.st`` move fewer bytes *into* a GPU, but both phases are bound by what every
        GPU has to send / receive in total, so the plain peer loads / stores are the default (the two have not been
        compared on H100).  ``D9D_NVLINK_MULTIMEM=1`` selects the multicast path.
        """
        available = self.param_arena.multicast_ptr != 0 and self.grad_arena.multicast_ptr != 0
        return available and os.environ.get("D9D_NVLINK_MULTIMEM", "0") == "1"

    state_is_materialized = True  # nothing is created lazily: checkpoint loading needs no warm-up step

    @property
    def max_norm(self) -> float | None:
        return self._max_norm

    @max_norm.setter
    def max_norm(self, value: float | None) -> None:
        self._max_norm = value

    def set_grad_scale(self, scale: torch.Tensor) -> None:
        """Device scalar multiplied into every (reduced) gradient inside the update kernel, e.g. ``1/sum(weights)``."""
        if self.grad_scale is None:
            self.grad_scale = torch.ones(1, dtype=torch.float32, device=self._sumsq.device)
        self.grad_scale.copy_(scale.reshape(-1)[:1])

    @torch.no_grad()
    def step(self, closure: Any = None) -> None:  # type: ignore[override]
        if closure is not None:
            raise ValueError("closures are not supported")
        ops = native_ops()
        self._step_count += 1
        multicast = self.uses_multicast
        remaining = range(0, self._rows - self._reduced_rows)
        if self._reduced_rows > 0:
            # part of the arena was reduced while backward was still running; finish the rest behind it
            main = torch.cuda.current_stream()
            self._side.wait_stream(main)
            with torch.cuda.stream(self._side):
                if len(remaining) > 0:
                    self.grad_arena.barrier()
                    self._reduce_rows(remaining)
            main.wait_stream(self._side)
        else:
            self.grad_arena.barrier()  # every replica finished its backward; its gradients are visible
            self._sumsq.zero_()
            self._reduce_rows(remaining)
        scale = self.grad_scale if self.grad_scale is not None else None
        if self._max_norm is not None:
            dist.all_reduce(self._sumsq, group=self._group)
            norm = self._sumsq.sqrt()
            if scale is not None:
                norm = norm * scale
            self.last_grad_norm = norm
            clip = torch.clamp(self._max_norm / (norm + 1e-6), max=1.0)
            self._scale.copy_(clip if scale is None else clip * scale)
            scale = self._scale
        self.grad_arena.barrier()  # all replicas have read my gradients: they may be overwritten / zeroed
        mc_param = self.param_arena.multicast_ptr if multicast else 0
        for row in range(self._rows):
            group = self.param_groups[self._row_group[row]]  # a row of chunks never mixes parameter groups
            beta1, beta2 = group["betas"]
            begin, end = self._owned_range(row)
            slot = slice(row * self._chunk, (row + 1) * self._chunk)
            ops.nvl_adamw_shard_(self.param_arena.buffer, self.grad_arena.buffer, self.exp_avg[slot], self.exp_avg_sq[slot],
                                 self.param_arena.peer_ptrs_dev, mc_param, begin, end, self._world, self._rank,
                                 float(group["lr"]), beta1, beta2, group["eps"], group["weight_decay"],
                                 1.0 - beta1**self._step_count, 1.0 - beta2**self._step_count,
                                 self._seed + 7919 * self._step_count, scale)
        self.grad_arena.buffer.zero_()
        self.param_arena.barrier()  # every shard owner's parameter writes have landed here before the next forward
        if self._required is not None:
            self._reset_readiness()

    def zero_grad(self, set_to_none: bool = False) -> None:  # gradients are zeroed inside step()
        if set_to_none:
            raise ValueError("gradients alias the symmetric arena and cannot be set to None")
        self.grad_arena.buffer.zero_()

    def state_dict(self) -> dict[str, Any]:
        """Moments are stored per *global chunk* (``chunks/<chunk id>``), so a checkpoint does not depend on the number of
        replicas it was written with as long as the chunk size is the same (it is ``chunk_numel`` for every model with more
        than ``world * chunk_numel`` parameters): each rank saves the chunks it owns, and after a restart with another world
        size every rank asks for the chunks it owns *now*."""
        return {"chunks": chunk_state_views(self.exp_avg, self.exp_avg_sq, self._chunk, self._world, self._rank, self._real_numel),
                "chunk_numel": self._chunk, "numel": self._real_numel,
                "step": self._step_count, "param_groups": [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups]}

    def load_state_dict(self, state_dict: dict[str, Any]) -> None:
        if int(state_dict.get("chunk_numel", self._chunk)) != self._chunk:
            raise ValueError(f"checkpoint was written with chunk size {state_dict.get('chunk_numel')} but this run uses {self._chunk} "
                             "(small models derive the chunk size from the replica count): the ownership layout differs")
        legacy = f"shard_{self._rank}_of_{self._world}"
        if "chunks" in state_dict:
            load_chunk_state(state_dict["chunks"], self.exp_avg, self.exp_avg_sq, self._chunk, self._world, self._rank, self._real_numel)
        elif legacy in state_dict:  # format of the first round: one blob per (rank, world)
            self.exp_avg.copy_(state_dict[legacy]["exp_avg"])
            self.exp_avg_sq.copy_(state_dict[legacy]["exp_avg_sq"])
        else:
            raise KeyError("optimizer checkpoint has neither per-chunk moments nor a shard for this (rank, world)")
        self._step_count = int(state_dict["step"])
        for g, saved in zip(self.param_groups, state_dict["param_groups"], strict=True):
            g.update(saved)


@dataclasses.dataclass(frozen=True)
class ArenaLayout:
    offsets: list[int]      # element offset of every parameter (groups concatenated in order)
    chunk: int              # elements per chunk
    rows: int               # chunks per rank
    total: int              # arena elements (= rows * world * chunk)
    real_numel: int         # end of the last parameter
    row_group: list[int]    # parameter group owning each row of chunks


def plan_arena_layout(group_sizes: list[list[int]], world: int, chunk_numel: int) -> ArenaLayout:
    """Flat arena layout: parameters 8-element aligned, the arena cut into ``rows x world`` chunks of equal size.  A single
    group is laid out densely; with several groups each one starts on a row boundary (``world * chunk`` elements), so that
    every chunk has one set of hyper-parameters."""
    def aligned(n: int) -> int:
        return (n + _ALIGN - 1) // _ALIGN * _ALIGN

    dense_total = sum(aligned(n) for sizes in group_sizes for n in sizes)
    per_rank = -(-dense_total // world)
    chunk = max(1024, min(int(chunk_numel), -(-per_rank // 1024) * 1024))
    row = chunk * world
    offsets: list[int] = []
    row_group: list[int] = []
    total = real = 0
    for g, sizes in enumerate(group_sizes):
        start = total
        for n in sizes:
            offsets.append(total)
            real = total + n
            total += aligned(n)
        total = -(-total // row) * row if (len(group_sizes) > 1 or g == len(group_sizes) - 1) else total
        row_group += [g] * ((total - start) // row)
    return ArenaLayout(offsets=offsets, chunk=chunk, rows=total // row, total=total, real_numel=real, row_group=row_group)


def owned_real_chunks(chunk: int, world: int, rank: int, real_numel: int, rows: int) -> list[tuple[int, int]]:
    """``(global chunk id, local slot)`` of the chunks of ``rank`` that hold parameters (chunks past ``real_numel`` are padding
    of the arena to a multiple of ``world`` chunks)."""
    last = -(-real_numel // chunk)  # number of chunks that contain at least one real element
    return [(row * world + rank, row) for row in range(rows) if row * world + rank < last]


def chunk_state_views(exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, chunk: int, world: int, rank: int, real_numel: int
                      ) -> dict[str, dict[str, torch.Tensor]]:
    rows = exp_avg.numel() // chunk
    return {str(c): {"exp_avg": exp_avg[slot * chunk : (slot + 1) * chunk], "exp_avg_sq": exp_avg_sq[slot * chunk : (slot + 1) * chunk]}
            for c, slot in owned_real_chunks(chunk, world, rank, real_numel, rows)}


def load_chunk_state(chunks: dict[str, dict[str, torch.Tensor]], exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, chunk: int, world: int,
                     rank: int, real_numel: int) -> None:
    rows = exp_avg.numel() // chunk
    for c, slot in owned_real_chunks(chunk, world, rank, real_numel, rows):
        entry = chunks.get(str(c))
        if entry is None:
            raise KeyError(f"optimizer checkpoint lacks the moments of chunk {c}")
        exp_avg[slot * chunk : (slot + 1) * chunk].copy_(entry["exp_avg"])
        exp_avg_sq[slot * chunk : (slot + 1) * chunk].copy_(entry["exp_avg_sq"])

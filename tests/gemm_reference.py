"""fp64 reference and per-element error bound for the bf16 wgmma GEMMs, plus operand / output buffers that catch stray
reads and writes.  Pure torch: works on CPU tensors (self-test) and CUDA tensors alike.

Bound for d ~= A @ B (+ d0), with S = |A| @ |B| computed in fp64 from the tensors actually passed to the kernel:

    |d - ref| <= c_k * S                   fp32 accumulation over K (c_k = max(K / 16, 1) * 2^-22)
               + c_o * |ref|               rounding of the output (2^-8 for bf16, 2^-23 for fp32)
               + 2^-8 * |A @ B|            bf16 accumulate: the product is rounded to bf16 before it is added to d0
               + splits * 2^-23 * (S + |d0|)   fp32 accumulate: one rounded add per K slice, in any order
"""

from __future__ import annotations

import torch

U_BF16 = 2.0**-8
U_F32 = 2.0**-24
CANARY = {torch.bfloat16: -7168.0, torch.float32: -6.5e5}  # exactly representable


def ck(K: int) -> float:
    return max(K / 16.0, 1.0) * 2.0**-22


def matmul_ref(a: torch.Tensor, b: torch.Tensor, a_mn: bool, b_mn: bool) -> tuple[torch.Tensor, torch.Tensor]:
    """(A @ B, |A| @ |B|) in fp64. a: [M, K] or (a_mn) [K, M]; b: [N, K] or (b_mn) [K, N]."""
    A = a.double().t() if a_mn else a.double()
    B = b.double() if b_mn else b.double().t()
    return A @ B, A.abs() @ B.abs()


def gemm_bound(prod: torch.Tensor, S: torch.Tensor, K: int, out_dtype: torch.dtype, d0: torch.Tensor | None = None,
               k_splits: int = 1) -> tuple[torch.Tensor, torch.Tensor]:
    """(reference, bound) for d = prod (+ d0) computed by a kernel with fp32 accumulation over K."""
    ref = prod if d0 is None else prod + d0.double()
    bound = ck(K) * S
    if out_dtype == torch.bfloat16:
        bound = bound + U_BF16 * ref.abs()
        if d0 is not None:
            bound = bound + U_BF16 * prod.abs()
    else:
        bound = bound + 2 * U_F32 * ref.abs()
        if d0 is not None:
            bound = bound + k_splits * 2 * U_F32 * (S + d0.double().abs())
    return ref, bound


def err_ratio(d: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |d - ref| / bound; inf when d holds a NaN or Inf.  Elements with a zero bound must match exactly."""
    err = (d.double() - ref).abs()
    if not bool(torch.isfinite(err).all()):
        return float("inf")
    if err.numel() == 0:
        return 0.0
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, torch.inf, 0.0))
    return float(ratio.max())


def assert_within(d: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, what: str = "") -> float:
    r = err_ratio(d, ref, bound)
    if not r <= 1.0:
        err = (d.double() - ref).abs()
        bad = ~(err <= bound)
        idx = bad.nonzero()[:5].tolist()
        vals = [(i, float(d[tuple(i)]), float(ref[tuple(i)]), float(bound[tuple(i)])) for i in idx]
        raise AssertionError(f"{what}: err/bound = {r:.3g}, {int(bad.sum())} bad elements, first (index, got, ref, bound): {vals}")
    return r


# ----------------------------------------------------------------------------- buffers
def padded(rows: int, cols: int, pad: int, *, device, gen: torch.Generator | None = None, scale: float = 1.0) -> torch.Tensor:
    """bf16 [rows, cols] view with row pitch cols + pad; the padding holds NaN, so any read past `cols` poisons the result."""
    buf = torch.full((rows, cols + pad), float("nan"), device=device, dtype=torch.bfloat16)
    buf[:, :cols] = (torch.randn(rows, cols, device=device, generator=gen) * scale).bfloat16()
    return buf[:, :cols]


class Canaried:
    """An output view into a larger buffer filled with a canary value.

    tma=True: base 16-byte aligned and row pitch a multiple of 16 bytes (the TMA epilogue takes it when the row width is a
    multiple of 16 bytes too); tma=False: base one element past a 16-byte boundary and an odd row pitch (direct stores).
    """

    def __init__(self, rows: int, cols: int, dtype: torch.dtype, *, tma: bool, device, init: torch.Tensor | None = None):
        per16 = 16 // torch.empty((), dtype=dtype).element_size()
        c0 = per16 if tma else 1
        pitch = -(-(c0 + cols + per16) // per16) * per16
        if not tma:
            pitch += 1
        self.buf = torch.full((rows + 2, pitch), CANARY[dtype], device=device, dtype=dtype)
        self.view = self.buf[1 : rows + 1, c0 : c0 + cols]
        if init is not None:
            self.view.copy_(init)
        self.mask = torch.zeros(self.buf.shape, dtype=torch.bool, device=device)
        self.mask[1 : rows + 1, c0 : c0 + cols] = True
        self.before = self.buf.clone()

    def assert_untouched(self) -> None:
        int_t = torch.int16 if self.buf.element_size() == 2 else torch.int32
        outside = ~self.mask
        changed = (self.buf.view(int_t) != self.before.view(int_t)) & outside
        n = int(changed.sum())
        assert n == 0, f"{n} elements outside the output view were written, first at {changed.nonzero()[:4].tolist()}"


def shard_rows(full: torch.Tensor, world: int, block_rows: int) -> list[list[int]]:
    """Row index lists per rank for the blocked, rank-interleaved layout of the fused tensor-parallel GEMMs:
    row idx -> block b = idx // block_rows, owner b % world, local row (b // world) * block_rows + idx % block_rows."""
    rows = full.shape[0]
    assert rows % (world * block_rows) == 0
    owners: list[list[int]] = [[] for _ in range(world)]
    for blk in range(rows // block_rows):
        owners[blk % world].extend(range(blk * block_rows, (blk + 1) * block_rows))
    return owners

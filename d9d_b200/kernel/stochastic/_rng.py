from __future__ import annotations

import torch


def draw_seed(generator: torch.Generator | None) -> int:
    """One 31-bit seed per call from a CPU generator (no device sync)."""
    return int(torch.randint(0, 2**31 - 1, (1,), device="cpu", generator=generator).item())


def sr_round_reference(x: torch.Tensor, seed: int) -> torch.Tensor:
    """CPU oracle: unbiased stochastic rounding fp32 -> bf16 (different random stream than the CUDA kernel)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    bits = x.detach().float().cpu().contiguous().view(torch.int32)
    noise = torch.randint(0, 1 << 16, bits.shape, generator=g, dtype=torch.int32)
    finite = (bits & 0x7F800000) != 0x7F800000
    # a NaN whose payload lies only in the dropped low bits keeps a quiet bit, so it does not turn into an inf
    quiet = torch.where((bits & 0xFFFF) != 0, 0x00400000, 0).to(torch.int32)
    rounded = torch.where(finite, bits + noise, bits | quiet) & ~0xFFFF
    return rounded.view(torch.float32).to(torch.bfloat16).to(x.device)

"""ncu target: flash-attention forward + backward at the flagship shape (B8 S2048 16q/4kv D128 causal)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from d9d_b200 import ops as _ops

ops = _ops.load()
B, S, Hq, Hk, D = 8, 2048, 16, 4, 128
q = torch.randn(B, S, Hq, D, device="cuda").bfloat16()
k = torch.randn(B, S, Hk, D, device="cuda").bfloat16()
v = torch.randn_like(k)
for _ in range(2):
    out, lse = ops.flash_attn_fwd(q, k, v, D ** -0.5, -1, 0, 0.0, None, None, None, 0, 0)
    ops.flash_attn_bwd(torch.randn_like(q), q, k, v, out, lse, D ** -0.5, -1, 0, 0.0, None, None, 0, 0, None)
torch.cuda.synchronize()

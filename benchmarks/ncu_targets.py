"""A handful of flagship-shaped launches of the hot kernels, for `ncu --set full` (one GPU, short).

    ncu --set full --clock-control none --import-source on -k regex:gemm_kernel -c 8 -o gpurun_out/prof_gemm \
        python benchmarks/ncu_targets.py
"""

from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from d9d_b200.kernel._native import native_ops
from d9d_b200.kernel.moe import build_moe_layout


def main() -> None:
    ops = native_ops()
    dev = "cuda"
    torch.manual_seed(0)
    T, H, F, E, k = 16384, 768, 576, 128, 8
    bf = dict(device=dev, dtype=torch.bfloat16)
    # 1) dense forward (q_proj): [T,768] x [2048,768]^T
    x = torch.randn(T, H, **bf)
    wq = torch.randn(2048, H, **bf)
    y = torch.empty(T, 2048, **bf)
    ops.gemm(x, wq, y, False, False, False)
    # 2) dense dgrad: dy[T,2048] @ W[2048,768]
    dx = torch.empty(T, H, **bf)
    ops.gemm(y, wq, dx, False, True, False)
    # 3) dense wgrad with fp32 reduce-add epilogue + split-K: dW[2048,768] += dy^T x
    gw = torch.zeros(2048, H, device=dev, dtype=torch.float32)
    ops.gemm(y, x, gw, True, True, True)
    # 4-6) grouped expert GEMMs over a routed layout
    ids = torch.stack([torch.randperm(E, device=dev)[:k] for _ in range(T)])
    layout = build_moe_layout(ids, E)
    xp = torch.randn(layout.capacity, H, **bf)
    w_gate = torch.randn(E, H, F, **bf)
    hid = torch.empty(layout.capacity, F, **bf)
    ops.gemm_grouped_m(xp, w_gate, hid, layout.tile_group, True)  # forward
    dxp = torch.empty(layout.capacity, H, **bf)
    ops.gemm_grouped_m(hid, w_gate, dxp, layout.tile_group, False)  # dgrad
    gwe = torch.zeros(E, H, F, device=dev, dtype=torch.float32)
    ops.gemm_grouped_k(xp, hid, gwe, layout.seg_offsets, True)  # wgrad, reduce-add epilogue
    # 7-8) fused linear cross entropy
    V = 151669
    wv = torch.randn(V, H, **bf) * 0.02
    tgt = torch.randint(0, V, (T,), device=dev)
    nll, lse = ops.ce_forward(x, wv, tgt, -100)
    chunk = 2048
    pitch = (V + 7) // 8 * 8
    dl = torch.empty(chunk, pitch, **bf)[:, :V]
    ops.ce_dlogits(x[:chunk], wv, tgt[:chunk], lse[:chunk], torch.ones(chunk, device=dev), dl, -100)
    # 9) flash-attention forward (own wgmma kernel), flagship shape
    B, S, Hq, Hk, D = 8, 2048, 16, 4, 128
    q = torch.randn(B, S, Hq, D, **bf)
    kk = torch.randn(B, S, Hk, D, **bf)
    vv = torch.randn(B, S, Hk, D, **bf)
    out, lse = ops.flash_attn_fwd(q, kk, vv, D ** -0.5, -1, 0, 0.0, None, None, None, 0, 0)
    ops.flash_attn_bwd(torch.randn_like(q), q, kk, vv, out, lse, D ** -0.5, -1, 0, 0.0, None, None, 0, 0, None)
    # 10) fused q/k RMSNorm + RoPE, 11) router
    wqn = torch.ones(D, **bf)
    ang = torch.rand(B * S, D, device=dev)
    ops.qk_norm_rope_fwd(q.view(B * S, Hq, D), kk.view(B * S, Hk, D), wqn, wqn, ang.cos(), ang.sin(), 1e-6, False, 0)
    ops.router_topk_fwd(torch.randn(T, E, **bf), None, k, True, "softmax", 1, 1, 1.0, 0)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()

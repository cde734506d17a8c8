"""Round-2 kernels for one `ncu --set full` capture (one GPU, a dozen launches):

    ncu --set full --clock-control none --import-source on -k regex:"gemm_kernel|gemm_fp8_kernel|flash_" -c 12 \
        -o gpurun_out/prof_r2 python benchmarks/ncu_targets_r2.py

Order of the profiled launches: CTA-pair GEMM (qkv shape), single-CTA GEMM (same shape), CTA-pair GEMM 16384x4096x4096,
fp8 GEMM, MXFP8 GEMM (same shape), fused linear-CE forward on CTA pairs, flash-attention forward, backward (dK/dV, dQ).
"""

from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch

from d9d_b200.kernel._native import native_ops


def main() -> None:
    ops = native_ops()
    dev = "cuda"
    torch.manual_seed(0)
    bf = dict(device=dev, dtype=torch.bfloat16)
    T, H = 16384, 768
    x = torch.randn(T, H, **bf)
    wq = torch.randn(2048, H, **bf)
    y = torch.empty(T, 2048, **bf)
    ops.gemm(x, wq, y, False, False, False, 2)
    ops.gemm(x, wq, y, False, False, False, 1)
    a = torch.randn(T, 4096, **bf)
    b = torch.randn(4096, 4096, **bf)
    d = torch.empty(T, 4096, **bf)
    ops.gemm(a, b, d, False, False, False, 2)
    aq, sa = ops.quantize_rowwise(a)
    bq, sb = ops.quantize_rowwise(b)
    ops.gemm_fp8(aq, bq, sa, sb, 1.0, d)
    am, sfa = ops.quantize_mx(a)
    bm, sfb = ops.quantize_mx(b)
    ops.gemm_mxfp8(am, sfa, bm, sfb, d)
    V = 151669
    wv = torch.randn(V, H, **bf) * 0.02
    tgt = torch.randint(0, V, (T,), device=dev)
    prev = ops.gemm_set_pair_mode(1)
    ops.ce_forward(x, wv, tgt, -100)
    ops.gemm_set_pair_mode(prev)
    B, S, Hq, Hk, D = 8, 2048, 16, 4, 128
    q = torch.randn(B, S, Hq, D, **bf)
    kk = torch.randn(B, S, Hk, D, **bf)
    vv = torch.randn(B, S, Hk, D, **bf)
    out, lse = ops.flash_attn_fwd(q, kk, vv, D ** -0.5, -1, 0, 0.0, None, None, None, 0, 0)
    ops.flash_attn_bwd(torch.randn_like(q), q, kk, vv, out, lse, D ** -0.5, -1, 0, 0.0, None, None, 0, 0, None)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()

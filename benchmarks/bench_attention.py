"""Native wgmma flash attention (forward, both P variants, and backward) vs PyTorch SDPA on cuDNN, flagship shapes.

Device-timed with CUDA events, 256 MB L2 flush between iterations, median of 20 after 3 warm-ups.
FLOPs: forward 4*B*H*Sq*Sk*D (x0.5 causal); backward 2.5x forward (the usual convention: 5 GEMMs vs 2)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from torch.nn.attention import SDPBackend, sdpa_kernel

from d9d_b200.kernel._native import native_ops

ops = native_ops()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return sorted(ts)[len(ts) // 2]


res = []
shapes = [(8, 2048, 16, 4, 128, True), (8, 2048, 16, 4, 128, False), (2, 8192, 32, 8, 128, True), (8, 2048, 16, 4, 64, True),
          (1, 16384, 16, 4, 128, True)]
for (B, S, Hq, Hk, D, causal) in shapes:
    q = torch.randn(B, S, Hq, D, device="cuda").bfloat16()
    k = torch.randn(B, S, Hk, D, device="cuda").bfloat16()
    v = torch.randn_like(k)
    do = torch.randn_like(q)
    flops = 4.0 * B * Hq * S * S * D * (0.5 if causal else 1.0)
    wr = 0 if causal else -1
    row = {"B": B, "S": S, "Hq": Hq, "Hk": Hk, "D": D, "causal": causal}
    for variant, name in ((0, "native_fwd"),):
        try:
            t = timeit(lambda: ops.flash_attn_fwd(q, k, v, D ** -0.5, -1, wr, 0.0, None, None, None, 0, 0, variant))
            row[name + "_ms"], row[name + "_tflops"] = t, flops / t / 1e9
        except Exception as exc:  # noqa: BLE001
            row[name + "_error"] = str(exc)[:200]
    out, lse = ops.flash_attn_fwd(q, k, v, D ** -0.5, -1, wr, 0.0, None, None, None, 0, 0, 0)
    t = timeit(lambda: ops.flash_attn_bwd(do, q, k, v, out, lse, D ** -0.5, -1, wr, 0.0, None, None, 0, 0, None))
    row["native_bwd_ms"], row["native_bwd_tflops"] = t, 2.5 * flops / t / 1e9
    qh, kh, vh = (x.transpose(1, 2).detach().requires_grad_() for x in (q, k, v))
    with sdpa_kernel(SDPBackend.CUDNN_ATTENTION):
        with torch.no_grad():
            t = timeit(lambda: F.scaled_dot_product_attention(qh, kh, vh, is_causal=causal, enable_gqa=True))
        row["cudnn_fwd_ms"], row["cudnn_fwd_tflops"] = t, flops / t / 1e9
        o = F.scaled_dot_product_attention(qh, kh, vh, is_causal=causal, enable_gqa=True)
        doh = do.transpose(1, 2)
        t = timeit(lambda: torch.autograd.grad(o, (qh, kh, vh), doh, retain_graph=True))
        row["cudnn_bwd_ms"], row["cudnn_bwd_tflops"] = t, 2.5 * flops / t / 1e9
    res.append(row)
    print(row, flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(res, open("gpurun_out/bench_attention.json", "w"), indent=1)

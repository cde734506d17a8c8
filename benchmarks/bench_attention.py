"""Native wgmma flash attention (forward and backward) vs PyTorch SDPA on cuDNN, flagship shapes; then
multi-head latent attention rows (qk head dim 192, v head dim 128): native, the SDPA path on V zero-padded to 192 (default
backend selection, what non-native callers get) and cuDNN on the padded tensors.

Device-timed with CUDA events, 256 MB L2 flush between iterations, median of 20 after 3 warm-ups.
FLOPs: forward 4*B*H*Sq*Sk*D (x0.5 causal); backward 2.5x forward (the usual convention: 5 GEMMs vs 2).  At unequal head
dims the GEMMs over Dqk (S, dK, dQ) and over Dv (PV, dP, dV) are counted separately: forward 2*B*H*S^2*(Dqk + Dv),
backward 2*B*H*S^2*(3 Dqk + 2 Dv) (x0.5 causal), padding not counted."""
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
    t = timeit(lambda: ops.flash_attn_fwd(q, k, v, D ** -0.5, -1, wr, 0.0, None, None, None, 0, 0))
    row["native_fwd_ms"], row["native_fwd_tflops"] = t, flops / t / 1e9
    out, lse = ops.flash_attn_fwd(q, k, v, D ** -0.5, -1, wr, 0.0, None, None, None, 0, 0)
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
mla_shapes = [(4, 4096, 16, True), (1, 16384, 16, True)]
DQK, DV = 192, 128
for (B, S, H, causal) in mla_shapes:
    q = torch.randn(B, S, H, DQK, device="cuda").bfloat16()
    k = torch.randn(B, S, H, DQK, device="cuda").bfloat16()
    v = torch.randn(B, S, H, DV, device="cuda").bfloat16()
    do = torch.randn(B, S, H, DV, device="cuda").bfloat16()
    c = 0.5 if causal else 1.0
    fwd_flops = 2.0 * B * H * S * S * (DQK + DV) * c
    bwd_flops = 2.0 * B * H * S * S * (3 * DQK + 2 * DV) * c
    sc = DQK ** -0.5
    wr = 0 if causal else -1
    row = {"B": B, "S": S, "Hq": H, "Hk": H, "Dqk": DQK, "Dv": DV, "causal": causal}

    def put(name, t, flops):
        row[name + "_ms"], row[name + "_tflops"] = t, flops / t / 1e9

    put("native_fwd", timeit(lambda: ops.flash_attn_fwd(q, k, v, sc, -1, wr, 0.0, None, None, None, 0, 0)), fwd_flops)
    out, lse = ops.flash_attn_fwd(q, k, v, sc, -1, wr, 0.0, None, None, None, 0, 0)
    put("native_bwd", timeit(lambda: ops.flash_attn_bwd(do, q, k, v, out, lse, sc, -1, wr, 0.0, None, None, 0, 0, None)), bwd_flops)
    qh, kh, vh = (x.transpose(1, 2).detach().requires_grad_() for x in (q, k, v))
    doh = do.transpose(1, 2)

    def padded_sdpa(vv):
        o = F.scaled_dot_product_attention(qh, kh, F.pad(vv, (0, DQK - DV)), is_causal=causal, scale=sc)
        return o[..., :DV]

    # the SDPA path as non-native callers get it: pad V, default backend selection, slice the output
    with torch.no_grad():
        put("sdpa_padded_fwd", timeit(lambda: padded_sdpa(vh)), fwd_flops)
    o = padded_sdpa(vh)
    put("sdpa_padded_bwd", timeit(lambda: torch.autograd.grad(o, (qh, kh, vh), doh, retain_graph=True)), bwd_flops)
    # cuDNN on tensors padded beforehand (the padding itself untimed)
    vp = F.pad(vh.detach(), (0, DQK - DV)).requires_grad_()
    dop = F.pad(doh, (0, DQK - DV))
    try:
        with sdpa_kernel(SDPBackend.CUDNN_ATTENTION):
            with torch.no_grad():
                put("cudnn_padded_fwd", timeit(lambda: F.scaled_dot_product_attention(qh, kh, vp, is_causal=causal, scale=sc)), fwd_flops)
            o = F.scaled_dot_product_attention(qh, kh, vp, is_causal=causal, scale=sc)
            put("cudnn_padded_bwd", timeit(lambda: torch.autograd.grad(o, (qh, kh, vp), dop, retain_graph=True)), bwd_flops)
    except Exception as exc:  # noqa: BLE001
        row["cudnn_padded_error"] = str(exc)[:200]
    res.append(row)
    print(row, flush=True)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(res, open("gpurun_out/bench_attention.json", "w"), indent=1)

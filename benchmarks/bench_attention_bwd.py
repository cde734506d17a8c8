"""Per-kernel device time of the native flash attention backward (delta pre-pass, dK/dV kernel, dQ kernel) under
torch.profiler, with each kernel's rate on the FLOPs its GEMMs execute.

Shapes: the flagship (8 x 2048, 16 / 4 heads x 128, causal), the same at head dim 64, and multi-head latent attention
(4 x 4096, 16 heads, qk 192 / v 128, causal).  A GEMM over head dim d counts 2 d FLOPs per (query, key) pair of every
query head, S^2 / 2 pairs per head under a causal mask (what the masked diagonal tiles also compute is not counted).
The dK/dV kernel runs 4 GEMMs per tile (S^T and dK over the qk head dim, dP^T and dV over the v head dim), the dQ
kernel 3 (S and dQ over qk, dP over v).  Each kernel's time is its mean over ``--iters`` backward calls after ``--warmup``.

    python benchmarks/bench_attention_bwd.py [--iters 20] [--warmup 3] [--out FILE.json]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

from d9d_b200 import ops as _ops

SHAPES = [  # B, S, Hq, Hk, Dqk, Dv, causal
    (8, 2048, 16, 4, 128, 128, True),
    (8, 2048, 16, 4, 64, 64, True),
    (4, 4096, 16, 16, 192, 128, True),
]


def kernel_times(fn, iters, warmup):
    """Mean device time (ms) per call of each kernel fn launches, keyed by dkv / dq / delta."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        if "flash_attn_bwd_kernel" in name:
            key = "dkv" if "true>" in name else "dq"
        elif "flash_attn_delta_kernel" in name:
            key = "delta"
        else:
            continue
        out[key] = out.get(key, 0.0) + ev.device_time_total / 1e3 / iters
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()
    ops = _ops.load()
    rows = []
    for B, S, Hq, Hk, Dqk, Dv, causal in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        q = torch.randn(B, S, Hq, Dqk, device="cuda", generator=g).bfloat16()
        k = torch.randn(B, S, Hk, Dqk, device="cuda", generator=g).bfloat16()
        v = torch.randn(B, S, Hk, Dv, device="cuda", generator=g).bfloat16()
        do = torch.randn(B, S, Hq, Dv, device="cuda", generator=g).bfloat16()
        sc, wr = Dqk**-0.5, (0 if causal else -1)
        out, lse = ops.flash_attn_fwd(q, k, v, sc, -1, wr, 0.0, None, None, None, 0, 0)
        t = kernel_times(lambda: ops.flash_attn_bwd(do, q, k, v, out, lse, sc, -1, wr, 0.0, None, None, 0, 0, None),
                         args.iters, args.warmup)
        pairs = B * Hq * S * S * (0.5 if causal else 1.0)  # (query, key) pairs of one head, summed
        flops = {"dkv": 2 * pairs * (2 * Dqk + 2 * Dv), "dq": 2 * pairs * (2 * Dqk + Dv)}
        row = {"B": B, "S": S, "Hq": Hq, "Hk": Hk, "Dqk": Dqk, "Dv": Dv, "causal": causal}
        for key in ("delta", "dkv", "dq"):
            row[f"{key}_ms"] = round(t.get(key, float("nan")), 4)
            if key in flops:
                row[f"{key}_tflops"] = round(flops[key] / t[key] / 1e9, 1)
        row["bwd_ms"] = round(sum(t.values()), 4)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()

"""The MoE expert block (``grouped_swiglu``) in bf16 against fp8 under the row-wise recipe (e4m3 grouped GEMMs with per-expert
scales; the ``fp8`` keys) and under DeepSeek-V3's blockwise recipe (1x128 / 128x128 scales promoted per k-block; the
``blockwise`` keys), forward and forward + backward, at the flagship shape (T = 16 384 tokens, k = 8, E = 128, hidden 768, expert FFN 576) and at the
Qwen3-30B-A3B expert shape of ``bench.py`` (hidden 2048, expert FFN 768, same T / k / E).

Timing: CUDA events around ``--iters`` calls; the three arms alternate window by window (``--repeats`` windows
each) so that drifting clocks hit both alike; the median window is reported.  A separate ``torch.profiler`` run then splits
one forward + backward of each arm into GEMMs, quantisers and the rest, with achieved TFLOP/s of the GEMMs (FLOPs
counted from the routed tokens: 2 x tokens x in x out per GEMM, no padding).

Usage: python benchmarks/bench_fp8_experts.py [--out results/bench_fp8_experts.json]
"""

from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.bench_gemm_flagship import card  # noqa: E402
from d9d_b200.kernel.moe import build_moe_layout, grouped_swiglu, moe_permute  # noqa: E402

SHAPES = [("flagship", 16384, 8, 128, 768, 576), ("30b_a3b_experts", 16384, 8, 128, 2048, 768)]


def setup(T, k, E, H, F):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(T, H, device="cuda", generator=g).bfloat16()
    ids = torch.rand(T, E, device="cuda", generator=g).topk(k, dim=1).indices
    probs = torch.rand(T, k, device="cuda", generator=g)
    layout = build_moe_layout(ids, E)
    xp, pp = moe_permute(x, probs, layout)
    w = [(torch.randn(E, a, b, device="cuda", generator=g) * 0.02).bfloat16().requires_grad_() for a, b in ((H, F), (H, F), (F, H))]
    xp = xp.detach().requires_grad_()
    dy = torch.randn(xp.shape[0], H, device="cuda", generator=g).bfloat16()
    return xp, pp.detach(), w, layout, dy


# arm -> grouped_swiglu arguments; the keys name the arms in the JSON
ARMS = {"bf16": {}, "fp8": {"fp8": True}, "blockwise": {"fp8": True, "recipe": "blockwise"}}


def step(inputs, arm, backward):
    xp, pp, w, layout, dy = inputs
    if not backward:
        with torch.no_grad():
            grouped_swiglu(xp, pp, *w, layout, **ARMS[arm])
        return
    y = grouped_swiglu(xp, pp, *w, layout, **ARMS[arm])
    y.backward(dy)
    xp.grad = None
    for t in w:
        t.grad = None


def window_ms(inputs, arm, backward, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        step(inputs, arm, backward)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def classify(name: str) -> str:
    if "gemm_fp8_kernel" in name or "gemm_kernel" in name:
        return "gemm"
    if "quant" in name or "col_amax" in name:
        return "quantise"
    return "other"


def profile(inputs, arm, routed, H, F):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile

    step(inputs, arm, True)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        step(inputs, arm, True)
        torch.cuda.synchronize()
    us = {"gemm": 0.0, "quantise": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        us[classify(ev.key)] += t
    flops = 9 * 2 * routed * H * F  # forward 3 GEMMs, backward 6
    return {"gemm_ms": us["gemm"] / 1e3, "quantise_ms": us["quantise"] / 1e3, "other_ms": us["other"] / 1e3,
            "gemm_tflops": flops / (us["gemm"] * 1e-6) / 1e12 if us["gemm"] else None}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_experts needs a GPU")
    result = {"card": card(), "shapes": []}
    print(json.dumps(result["card"]))
    for name, T, k, E, H, F in SHAPES:
        inputs = setup(T, k, E, H, F)
        row = {"name": name, "T": T, "k": k, "E": E, "hidden": H, "ffn": F}
        for backward in (False, True):
            for arm in ARMS:
                window_ms(inputs, arm, backward, 2)  # warm-up
            times = {arm: [] for arm in ARMS}
            for _ in range(args.repeats):
                for arm in ARMS:
                    times[arm].append(window_ms(inputs, arm, backward, args.iters))
            tag = "fwd_bwd" if backward else "fwd"
            for arm in ARMS:
                row[f"{tag}_{arm}_ms"] = statistics.median(times[arm])
            for arm in ARMS:
                row[f"{tag}_{arm}_spread_ms"] = max(times[arm]) - min(times[arm])
        for arm in ARMS:
            row[f"profile_{arm}"] = profile(inputs, arm, T * k, H, F)
        print(json.dumps(row))
        result["shapes"].append(row)
        del inputs
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

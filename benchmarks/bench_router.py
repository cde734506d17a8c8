"""The fused router kernel (``route_topk``) against the PyTorch definition (``route_topk_general``), forward and
forward+backward, on the DeepSeek-V3 routing (sigmoid scores, 8 groups of which 4 stay eligible, bias, renormalised,
scale 2.5, E = 256, k = 8) and on the flagship softmax router (Qwen3-MoE: E = 128, k = 8), whose kernel path the
DeepSeek options leave unchanged.  An auxiliary-loss arm times the fused kernel with the load-balancing and router z
losses off and on, at the flagship shape and at a group-limited softmax shape (DeepSeek-V2 style: E = 160, 8 groups of
which 3 stay eligible, k = 6).  A sequence-balance arm times the fused kernel with the sequence-wise balance loss off and
on at the DeepSeek-V3 routing, T = 16 384 tokens in sequences of S = 4 096 (DeepSeek-V3's pre-training length).

Timing: CUDA events around ``--iters`` back-to-back calls after ``--warmup`` calls; median of ``--repeats`` windows.
Usage: python benchmarks/bench_router.py [--out results/bench_router.json]
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.bench_gemm_flagship import card  # noqa: E402
from d9d_b200.kernel.router import route_topk, route_topk_general  # noqa: E402

SHAPES = [  # name, T, E, k, options
    ("deepseek_v3", 4096, 256, 8, {"score_function": "sigmoid", "num_groups": 8, "topk_groups": 4, "scaling_factor": 2.5}),
    ("deepseek_v3", 16384, 256, 8, {"score_function": "sigmoid", "num_groups": 8, "topk_groups": 4, "scaling_factor": 2.5}),
    ("flagship_softmax", 16384, 128, 8, {}),
]
AUX_SHAPES = [  # name, T, E, k, options; renormalised
    ("flagship_softmax", 16384, 128, 8, {}),
    ("grouped_softmax", 16384, 160, 6, {"num_groups": 8, "topk_groups": 3}),
]
AUX_ON = {"load_balancing_coef": 1e-2, "z_loss_coef": 1e-3, "token_loss_weight": 1e-3}
SEQ_SHAPES = [  # name, T, E, k, sequence length, options; biased, renormalised
    ("deepseek_v3", 16384, 256, 8, 4096, {"score_function": "sigmoid", "num_groups": 8, "topk_groups": 4, "scaling_factor": 2.5}),
]
SEQ_ON = {"sequence_balance_coef": 1e-4, "token_loss_weight": 1e-3}  # DeepSeek-V3's alpha


def _time_ms(fn, iters: int, warmup: int, repeats: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    windows = []
    for _ in range(repeats):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(iters):
            fn()
        end.record()
        torch.cuda.synchronize()
        windows.append(start.elapsed_time(end) / iters)
    return sorted(windows)[len(windows) // 2]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_router needs a CUDA device")

    results = {"card": card(), "shapes": []}
    print(json.dumps(results["card"]), flush=True)
    for name, T, E, k, opts in SHAPES:
        torch.manual_seed(0)
        logits = torch.randn(T, E, device="cuda").bfloat16()
        bias = (torch.randn(E, device="cuda") * 0.01) if opts else None
        dprobs = torch.randn(T, k, device="cuda")
        row = {"name": name, "T": T, "E": E, "k": k, **opts}
        for impl, fn in (("native", route_topk), ("general", route_topk_general)):
            x = logits.clone().requires_grad_()

            def fwd(fn=fn, x=x):
                with torch.no_grad():
                    fn(x, k, True, bias, **opts)

            def fwd_bwd(fn=fn, x=x):
                _, probs = fn(x, k, True, bias, **opts)
                x.grad = None
                probs.backward(dprobs)

            row[f"{impl}_fwd_us"] = round(1e3 * _time_ms(fwd, args.iters, args.warmup, args.repeats), 2)
            row[f"{impl}_fwd_bwd_us"] = round(1e3 * _time_ms(fwd_bwd, args.iters, args.warmup, args.repeats), 2)
        row["speedup_fwd"] = round(row["general_fwd_us"] / row["native_fwd_us"], 2)
        row["speedup_fwd_bwd"] = round(row["general_fwd_bwd_us"] / row["native_fwd_bwd_us"], 2)
        results["shapes"].append(row)
        print(json.dumps(row), flush=True)
    results["aux_shapes"] = []
    for name, T, E, k, opts in AUX_SHAPES:
        torch.manual_seed(0)
        x = torch.randn(T, E, device="cuda").bfloat16().requires_grad_()
        dprobs = torch.randn(T, k, device="cuda")
        sums = torch.zeros(3, device="cuda")
        row = {"name": name, "T": T, "E": E, "k": k, **opts}
        for arm, aux in (("off", {}), ("on", {**AUX_ON, "aux_loss_sums": sums})):

            def fwd(aux=aux):
                with torch.no_grad():
                    route_topk(x, k, True, **opts, **aux)

            def fwd_bwd(aux=aux):
                _, probs = route_topk(x, k, True, **opts, **aux)
                x.grad = None
                probs.backward(dprobs)

            row[f"aux_{arm}_fwd_us"] = round(1e3 * _time_ms(fwd, args.iters, args.warmup, args.repeats), 2)
            row[f"aux_{arm}_fwd_bwd_us"] = round(1e3 * _time_ms(fwd_bwd, args.iters, args.warmup, args.repeats), 2)
        results["aux_shapes"].append(row)
        print(json.dumps(row), flush=True)
    results["seq_shapes"] = []
    for name, T, E, k, S, opts in SEQ_SHAPES:
        torch.manual_seed(0)
        x = torch.randn(T, E, device="cuda").bfloat16().requires_grad_()
        bias = torch.randn(E, device="cuda") * 0.01
        dprobs = torch.randn(T, k, device="cuda")
        sums = torch.zeros(2, device="cuda")
        row = {"name": name, "T": T, "E": E, "k": k, "S": S, **opts}
        for arm, seq in (("off", {}), ("on", {**SEQ_ON, "sequence_length": S, "sequence_balance_sums": sums})):

            def fwd(seq=seq):
                with torch.no_grad():
                    route_topk(x, k, True, bias, **opts, **seq)

            def fwd_bwd(seq=seq):
                _, probs = route_topk(x, k, True, bias, **opts, **seq)
                x.grad = None
                probs.backward(dprobs)

            row[f"seq_{arm}_fwd_us"] = round(1e3 * _time_ms(fwd, args.iters, args.warmup, args.repeats), 2)
            row[f"seq_{arm}_fwd_bwd_us"] = round(1e3 * _time_ms(fwd_bwd, args.iters, args.warmup, args.repeats), 2)
        results["seq_shapes"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

"""Cost of label smoothing and the z-loss in the fused linear cross-entropy at the flagship LM head (T = 16 384 tokens,
hidden 768, V = 151 669 classes in one block): forward and forward + backward of ``linear_cross_entropy`` with
``reduction="mean"``, plain against ``label_smoothing=0.1``, ``z_loss_coef=1e-4`` and both.

Timing: CUDA events around ``--iters`` back-to-back calls; the variants are warmed up, then timed in alternation,
``--repeats`` windows each, and the median window is reported.  The card's name and power limit are recorded with the
numbers.
Usage: python benchmarks/bench_cce_regularised.py [--out results/bench_cce_regularised.json]
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.bench_gemm_flagship import card  # noqa: E402
from d9d_b200.kernel.cce import linear_cross_entropy  # noqa: E402

T, H, V = 16384, 768, 151669
VARIANTS = {"plain": {}, "label_smoothing": {"label_smoothing": 0.1}, "z_loss": {"z_loss_coef": 1e-4},
            "both": {"label_smoothing": 0.1, "z_loss_coef": 1e-4}}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cce_regularised needs a GPU")
    torch.manual_seed(0)
    e = (torch.randn(T, H, device="cuda") * 0.5).bfloat16().requires_grad_()
    w = (torch.randn(V, H, device="cuda") * 0.05).bfloat16().requires_grad_()
    tgt = torch.randint(0, V, (T,), device="cuda")
    tgt[::17] = -100

    def forward(kw):
        with torch.no_grad():
            linear_cross_entropy(e, w, tgt, **kw)

    def forward_backward(kw):
        e.grad = w.grad = None
        linear_cross_entropy(e, w, tgt, **kw).backward()

    results = {"card": card(), "shape": {"T": T, "H": H, "V": V}, "iters": args.iters, "repeats": args.repeats,
               "forward_ms": {}, "forward_backward_ms": {}}
    for key, fn in (("forward_ms", forward), ("forward_backward_ms", forward_backward)):
        for kw in VARIANTS.values():
            for _ in range(args.warmup):
                fn(kw)
        torch.cuda.synchronize()
        windows: dict[str, list[float]] = {name: [] for name in VARIANTS}
        for _ in range(args.repeats):
            for name, kw in VARIANTS.items():  # alternated: drifting clocks and neighbours hit every variant alike
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(args.iters):
                    fn(kw)
                end.record()
                torch.cuda.synchronize()
                windows[name].append(start.elapsed_time(end) / args.iters)
        for name, ws in windows.items():
            results[key][name] = {"median": sorted(ws)[len(ws) // 2], "min": min(ws), "max": max(ws)}
    print(json.dumps(results, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

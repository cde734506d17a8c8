"""Dense linear layers in bf16 (the native wgmma GEMM) against the three fp8 recipes of ``fp8_linear``: ``rowwise``,
``mx`` (where every size is a multiple of 128) and ``blockwise`` (DeepSeek-V3's 1x128 / 128x128 scaling with promoted
accumulation), forward and forward + backward.

Shapes: DeepSeek-V3's dense layers at T = 8 192 tokens (hidden 7168 <-> FFN 18 432, q_up 1536 -> 24 576, kv_down
7168 -> 576, o_proj 16 384 -> 7168) and the flagship's attention projections at T = 16 384 (q 768 -> 2048, k / v
768 -> 512, o 2048 -> 768).

Timing: CUDA events around ``--iters`` calls; the arms alternate window by window (``--repeats`` windows each) so that
drifting clocks hit them alike; the median window is reported.  A separate ``torch.profiler`` run then splits one forward
+ backward of each arm into GEMMs, quantisers and the rest, with the GEMMs' achieved TFLOP/s (6 x T x in x out).

Accuracy, on the same seeded inputs: norm-wise relative error of y, dx and dW against fp64 of the bf16 inputs, without
and with an outlier (three elements of one token's first 128-group at 2^16 times the inputs' scale).  With the outlier
the whole-tensor errors are dominated by the outlier's own products, so the errors of the outlier's row of y and the
outlier channel's column of dW are reported too.

Usage: python benchmarks/bench_fp8_blockwise.py [--out benchmarks/results/bench_fp8_blockwise.json]
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
from d9d_b200.kernel.fp8 import fp8_linear  # noqa: E402
from d9d_b200.kernel.gemm import linear  # noqa: E402

SHAPES = [  # name, tokens, in, out
    ("dsv3_mlp_up", 8192, 7168, 18432),
    ("dsv3_mlp_down", 8192, 18432, 7168),
    ("dsv3_q_up", 8192, 1536, 24576),
    ("dsv3_kv_down", 8192, 7168, 576),
    ("dsv3_o_proj", 8192, 16384, 7168),
    ("flagship_q", 16384, 768, 2048),
    ("flagship_kv", 16384, 768, 512),
    ("flagship_o", 16384, 2048, 768),
]
OUTLIER_ROW, OUTLIER_COLS = 17, slice(5, 8)


def arms_for(T, fin, fout):
    arms = ["bf16", "rowwise"]
    if T % 128 == 0 and fin % 128 == 0 and fout % 128 == 0:
        arms.append("mx")
    return arms + ["blockwise"]


def run(arm, x, w):
    return linear(x, w) if arm == "bf16" else fp8_linear(x, w, recipe=arm)


def setup(T, fin, fout, outlier=False):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(T, fin, device="cuda", generator=g)
    if outlier:
        x[OUTLIER_ROW, OUTLIER_COLS] = 2.0**16
    w = torch.randn(fout, fin, device="cuda", generator=g) * fin**-0.5
    dy = torch.randn(T, fout, device="cuda", generator=g)
    return x.bfloat16().requires_grad_(), w.bfloat16().requires_grad_(), dy.bfloat16()


def step(arm, inputs, backward):
    x, w, dy = inputs
    if not backward:
        with torch.no_grad():
            run(arm, x, w)
        return
    run(arm, x, w).backward(dy)
    x.grad = None
    w.grad = None


def window_ms(arm, inputs, backward, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        step(arm, inputs, backward)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def classify(name: str) -> str:
    if "gemm_fp8_kernel" in name or "gemm_kernel" in name:
        return "gemm"
    if "quant" in name or "col_amax" in name:
        return "quantise"
    return "other"


def profile(arm, inputs, flops):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile

    step(arm, inputs, True)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        step(arm, inputs, True)
        torch.cuda.synchronize()
    us = {"gemm": 0.0, "quantise": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        us[classify(ev.key)] += t
    return {"gemm_ms": us["gemm"] / 1e3, "quantise_ms": us["quantise"] / 1e3, "other_ms": us["other"] / 1e3,
            "gemm_tflops": flops / (us["gemm"] * 1e-6) / 1e12 if us["gemm"] else None}


def _rel(a, b):
    return float((a.double() - b).norm() / b.norm())


def accuracy(arms, T, fin, fout):
    out = {}
    for outlier in (False, True):
        x, w, dy = setup(T, fin, fout, outlier)
        xd, wd = x.detach().double().requires_grad_(), w.detach().double().requires_grad_()
        yd = xd @ wd.t()
        yd.backward(dy.double())
        for arm in arms:
            y = run(arm, x, w)
            y.backward(dy)
            tag = f"{arm}{'_outlier' if outlier else ''}"
            out[tag] = {"y": _rel(y, yd), "dx": _rel(x.grad, xd.grad), "dw": _rel(w.grad, wd.grad)}
            if outlier:
                c = OUTLIER_COLS.start
                out[tag]["y_outlier_row"] = _rel(y[OUTLIER_ROW], yd[OUTLIER_ROW])
                out[tag]["dw_outlier_col"] = _rel(w.grad[:, c], wd.grad[:, c])
            x.grad = None
            w.grad = None
            del y
        del xd, wd, yd
        torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--shapes", default=None, help="comma-separated subset of the shape names")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_blockwise needs a GPU")
    result = {"card": card(), "shapes": []}
    print(json.dumps(result["card"]), flush=True)
    wanted = set(args.shapes.split(",")) if args.shapes else None
    for name, T, fin, fout in SHAPES:
        if wanted is not None and name not in wanted:
            continue
        arms = arms_for(T, fin, fout)
        inputs = setup(T, fin, fout)
        row = {"name": name, "T": T, "in": fin, "out": fout, "arms": arms}
        for backward in (False, True):
            for arm in arms:
                window_ms(arm, inputs, backward, 2)  # warm-up
            times = {arm: [] for arm in arms}
            for _ in range(args.repeats):
                for arm in arms:
                    times[arm].append(window_ms(arm, inputs, backward, args.iters))
            tag = "fwd_bwd" if backward else "fwd"
            for arm in arms:
                row[f"{tag}_{arm}_ms"] = statistics.median(times[arm])
                row[f"{tag}_{arm}_spread_ms"] = max(times[arm]) - min(times[arm])
        for arm in arms:
            row[f"profile_{arm}"] = profile(arm, inputs, 6.0 * T * fin * fout)
        del inputs
        torch.cuda.empty_cache()
        row["accuracy"] = accuracy(arms, T, fin, fout)
        print(json.dumps(row), flush=True)
        result["shapes"].append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

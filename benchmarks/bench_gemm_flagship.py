"""Kernel-level timing of the bf16 GEMM calls one flagship microbatch makes (Qwen3-MoE example model, 8 x 2048 tokens).

    python benchmarks/bench_gemm_flagship.py [--out results/bench_gemm_flagship.json]

Calls, at the flagship's shapes (T = 16,384 tokens, hidden 768, vocabulary 151,643 + 26):
* fused linear-cross-entropy: the forward over the regular vocabulary block, and for one backward column chunk of the
  width ``plan_vocab_chunks`` picks: the dlogits recompute, dE += dL C and dC += dL^T E;
* experts (128 experts, top-8, the 128-row aligned layout of uniformly routed tokens, ffn 576): the gate / up / down
  forward GEMMs (``gemm_grouped_m``), the down-proj and gate / up dgrads, and the weight gradients (``gemm_grouped_k``);
* attention projections: q (768 -> 2048), k / v (768 -> 512) and o (2048 -> 768), forward, dgrad and wgrad.

Every call is warmed up, then timed with CUDA events around single launches with an L2 flush in between; the median of
``--iters`` is reported with TFLOP/s computed from the shapes (expert GEMMs count the T x top-k routed rows, not the
padding of the aligned layout).  Weight gradients accumulate into fp32, as into the fused-wgrad buffers of the model.
The card's name, power limit and SM clock limit are read in the same run.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.bench_ops import timeit  # noqa: E402
from d9d_b200 import ops as _ops  # noqa: E402

T, HIDDEN, FFN, EXPERTS, TOP_K = 16384, 768, 576, 128, 8
VOCAB = (151643, 26)
Q_OUT, KV_OUT = 16 * 128, 4 * 128


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"], info["sm_clock_idle"] = (s.strip() for s in q.split(","))
    except Exception as exc:  # noqa: BLE001
        info["nvidia_smi_error"] = repr(exc)[:200]
    return info


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the results as JSON to this file")
    ap.add_argument("--iters", type=int, default=21)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gemm_flagship needs a GPU"
    ops = _ops.load()
    from d9d_b200.kernel.cce.main import IGNORE_INDEX, _CHUNK_BYTES, plan_vocab_chunks
    from d9d_b200.kernel.moe.layout import build_moe_layout

    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)

    def randn(*shape, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=gen) * scale).to(torch.bfloat16)

    rows = []

    def run(name, fn, flops):
        ms = timeit(fn, iters=args.iters)
        rows.append({"call": name, "ms": ms, "tflops": flops / ms / 1e9})
        print(f"{name:<34} {ms:8.3f} ms  {flops / ms / 1e9:7.1f} TFLOP/s", flush=True)

    # ---- fused linear-cross-entropy ----
    e = randn(T, HIDDEN)
    w = randn(VOCAB[0], HIDDEN, scale=0.05)
    targets = torch.randint(0, sum(VOCAB), (T,), device=dev, generator=gen)
    run("ce_forward (V = 151,643)", lambda: ops.ce_forward_ex(e, w, targets, IGNORE_INDEX, None, 0.0, 0),
        2.0 * T * VOCAB[0] * HIDDEN)
    _, lse, _ = ops.ce_forward_ex(e, w, targets, IGNORE_INDEX, None, 0.0, 0)
    chunks, width, _ = plan_vocab_chunks(list(VOCAB), T, HIDDEN, _CHUNK_BYTES, torch.cuda.get_device_properties(dev).multi_processor_count)
    wc = w[:width]
    g = torch.full((T,), 1.0 / T, device=dev)
    dl = torch.empty(T, width, device=dev, dtype=torch.bfloat16)
    de = torch.zeros(T, HIDDEN, device=dev, dtype=torch.float32)
    dc = torch.zeros(width, HIDDEN, device=dev, dtype=torch.float32)
    f_chunk = 2.0 * T * width * HIDDEN
    run(f"ce_dlogits (chunk {width})", lambda: ops.ce_dlogits(e, wc, targets, lse, g, dl, IGNORE_INDEX, None, 0.0, 0), f_chunk)
    run(f"ce_dE += dL C (chunk {width})", lambda: ops.gemm(dl, wc, de, False, True, True), f_chunk)
    run(f"ce_dC += dL^T E (chunk {width})", lambda: ops.gemm(dl, e, dc, True, True, True), f_chunk)
    del w, dl, de, dc

    # ---- experts ----
    scores = torch.rand(T, EXPERTS, device=dev, generator=gen)
    topk = scores.topk(TOP_K, dim=1).indices.to(torch.int64)
    layout = build_moe_layout(topk, EXPERTS)
    cap = layout.capacity
    routed = T * TOP_K
    xp, hp = randn(cap, HIDDEN), randn(cap, FFN)
    dyp, dgp = randn(cap, HIDDEN), randn(cap, FFN)
    wg, wd = randn(EXPERTS, HIDDEN, FFN, scale=0.03), randn(EXPERTS, FFN, HIDDEN, scale=0.03)
    gate = torch.empty(cap, FFN, device=dev, dtype=torch.bfloat16)
    y = torch.empty(cap, HIDDEN, device=dev, dtype=torch.bfloat16)
    dxp = torch.zeros(cap, HIDDEN, device=dev, dtype=torch.bfloat16)
    dwg = torch.zeros(EXPERTS, HIDDEN, FFN, device=dev, dtype=torch.float32)
    dwd = torch.zeros(EXPERTS, FFN, HIDDEN, device=dev, dtype=torch.float32)
    f_exp = 2.0 * routed * HIDDEN * FFN
    tg, seg = layout.tile_group, layout.seg_offsets
    run("expert gate/up fwd (grouped_m)", lambda: ops.gemm_grouped_m(xp, wg, gate, tg, True), f_exp)
    run("expert down fwd (grouped_m)", lambda: ops.gemm_grouped_m(hp, wd, y, tg, True), f_exp)
    run("expert down dgrad (grouped_m)", lambda: ops.gemm_grouped_m(dyp, wd, gate, tg, False), f_exp)
    run("expert gate dgrad (grouped_m)", lambda: ops.gemm_grouped_m(dgp, wg, dxp, tg, False), f_exp)
    run("expert up dgrad += (grouped_m)", lambda: ops.gemm_grouped_m(dgp, wg, dxp, tg, False, True), f_exp)
    run("expert gate/up wgrad (grouped_k)", lambda: ops.gemm_grouped_k(xp, dgp, dwg, seg, True), f_exp)
    run("expert down wgrad (grouped_k)", lambda: ops.gemm_grouped_k(hp, dyp, dwd, seg, True), f_exp)
    del xp, hp, dyp, dgp, gate, y, dxp, dwg, dwd

    # ---- attention projections ----
    for name, n_in, n_out in (("q", HIDDEN, Q_OUT), ("k/v", HIDDEN, KV_OUT), ("o", Q_OUT, HIDDEN)):
        x, wt, dy = randn(T, n_in), randn(n_out, n_in, scale=0.03), randn(T, n_out)
        out = torch.empty(T, n_out, device=dev, dtype=torch.bfloat16)
        dx = torch.empty(T, n_in, device=dev, dtype=torch.bfloat16)
        dw = torch.zeros(n_out, n_in, device=dev, dtype=torch.float32)
        f = 2.0 * T * n_in * n_out
        run(f"{name}_proj fwd", lambda: ops.gemm(x, wt, out, False, False, False), f)
        run(f"{name}_proj dgrad", lambda: ops.gemm(dy, wt, dx, False, True, False), f)
        run(f"{name}_proj wgrad +=", lambda: ops.gemm(dy, x, dw, True, True, True), f)

    result = {"card": card(), "iters": args.iters, "ce_chunk_width": width, "ce_chunks": len(chunks), "calls": rows}
    print(json.dumps(result["card"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()

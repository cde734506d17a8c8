"""Micro-benchmarks of the native kernels vs the measured roofline (MEASURED_PEAKS.json).

Timing: CUDA events on the launching stream, warm-up, L2 flush (write > L2) between timed iterations.
Usage: python benchmarks/bench_ops.py [--out gpurun_out/bench_ops.json]
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from d9d_b200 import ops as _ops  # noqa: E402


def peaks():
    p = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return d["hbm_gbs"], d["bf16_tflops"], "measured"
    return 3350.0, 989.0, "H100 SXM data sheet (HBM3, dense bf16)"


_flush = None


def timeit(fn, iters=10, warmup=3):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        _flush.zero_()  # L2 flush
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    return times[len(times) // 2]


def timeit_rotating(make_call, working_set_bytes, iters=5, min_total_bytes=1 << 30):
    """Throughput timing for short memory-bound kernels: ``n`` argument sets whose combined footprint is far larger than
    the 50 MB L2 are processed back to back between two events (no launch gap in the measurement, every byte comes from
    HBM).  ``make_call(i)`` returns the zero-argument callable for set ``i``.  Returns ms per call."""
    n = max(2, -(-min_total_bytes // max(working_set_bytes, 1)))
    calls = [make_call(i) for i in range(n)]
    for c in calls[: min(n, 3)]:
        c()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for c in calls:
            c()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e) / n)
    times.sort()
    return times[len(times) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/bench_ops.json")
    args = ap.parse_args()
    ops = _ops.load()
    hbm, tf, kind = peaks()
    res = []

    def rec(name, ms, flops=None, bytes_=None, ref_ms=None):
        r = {"name": name, "ms": round(ms, 4)}
        if flops:
            r["tflops"] = round(flops / ms / 1e9, 1)
            r["frac_of_%s_bf16" % kind] = round(flops / ms / 1e9 / tf, 3)
        if bytes_:
            r["gbs"] = round(bytes_ / ms / 1e6, 1)
            r["frac_of_%s_hbm" % kind] = round(bytes_ / ms / 1e6 / hbm, 3)
        if ref_ms:
            r["torch_ms"] = round(ref_ms, 4)
            r["speedup_vs_torch"] = round(ref_ms / ms, 2)
        res.append(r)
        print(json.dumps(r), flush=True)

    # ---------------- GEMM
    for (M, N, K) in [(8192, 8192, 8192), (16384, 2048, 768), (16384, 768, 2048), (16384, 4096, 4096), (65536, 768, 576)]:
        a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
        d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        ms = timeit(lambda: ops.gemm(a, b, d, False, False, False))
        ref = timeit(lambda: torch.matmul(a, b.t()))
        rec(f"gemm_nt_{M}x{N}x{K}", ms, flops=2 * M * N * K, ref_ms=ref)
        bt = b.t().contiguous()
        ms = timeit(lambda: ops.gemm(a, bt, d, False, True, False))
        rec(f"gemm_nn(dgrad)_{M}x{N}x{K}", ms, flops=2 * M * N * K)
        at = a.t().contiguous()
        df = torch.empty(M, N, device="cuda", dtype=torch.float32)
        ms = timeit(lambda: ops.gemm(at, bt, df, True, True, False))
        rec(f"gemm_tn(wgrad,f32)_{M}x{N}x{K}", ms, flops=2 * M * N * K)
        del a, b, d, bt, at, df

    # ---------------- grouped GEMM (MoE example config: E=128, H=768, I=576, 16384 tokens top-8)
    E, H, I, T, k = 128, 768, 576, 16384, 8
    ids = torch.stack([torch.randperm(E, device="cuda")[:k] for _ in range(T)])
    cap = (T * k + E * 127 + 127) // 128 * 128
    counts, seg, row_map, tile_group = ops.moe_build_layout(ids, E, 128, cap)
    x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
    probs = torch.rand(T, k, device="cuda")
    ms = timeit(lambda: ops.moe_build_layout(ids, E, 128, cap))
    rec("moe_build_layout_16k_top8_E128", ms)
    ms = timeit(lambda: ops.moe_permute(x, probs, row_map, counts, seg, cap))
    rec("moe_permute", ms, bytes_=T * H * 2 + T * k * H * 2)
    xp, pp = ops.moe_permute(x, probs, row_map, counts, seg, cap)
    w1 = torch.randn(E, H, I, device="cuda", dtype=torch.bfloat16)
    h = torch.empty(cap, I, device="cuda", dtype=torch.bfloat16)
    ms = timeit(lambda: ops.gemm_grouped_m(xp, w1, h, tile_group, True))
    rec("grouped_m_fwd_gateproj", ms, flops=2 * T * k * H * I)
    dxp = torch.empty_like(xp)
    ms = timeit(lambda: ops.gemm_grouped_m(h, w1, dxp, tile_group, False))
    rec("grouped_m_dgrad", ms, flops=2 * T * k * H * I)
    dw = torch.empty(E, H, I, device="cuda", dtype=torch.float32)
    ms = timeit(lambda: ops.gemm_grouped_k(xp, h, dw, seg, False))
    rec("grouped_k_wgrad", ms, flops=2 * T * k * H * I)
    ms = timeit(lambda: ops.moe_gather(xp, None, row_map, T, k))
    rec("moe_unpermute", ms, bytes_=T * H * 2 + T * k * H * 2)
    g = torch.randn(cap, I, device="cuda", dtype=torch.bfloat16)
    ms = timeit(lambda: ops.silu_mul_probs_fwd(h, g, pp))
    rec("silu_mul_probs_fwd", ms, bytes_=cap * I * 2 * 3)

    # ---------------- fused linear CE
    T2, V, K = 16384, 151669 // 8 * 8, 768
    hdn = (torch.randn(T2, K, device="cuda") * 0.5).bfloat16()
    wv = (torch.randn(V, K, device="cuda") * 0.05).bfloat16()
    tgt = torch.randint(0, V, (T2,), device="cuda")
    ms = timeit(lambda: ops.ce_forward(hdn, wv, tgt, -100), iters=5)
    rec("ce_forward_16k_x_151k", ms, flops=2 * T2 * V * K)
    nll, lse = ops.ce_forward(hdn, wv, tgt, -100)
    gg = torch.ones(T2, device="cuda")
    buf = torch.empty(4096, V, device="cuda", dtype=torch.bfloat16)
    ms = timeit(lambda: ops.ce_dlogits(hdn[:4096], wv, tgt[:4096], lse[:4096], gg[:4096], buf, -100), iters=5)
    rec("ce_dlogits_4k_x_151k", ms, flops=2 * 4096 * V * K)
    del buf

    # ---------------- bandwidth-bound kernels
    for N in (128, 768, 1024, 4096, 7168):
        M = 32768
        ww = torch.ones(N, device="cuda", dtype=torch.bfloat16)
        sets = max(2, -(-(1 << 30) // (2 * M * N * 2)))
        xs = [torch.randn(M, N, device="cuda", dtype=torch.bfloat16) for _ in range(sets)]
        ms = timeit_rotating(lambda i: (lambda: ops.rms_norm_fwd(xs[i % sets], ww, 1e-6, False)), 2 * M * N * 2)
        ref = timeit_rotating(lambda i: (lambda: torch.nn.functional.rms_norm(xs[i % sets], (N,), ww, 1e-6)), 2 * M * N * 2)
        rec(f"rms_norm_fwd_N{N}", ms, bytes_=2 * M * N * 2, ref_ms=ref)
        outs = [ops.rms_norm_fwd(x_, ww, 1e-6, False) for x_ in xs]
        ms = timeit_rotating(lambda i: (lambda: ops.rms_norm_bwd(outs[i % sets][0], xs[i % sets], ww, outs[i % sets][1], False)), 3 * M * N * 2)
        rec(f"rms_norm_bwd_N{N}", ms, bytes_=3 * M * N * 2)
        del xs, outs
    n = 1 << 26
    a = torch.randn(n, device="cuda", dtype=torch.bfloat16)
    b = torch.randn(n, device="cuda", dtype=torch.bfloat16)
    ms = timeit(lambda: ops.silu_mul_fwd(a, b))
    rec("silu_mul_fwd_6.7e7", ms, bytes_=3 * n * 2)
    src = torch.randn(n, device="cuda")
    dst = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    ms = timeit(lambda: ops.sr_copy_(dst, src, 1))
    rec("sr_copy_6.7e7", ms, bytes_=n * 6)
    from d9d_b200.kernel.stochastic.adamw_step import AdamWLaunchPlan, adamw_stochastic_bf16_multi_

    p = torch.randn(n, device="cuda").bfloat16()
    g32 = torch.randn(n, device="cuda")
    m = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    v = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    plan = AdamWLaunchPlan([p], [g32], [m], [v])
    ms = timeit(lambda: adamw_stochastic_bf16_multi_([p], [g32], [m], [v], lr=1e-3, beta1=0.9, beta2=0.95, eps=1e-8, weight_decay=0.01, step=2, seed=3, plan=plan))
    rec("adamw_sr_bf16state_f32grad_6.7e7", ms, bytes_=n * (2 + 4 + 2 + 2 + 2 + 2 + 2))

    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()

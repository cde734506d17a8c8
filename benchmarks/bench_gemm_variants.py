"""GEMM variants side by side on one H100: single-CTA wgmma kernel, CTA-pair (two-CTA cluster, B multicast) kernel, cuBLAS (torch.matmul),
fp8 (row/column scaled) and MXFP8 kernels.  CUDA events, warm-up, L2 flush between iterations, median of ``--iters``.

    python benchmarks/bench_gemm_variants.py --out gpurun_out/bench_gemm_variants.json

Every variant is guarded: a failing variant records its error text instead of aborting the run.
"""

from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.bench_ops import timeit  # noqa: E402
from d9d_b200 import ops as _ops  # noqa: E402

SHAPES = [  # (M, N, K, note)
    (8192, 8192, 8192, "square"),
    (16384, 4096, 4096, "large"),
    (16384, 2048, 768, "flagship qkv"),
    (16384, 768, 2048, "flagship o-proj"),
    (16384, 14336, 4096, "llama-8b mlp up"),
    (4096, 4096, 16384, "deep K"),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/bench_gemm_variants.json")
    ap.add_argument("--iters", type=int, default=7)
    ap.add_argument("--variants", default="single,pair,cublas,fp8,mxfp8")
    args = ap.parse_args()
    ops = _ops.load()
    variants = args.variants.split(",")
    out = []
    for M, N, K, note in SHAPES:
        a = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        b = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
        d = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        flops = 2.0 * M * N * K
        row = {"M": M, "N": N, "K": K, "note": note}
        ref = None

        def run(name, fn, check=None):
            try:
                ms = timeit(fn, iters=args.iters)
                row[f"{name}_ms"] = ms
                row[f"{name}_tflops"] = flops / ms / 1e9
                if check is not None:
                    row[f"{name}_rel_err"] = check()
            except Exception as exc:  # noqa: BLE001
                row[f"{name}_error"] = repr(exc)[:300]

        if "cublas" in variants:
            run("cublas", lambda: torch.matmul(a, b.t(), out=d))
            ref = d.float().clone()

        def err():
            return ((d.float() - ref).norm() / ref.norm()).item() if ref is not None else None

        if "single" in variants:
            run("single", lambda: ops.gemm(a, b, d, False, False, False, 1), err)
        if "pair" in variants:
            run("pair", lambda: ops.gemm(a, b, d, False, False, False, 2), err)
        if "fp8" in variants:
            try:
                aq, sa = ops.quantize_rowwise(a)
                bq, sb = ops.quantize_rowwise(b)
                run("fp8", lambda: ops.gemm_fp8(aq, bq, sa, sb, 1.0, d), err)
                run("fp8_quantize_a", lambda: ops.quantize_rowwise(a))
            except Exception as exc:  # noqa: BLE001
                row["fp8_error"] = repr(exc)[:300]
        if "mxfp8" in variants and K % 128 == 0:
            try:
                aq, sfa = ops.quantize_mx(a)
                bq, sfb = ops.quantize_mx(b)
                run("mxfp8", lambda: ops.gemm_mxfp8(aq, sfa, bq, sfb, d), err)
            except Exception as exc:  # noqa: BLE001
                row["mxfp8_error"] = repr(exc)[:300]
        out.append(row)
        print(json.dumps(row), flush=True)
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

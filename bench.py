"""Headline benchmark: Qwen3-MoE pre-training throughput (tokens/s) on N H100s of one node.

Model/config = the reference's only end-to-end workload (``example/qwen3_moe/pretrain.json``): 16 layers,
hidden 768, 16 q / 4 kv heads x 128, 128 experts top-8 (expert FFN 576), vocab 151 669 (split regular/special),
bf16 weights, fp32 gradient accumulation, stochastic-rounding AdamW with bf16 states, grad-clip 5.0, microbatch 8.
Synthetic token data, random-init weights.  Weak scaling: every GPU processes ``--accum`` microbatches of
``8 x seq_len`` tokens per optimizer step (data-parallel replicas, summed gradients).

    python bench.py --gpus N --steps K --warmup W            # own implementation
    python bench.py --impl reference ...                     # unmodified reference from oracle/_ref (baseline/ref_bench.py)
    python bench.py --dump-outputs DIR ...                   # also write what the last timed step computed as DIR/*.npy

Prints ONE JSON line (rank 0).  Timed region = K optimizer steps bracketed by barrier + cuda synchronize, device
events, max over ranks.  ``e2e`` repeats the measurement through the public training API with every step's inputs
copied from pinned host memory and the loss read back to the host.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

FLAGSHIP = {
    "hidden_size": 768,
    "intermediate_size": 576,
    "num_experts": 128,
    "experts_top_k": 8,
    "num_attention_heads": 16,
    "num_key_value_heads": 4,
    "rms_norm_eps": 1e-6,
    "head_dim": 128,
    "num_hidden_layers": 16,
    "rope_base": 1_000_000,
    "split_vocab_size": {"regular": 151643, "special": 26},
    "split_vocab_order": ["regular", "special"],
}


def positive_int(text: str) -> int:
    value = int(text)
    if value < 1:
        raise argparse.ArgumentTypeError(f"must be >= 1, got {value}")
    return value


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=positive_int, default=5, help="timed optimizer steps")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="own", choices=["own", "reference"])
    ap.add_argument("--seq-len", type=int, default=2048)
    ap.add_argument("--microbatch", type=int, default=8)
    ap.add_argument("--accum", type=int, default=2, help="microbatches per GPU per optimizer step")
    ap.add_argument("--layers", type=int, default=FLAGSHIP["num_hidden_layers"])
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--fp8-dense", action="store_true",
                    help="EXPERIMENT (not the headline: reduced precision): attention projections run forward / dgrad / wgrad in e4m3 "
                         "(d9d_b200.kernel.fp8.Fp8Linear); experts, router and LM head stay bf16")
    ap.add_argument("--dp-impl", default="nvlink", choices=["nvlink", "nccl"],
                    help="multi-GPU gradient path of the device-timed arm: own NVLink peer-memory kernels or NCCL all-reduce")
    ap.add_argument("--layout", default="dp", choices=["dp", "ep", "example"],
                    help="dp: every GPU holds the whole model (headline, comparable with the reference arm); ep: experts sharded "
                         "over all GPUs (expert parallel = N, NVLink dispatch / combine), dense parameters replicated; example: the "
                         "reference example's PP4 x DP2 x EP2 layout with looped_bfs, 2 stages per rank (8 GPUs)")
    ap.add_argument("--model", default="example", choices=["example", "30b-a3b"],
                    help="example: the reference's example/qwen3_moe/pretrain.json model; 30b-a3b: Qwen3-30B-A3B shape (needs --layout ep on 8 GPUs)")
    ap.add_argument("--checkpointing", action="store_true", help="per-layer activation checkpointing (needed by the 30b-a3b shape)")
    ap.add_argument("--ep-capacity-factor", type=float, default=2.0,
                    help="receive capacity of an expert-parallel rank as a multiple of its fair share (0 = worst case)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the loss of the last step and a fixed sample of the updated parameters "
                         "as DIR/<name>.npy (float32), so that two builds can be compared output for output (--layout dp)")
    return ap.parse_args()


class ClockSampler:
    """Samples nvidia-smi clocks / throttle reasons during the timed region."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index = index
        self.samples: list[list[str]] = []
        self._stop = threading.Event()
        self._thread: threading.Thread | None = None

    def _run(self):
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", str(self.index)],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.samples.append([c.strip() for c in out.split(",")])
            except Exception:
                pass
            self._stop.wait(0.2)

    def start(self):
        self._thread = threading.Thread(target=self._run, daemon=True)
        self._thread.start()

    def stop(self) -> dict:
        self._stop.set()
        if self._thread:
            self._thread.join(timeout=6)
        sm = sorted(float(s[0]) for s in self.samples if s and s[0].replace(".", "").isdigit())
        reasons = set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for s in self.samples:
            for name, val in zip(names, s[3:7]):
                if val.lower().startswith("active"):
                    reasons.add(name)
        return {
            "sm_mhz": sm[len(sm) // 2] if sm else None,
            "sm_max_mhz": float(self.samples[0][1]) if self.samples else None,
            "reasons": sorted(reasons),
            "samples": len(self.samples),
        }


def reference_arm(args) -> None:
    """Runs the UNMODIFIED reference (``oracle/_ref``, made by ``build()``; see ``baseline/ref_bench.py``) on the same workload."""
    import importlib.util

    here = os.path.dirname(os.path.abspath(__file__))
    rank0 = int(os.environ.get("RANK", "0")) == 0

    def unavailable(why: str) -> None:
        if rank0:
            print(json.dumps({"impl": "reference", "unavailable": why}))

    def load(name: str):
        spec = importlib.util.spec_from_file_location(name, os.path.join(here, "baseline", f"{name}.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod

    if not os.path.isdir(os.path.join(here, "oracle", "_ref", "d9d")):
        return unavailable("oracle/_ref is missing: build() makes it where the reference source is present")
    try:
        result = load("ref_bench").run(args, FLAGSHIP, ClockSampler)
    except Exception as exc:  # noqa: BLE001 - the contract is: print the reason, exit 0
        import traceback

        traceback.print_exc()
        return unavailable(f"reference failed to run: {type(exc).__name__}: {str(exc)[:300]}".replace("\n", " "))
    if rank0:
        print(json.dumps(result))


QWEN3_30B_A3B = {**FLAGSHIP, "hidden_size": 2048, "intermediate_size": 768, "num_attention_heads": 32, "num_key_value_heads": 4,
                 "num_hidden_layers": 48}


def model_spec(args) -> dict:
    return QWEN3_30B_A3B if getattr(args, "model", "example") == "30b-a3b" else FLAGSHIP


def model_name(args) -> str:
    m = model_spec(args)
    tag = "Qwen3-30B-A3B shape" if m is QWEN3_30B_A3B else "qwen3_moe example/pretrain.json"
    return (f"{tag} ({args.layers}L h{m['hidden_size']} {m['num_attention_heads']}q/{m['num_key_value_heads']}kv x{m['head_dim']} "
            f"E{m['num_experts']} top{m['experts_top_k']} ffn{m['intermediate_size']} vocab{sum(m['split_vocab_size'].values())})")


def expert_parallel_arm(args) -> None:
    """Experts sharded over all N GPUs (EP = N, NVLink peer-memory dispatch / combine), dense parameters replicated and
    reduced by the bucketed gradient synchroniser; everything runs through the public Trainer API, device-timed with CUDA
    events inside the run, so ``value`` and ``e2e`` are the same measurement."""
    import contextlib
    import tempfile

    import torch
    import torch.distributed as dist

    from d9d_b200 import ops
    from d9d_b200.bench_support import TrainerEndToEnd

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torch.distributed.run --nproc-per-node {args.gpus}")
    os.environ["D9D_EP_CAPACITY_FACTOR"] = str(args.ep_capacity_factor)
    torch.cuda.set_device(local_rank)
    ops.load()
    vocab = sum(model_spec(args)["split_vocab_size"].values())
    sampler = ClockSampler(local_rank)
    with tempfile.TemporaryDirectory() as workdir, contextlib.redirect_stdout(sys.stderr):
        runner = TrainerEndToEnd(args, world, flagship_params(args), vocab, workdir, layout=args.layout)
        if rank == 0:
            sampler.start()
        res = runner.run()
    clocks = sampler.stop() if rank == 0 else None
    tokens = args.accum * args.microbatch * args.seq_len * world
    value = tokens / (res["ms_per_step"] / 1e3)
    if rank == 0:
        print(json.dumps({
            "metric": "Qwen3-MoE pretrain tokens/sec (max over ranks)", "value": value, "unit": "tokens/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": res["ms_per_step"], "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "bf16", "data": "synthetic tokens, random-init weights", "impl": "own",
            "config": {"model": model_name(args), "global_batch": args.accum * args.microbatch * world, "microbatch": args.microbatch,
                       "seq_len": args.seq_len,
                       "parallelism": (f"ep{world} x dp{world} (experts sharded {world}-way over NVLink peer-memory dispatch/combine, "
                                       f"capacity factor {args.ep_capacity_factor}; dense params replicated, NCCL bucketed all-reduce)"
                                       if args.layout == "ep" else
                                       "pp4 x dp2 x ep2, looped_bfs 2 stages/rank (the reference example's layout), NCCL p2p between "
                                       f"stages, NVLink EP dispatch/combine (capacity factor {args.ep_capacity_factor})"),
                       "optimizer": "stochastic_adamw bf16 states, fp32 grads, clip 5.0",
                       "activation_checkpointing": bool(args.checkpointing),
                       "l2": "working set exceeds the 50 MB L2"},
            "clocks": clocks,
            "e2e": {"value": value, "unit": "tokens/s", "h2d_bytes_per_step": res["h2d_bytes_per_step"],
                    "d2h_bytes_per_step": res["d2h_bytes_per_step"], "ms_per_step": res["ms_per_step"], "final_loss": res["final_loss"],
                    "ep_overflow": res.get("ep_overflow"),
                    "api": "d9d_b200.loop.run.TrainingConfigurator(...).configure().train(); pinned-memory StatefulDataLoader"},
            "gpu_launches": res["launches"], "final_loss": res["final_loss"]}))
    if dist.is_initialized():
        dist.destroy_process_group()


def flagship_params(args):
    from d9d_b200.module.model.qwen3_moe import Qwen3MoEForCausalLMParameters, Qwen3MoELayerParameters, Qwen3MoEParameters

    spec = model_spec(args)
    layer = Qwen3MoELayerParameters(**{k: spec[k] for k in (
        "hidden_size", "intermediate_size", "num_experts", "experts_top_k", "num_attention_heads",
        "num_key_value_heads", "rms_norm_eps", "head_dim")})
    return Qwen3MoEForCausalLMParameters(model=Qwen3MoEParameters(
        layer=layer, num_hidden_layers=args.layers, rope_base=FLAGSHIP["rope_base"],
        max_position_ids=max(args.seq_len, 4096), split_vocab_size=FLAGSHIP["split_vocab_size"],
        split_vocab_order=FLAGSHIP["split_vocab_order"]))


def build_model(args, device):
    import torch

    from d9d_b200.module.block.hidden_states_aggregator import HiddenStatesAggregationMode
    from d9d_b200.module.model.qwen3_moe import Qwen3MoEForCausalLM
    from d9d_b200.pipelining.api import PipelineStageInfo

    params = flagship_params(args)
    with torch.device(device):
        model = Qwen3MoEForCausalLM(params, PipelineStageInfo(0, 1), HiddenStatesAggregationMode.no, False).bfloat16()
    model.reset_parameters()
    if getattr(args, "fp8_dense", False):
        from d9d_b200.kernel.fp8 import convert_linears_to_fp8

        n = convert_linears_to_fp8(model, lambda name, m: "self_attn" in name)
        print(f"[bench] fp8: {n} attention projections converted to Fp8Linear", file=sys.stderr, flush=True)
    return model


# parameters sampled by --dump-outputs: at most this many elements of each, at fixed seeded positions
DUMP_SAMPLES_PER_PARAM = 16384


def dump_outputs(out_dir: str, loss, model) -> None:
    """The loss of the last timed step and a sample of every parameter after its optimizer update (what a caller of the
    training step receives), as float32 ``.npy`` files.  The sample positions depend only on the parameter's size."""
    import numpy as np
    import torch

    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "loss.npy"), loss.detach().float().cpu().numpy().reshape(-1))
    samples = []
    for _name, param in sorted(model.named_parameters(), key=lambda kv: kv[0]):
        flat = param.detach().reshape(-1)
        if flat.numel() > DUMP_SAMPLES_PER_PARAM:
            gen = torch.Generator().manual_seed(flat.numel())
            idx = torch.randint(0, flat.numel(), (DUMP_SAMPLES_PER_PARAM,), generator=gen).to(flat.device)
            flat = flat[idx]
        samples.append(flat.float().cpu())
    np.save(os.path.join(out_dir, "params_sample.npy"), torch.cat(samples).numpy())


def main():
    args = parse_args()
    if args.dump_outputs and (args.impl != "own" or args.layout != "dp"):
        raise SystemExit("--dump-outputs is implemented for the device-timed arm (--impl own --layout dp)")
    if args.model == "30b-a3b" and args.layers == FLAGSHIP["num_hidden_layers"]:
        args.layers = QWEN3_30B_A3B["num_hidden_layers"]
    if args.impl == "reference":
        reference_arm(args)
        return
    if args.layout in ("ep", "example"):
        expert_parallel_arm(args)
        return

    import torch
    import torch.distributed as dist

    from d9d_b200 import ops
    from d9d_b200.bench_support import TrainStepRunner

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus:
        raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={world}: launch with torch.distributed.run --nproc-per-node {args.gpus}")
    torch.cuda.set_device(local_rank)
    device = torch.device("cuda", local_rank)
    ops.load()

    runner = TrainStepRunner(args, device, world, build_model)
    vocab = sum(model_spec(args)["split_vocab_size"].values())
    tokens_per_step_per_gpu = args.accum * args.microbatch * args.seq_len
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=device)

    def barrier():
        if world > 1:
            dist.barrier(device_ids=[local_rank])
        torch.cuda.synchronize()

    # ---------------------------------------------------------------- device-timed headline number
    gen = torch.Generator(device=device).manual_seed(1234 + rank)
    batches = [runner.synthetic_batch(vocab, gen) for _ in range(max(args.warmup + args.steps, 1) * args.accum)]
    it = iter(batches)
    # the training loop of the framework collects garbage manually every N steps (loop/component/garbage_collector.py); do the
    # same here so that no cyclic collection (0.1 s+ on this heap) stalls the launching thread inside the timed region
    import gc as _gc

    _gc.collect()
    _gc.disable()
    for _ in range(args.warmup):
        runner.step([next(it) for _ in range(args.accum)])
    barrier()
    launches_before = runner.launch_count()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    flush.zero_()  # inputs/weights (6 GB) are far larger than the 50 MB L2; flush once before timing anyway
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    start.record()
    for _ in range(args.steps):
        loss = runner.step([next(it) for _ in range(args.accum)])
    end.record()
    barrier()
    clocks = sampler.stop() if rank == 0 else None
    ms = torch.tensor([start.elapsed_time(end)], device=device)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_per_step = ms.item() / args.steps
    _gc.enable()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss, runner.model)
    launches = runner.launch_count() - launches_before
    value = tokens_per_step_per_gpu * world / (ms_per_step / 1e3)

    # ---------------------------------------------------------------- end-to-end through the public Trainer API
    e2e = None
    if not args.no_e2e:
        import gc
        import tempfile

        from d9d_b200.bench_support import TrainerEndToEnd

        final_loss = float(loss)
        del runner, batches, it, loss
        gc.collect()
        torch.cuda.empty_cache()
        import contextlib

        with tempfile.TemporaryDirectory() as workdir, contextlib.redirect_stdout(sys.stderr):  # stdout carries ONE json line
            res = TrainerEndToEnd(args, world, flagship_params(args), vocab, workdir).run()
        e2e = {"value": tokens_per_step_per_gpu * world / (res["ms_per_step"] / 1e3), "unit": "tokens/s",
               "h2d_bytes_per_step": res["h2d_bytes_per_step"], "d2h_bytes_per_step": res["d2h_bytes_per_step"],
               "ms_per_step": res["ms_per_step"], "final_loss": res["final_loss"], "gpu_launches": res["launches"],
               "api": "d9d_b200.loop.run.TrainingConfigurator(...).configure().train(); pinned-memory StatefulDataLoader; optimizer="
                      + ("nvlink_sharded_adamw" if world > 1 and args.dp_impl == "nvlink" else "stochastic_adamw")}
    else:
        final_loss = float(loss)

    if rank == 0:
        print(json.dumps({
            "metric": "Qwen3-MoE pretrain tokens/sec (max over ranks)",
            "value": value,
            "unit": "tokens/s",
            "n_gpus": world,
            "steps": args.steps,
            "warmup": args.warmup,
            "ms_per_step": ms_per_step,
            "higher_is_better": True,
            "scaling": "weak",
            "vs_baseline": None,
            "dtype": "bf16" if not args.fp8_dense else "bf16 + e4m3 attention projections (EXPERIMENT, not the headline)",
            "data": "synthetic tokens, random-init weights",
            "impl": "own",
            "config": {
                "model": model_name(args),
                "global_batch": args.accum * args.microbatch * world,
                "microbatch": args.microbatch,
                "seq_len": args.seq_len,
                "parallelism": (f"dp{world} ({'NVLink reduce-scatter+AdamW+all-gather kernels' if args.dp_impl == 'nvlink' else 'NCCL all-reduce'})"
                                if world > 1 else "single"),
                "optimizer": "stochastic_adamw bf16 states, fp32 grads, clip 5.0",
                "l2": "working set (>10 GB weights+grads+activations) exceeds the 50 MB L2; 256 MB flush before timing",
            },
            "clocks": clocks,
            "e2e": e2e,
            "gpu_launches": launches,
            "final_loss": final_loss,
        }))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

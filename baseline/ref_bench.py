"""Reference arm of ``bench.py``: the UNMODIFIED reference (``oracle/_ref/d9d``, made by ``build()``) on the headline workload.

Everything on the measured path is the reference's own stock code: ``d9d.loop.run.TrainingConfigurator`` /
``Trainer.train()``, its ``Qwen3MoEForCausalLM``, its Triton kernels (RMSNorm, SiLU*mul, MoE permute, stochastic
AdamW), ``GradientSynchronizer`` and ``StochasticAdamW``, driven through the reference example's own
``ProjectModelProvider`` and ``SFTTask`` (``oracle/_ref/example/qwen3_moe/pretrain.py``).  The dataset provider is
synthetic (no network for datasets / tokenizers), batches leave a pinned-memory ``StatefulDataLoader`` exactly as in the
example.  Third-party wheels the reference imports but which cannot be installed offline are replaced by stand-in
*packages* that live in ``baseline/shims`` and are only importable from this process:

* ``flash_attn.cute`` (FlashAttention-4)  -> the real FA4 CuTe-DSL kernels vendored inside the image's vLLM wheel
  (``vllm/vllm_flash_attn/cute``), aliased under the upstream name; falls back to cuDNN SDPA if they fail to JIT;
* ``grouped_gemm``                        -> ``torch._grouped_mm`` (libtorch CUTLASS) / per-expert cuBLAS loop;
* ``cut_cross_entropy``                   -> row-chunked PyTorch + cuBLAS (exact gradients).

``d9d_b200`` is never imported here and its extension is never loaded (asserted below).
"""

from __future__ import annotations

import contextlib
import importlib
import importlib.machinery
import importlib.util
import json
import os
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
REF = os.path.join(REPO, "oracle", "_ref")


def _isolate_sys_path() -> None:
    drop = {REPO, "", "."}
    sys.path[:] = [p for p in sys.path if os.path.abspath(p or ".") not in {os.path.abspath(d or ".") for d in drop} or p == HERE]
    sys.path[:0] = [os.path.join(HERE, "shims"), REF, os.path.join(REF, "example", "qwen3_moe")]


def _stub_package(name: str, path: str) -> types.ModuleType:
    mod = types.ModuleType(name)
    mod.__path__ = [path]
    mod.__package__ = name
    mod.__spec__ = importlib.machinery.ModuleSpec(name, None, is_package=True)
    mod.__spec__.submodule_search_locations = [path]
    sys.modules[name] = mod
    return mod


STAND_INS: dict[str, str] = {}


def _install_flash_attn_cute() -> None:
    """Expose FlashAttention-4 under its upstream name ``flash_attn.cute`` (the reference imports its private
    ``_flash_attn_fwd`` / ``_flash_attn_bwd``)."""
    iface = types.ModuleType("flash_attn.cute.interface")
    state: dict = {"impl": None}

    def _load_fa4():
        spec = importlib.util.find_spec("vllm")
        if spec is None or spec.origin is None:
            raise ImportError("vllm wheel (vendoring FA4's cute kernels) not found")
        root = os.path.dirname(spec.origin)
        # bypass vllm/__init__ and vllm_flash_attn/__init__ (they load unrelated FA2/FA3 extensions)
        if "vllm" not in sys.modules:
            _stub_package("vllm", root)
        if "vllm.vllm_flash_attn" not in sys.modules:
            _stub_package("vllm.vllm_flash_attn", os.path.join(root, "vllm_flash_attn"))
        return importlib.import_module("vllm.vllm_flash_attn.cute.interface")

    def _sdpa_fwd(q, k, v, softmax_scale=None, causal=False, window_size_left=None, window_size_right=None,
                  learnable_sink=None, softcap=None, return_lse=False, lse=None, **_):
        import torch

        if learnable_sink is not None or softcap or window_size_left is not None or window_size_right not in (None, 0):
            raise NotImplementedError("cuDNN stand-in: plain / causal attention only")
        out, lse_, *_rest = torch.ops.aten._scaled_dot_product_cudnn_attention(
            q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), None, True, 0.0, causal, False, scale=softmax_scale)
        state["cudnn_ctx"] = _rest
        return out.transpose(1, 2), lse_

    def _sdpa_bwd(q, k, v, out, dout, lse, softmax_scale=None, causal=False, softcap=0.0, **_):
        import torch

        cum_q, cum_k, max_q, max_k, seed, offset, _dbg = state["cudnn_ctx"]
        dq, dk, dv = torch.ops.aten._scaled_dot_product_cudnn_attention_backward(
            dout.transpose(1, 2), q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), out.transpose(1, 2), lse,
            seed, offset, None, cum_q, cum_k, max_q, max_k, 0.0, causal, scale=softmax_scale)
        return dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2)

    def _pick():
        if state["impl"] is None:
            if os.environ.get("D9D_REF_ATTENTION", "fa4") == "fa4":
                try:
                    mod = _load_fa4()
                    state["impl"] = (mod._flash_attn_fwd, mod._flash_attn_bwd)
                    STAND_INS["flash_attn.cute"] = "FlashAttention-4 CuTe-DSL kernels vendored in the vLLM wheel (same upstream code)"
                except Exception as exc:  # noqa: BLE001
                    print(f"[ref] FA4 unavailable ({type(exc).__name__}: {exc}); using cuDNN SDPA", file=sys.stderr, flush=True)
            if state["impl"] is None:
                state["impl"] = (_sdpa_fwd, _sdpa_bwd)
                STAND_INS["flash_attn.cute"] = "cuDNN flash attention via torch.ops.aten._scaled_dot_product_cudnn_attention(+_backward)"
        return state["impl"]

    def _flash_attn_fwd(*a, **kw):
        fwd, _ = _pick()
        try:
            return fwd(*a, **kw)
        except Exception as exc:  # noqa: BLE001 - JIT failure on first use: switch to the library kernel once
            if fwd is _sdpa_fwd:
                raise
            print(f"[ref] FA4 forward failed ({type(exc).__name__}: {str(exc)[:200]}); using cuDNN SDPA", file=sys.stderr, flush=True)
            state["impl"] = (_sdpa_fwd, _sdpa_bwd)
            STAND_INS["flash_attn.cute"] = "cuDNN flash attention via torch.ops.aten._scaled_dot_product_cudnn_attention(+_backward)"
            kw.pop("num_splits", None), kw.pop("pack_gqa", None)
            return _sdpa_fwd(*a, **kw)

    def _flash_attn_bwd(*a, **kw):
        return _pick()[1](*a, **kw)

    iface._flash_attn_fwd, iface._flash_attn_bwd = _flash_attn_fwd, _flash_attn_bwd
    fa = _stub_package("flash_attn", os.path.join(HERE, "shims", "_flash_attn_stub"))
    cute = _stub_package("flash_attn.cute", os.path.join(HERE, "shims", "_flash_attn_stub", "cute"))
    fa.cute, cute.interface = cute, iface
    sys.modules["flash_attn.cute.interface"] = iface


def _synthetic_provider(num_samples: int, seq_len: int, vocab: int, seed: int):
    import torch
    from d9d.dataset import shard_dataset_data_parallel
    from d9d.loop.control import DatasetProvider, InitializeDatasetContext, InitializeDatasetResult
    from torch.utils.data import Dataset

    class SyntheticTokens(Dataset):
        def __len__(self) -> int:
            return num_samples

        def __getitem__(self, index: int):
            g = torch.Generator().manual_seed(seed * 1_000_003 + index)
            tok = torch.randint(0, vocab, (seq_len + 1,), generator=g)
            return {"input_ids": tok[:-1], "labels": tok[1:], "position_ids": torch.arange(seq_len)}

    def collate(batch):
        return {k: torch.stack([b[k] for b in batch]) for k in batch[0]}

    class Provider(DatasetProvider):
        def __call__(self, context: InitializeDatasetContext) -> InitializeDatasetResult:
            return InitializeDatasetResult(dataset=shard_dataset_data_parallel(SyntheticTokens(), context.dist_context),
                                           collator=collate)

    return Provider()


def run(args, flagship: dict, clock_sampler_cls) -> dict:
    _isolate_sys_path()
    _install_flash_attn_cute()
    STAND_INS["grouped_gemm"] = "torch._grouped_mm (libtorch CUTLASS grouped GEMM); per-expert cuBLAS loop fallback"
    STAND_INS["cut_cross_entropy"] = "row-chunked PyTorch/cuBLAS linear-cross-entropy, exact gradients (no gradient filtering)"

    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29517")
    os.environ.setdefault("RANK", "0"), os.environ.setdefault("LOCAL_RANK", "0"), os.environ.setdefault("WORLD_SIZE", "1")
    torch.cuda.set_device(local_rank)

    import pretrain as example  # the reference example module (providers / task), unmodified
    from d9d.core.dist_context import DeviceMeshParameters
    from d9d.loop.auto import AutoLRSchedulerProvider, AutoOptimizerProvider
    from d9d.loop.config import TrainerConfig
    from d9d.loop.event.catalogue.train import EVENT_TRAIN_STEP_POST, EVENT_TRAIN_STEP_PRE
    from d9d.loop.run import TrainingConfigurator
    from pydantic import TypeAdapter

    assert "d9d_b200" not in sys.modules, "reference arm must not import the repo's package"

    total_steps = args.warmup + args.steps
    global_batch = args.accum * args.microbatch * world
    vocab = sum(flagship["split_vocab_size"].values())
    model_cfg = {"model": {"model": {
        "layer": {k: flagship[k] for k in ("hidden_size", "intermediate_size", "num_experts", "experts_top_k",
                                           "num_attention_heads", "num_key_value_heads", "rms_norm_eps", "head_dim")},
        "num_hidden_layers": args.layers, "rope_base": flagship["rope_base"], "max_position_ids": max(args.seq_len, 4096),
        "split_vocab_size": flagship["split_vocab_size"], "split_vocab_order": flagship["split_vocab_order"],
        "pipeline_num_virtual_layers_pre": 0, "pipeline_num_virtual_layers_post": 0}}, "checkpointing": False}

    workdir = tempfile.mkdtemp(prefix="d9d_ref_bench_")
    trainer_cfg = {
        "run": {"name": "bench", "description": None, "hparams": {}},
        "batching": {"global_batch_size": global_batch, "microbatch_size": args.microbatch},
        "data_loading": {"num_workers": 0, "pin_memory": True, "persistent_workers": False},
        "logging": {"period_steps": 10_000, "tracker": {"provider": "null"}},
        "pipelining": {"schedule": {"schedule": "gpipe"}},
        "model_stage_factory": {"source_checkpoint": None, "checkpoint_only_trainable_parameters": False},
        "determinism": {"base_seed": 1337},
        "gc": {"period_steps": 10_000},
        "checkpointing": {"save_dir": workdir, "period_steps": "disable", "num_to_keep": 1},
        "gradient_clipping": {"max_norm": 5.0, "log_total_steps": 10_000},
        "profiling": None,
        "gradient_manager": {"grad_dtype": "float32", "bucket_size_mb": 32},
        "timeout": {"init_timeout": 10_000, "step_timeout": 600},
    }
    opt_cfg = TypeAdapter(example.AutoOptimizerConfig).validate_python(
        {"name": "stochastic_adamw", "lr": 2.5e-4, "state_dtype": "bfloat16"})
    lr_cfg = TypeAdapter(example.AutoLRSchedulerConfig).validate_python(
        {"name": "piecewise", "scheduler": {"initial_multiplier": 1.0, "phases": [
            {"mode": "rest", "target_multiplier": 1.0, "curve": {"type": "linear"}}]}})

    with contextlib.redirect_stdout(sys.stderr):
        trainer = TrainingConfigurator(
            mesh=DeviceMeshParameters(data_parallel_replicate=world),
            parameters=TrainerConfig.model_validate(trainer_cfg),
            task_provider=lambda ctx: example.SFTTask(ctx.dist_context),
            model_provider=example.ProjectModelProvider(example.ModelProviderConfig.model_validate(model_cfg)),
            data_provider=_synthetic_provider(global_batch * total_steps, args.seq_len, vocab, seed=5),
            optimizer_provider=AutoOptimizerProvider(opt_cfg),
            lr_scheduler_provider=AutoLRSchedulerProvider(lr_cfg),
        ).configure()
    state = trainer._state  # noqa: SLF001 - the reference exposes the job state only privately

    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler = clock_sampler_cls(local_rank)
    flush = torch.empty(192 * 1024 * 1024, dtype=torch.uint8, device="cuda")

    def pre(ctx) -> None:
        if ctx.stepper.current_step == args.warmup:
            state.dist_context.wait_world()
            torch.cuda.synchronize()
            flush.zero_()
            if rank == 0:
                sampler.start()
            torch.cuda.synchronize()
            start.record()

    def post(ctx) -> None:
        if ctx.stepper.current_step == total_steps - 1:
            end.record()
            state.dist_context.wait_world()
            torch.cuda.synchronize()

    state.event_bus.subscribe(EVENT_TRAIN_STEP_PRE, pre)
    state.event_bus.subscribe(EVENT_TRAIN_STEP_POST, post)
    with contextlib.redirect_stdout(sys.stderr):
        trainer.train()
    torch.cuda.synchronize()
    clocks = sampler.stop() if rank == 0 else None
    ms = torch.tensor([start.elapsed_time(end)], device="cuda")
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_per_step = ms.item() / args.steps
    assert "d9d_b200" not in sys.modules
    tokens_per_step = args.accum * args.microbatch * args.seq_len * world
    value = tokens_per_step / (ms_per_step / 1e3)
    h2d = args.accum * 3 * args.microbatch * args.seq_len * 8
    result = {
        "metric": "Qwen3-MoE pretrain tokens/sec (max over ranks)",
        "value": value, "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_per_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
        "data": "synthetic tokens, random-init weights", "impl": "reference",
        "reference_class": "stock code, stand-in third-party wheels",
        "stand_ins": STAND_INS,
        "config": {
            "model": f"qwen3_moe example/pretrain.json ({args.layers}L h768 16q/4kv x128 E128 top8 ffn576 vocab151669)",
            "global_batch": global_batch, "microbatch": args.microbatch, "seq_len": args.seq_len,
            "parallelism": f"dp{world} (reference GradientSynchronizer, NCCL all-reduce)" if world > 1 else "single",
            "optimizer": "stochastic_adamw bf16 states, fp32 grads, clip 5.0",
            "l2": "working set (>10 GB) exceeds the 50 MB L2; 256 MB flush before timing",
        },
        "clocks": clocks,
        # the reference has one code path: Trainer.train() - the device-timed number IS the end-to-end number
        "e2e": {"value": value, "unit": "tokens/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4, "ms_per_step": ms_per_step,
                "api": "d9d.loop.run.TrainingConfigurator(...).configure().train(); pinned-memory StatefulDataLoader; loss.item() per step"},
        "gpu_launches": 0,
    }
    if dist.is_initialized():
        with contextlib.suppress(Exception):
            dist.destroy_process_group()
    return result

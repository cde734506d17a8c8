"""The driver's contract with ``bench.py`` / ``__graft_entry__.py`` as far as it can be checked without a GPU: defaults, the
model the headline is quoted on, the reference arm's "unavailable" protocol."""

import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def _bench():
    import importlib.util

    spec = importlib.util.spec_from_file_location("bench_under_test", ROOT / "bench.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_defaults_are_one_gpu_and_a_short_run(monkeypatch):
    bench = _bench()
    monkeypatch.setattr(sys, "argv", ["bench.py"])
    args = bench.parse_args()
    assert args.gpus == 1 and args.impl == "own" and args.layout == "dp" and args.model == "example"
    assert args.warmup >= 3 and 1 <= args.steps <= 20  # the timing rules ask for >= 3 warm-up steps; finishes within minutes
    assert not args.fp8_dense and not args.checkpointing


def test_flagship_is_the_reference_example_model():
    bench = _bench()
    example = json.loads((ROOT / "example" / "qwen3_moe" / "pretrain.json").read_text())["model_provider"]["model"]["model"]
    for key, value in example["layer"].items():
        assert bench.FLAGSHIP[key] == value, key
    assert bench.FLAGSHIP["num_hidden_layers"] == example["num_hidden_layers"]
    assert bench.FLAGSHIP["split_vocab_size"] == example["split_vocab_size"]
    assert bench.FLAGSHIP["split_vocab_order"] == example["split_vocab_order"]


def test_reference_arm_reports_unavailable_as_one_json_line(tmp_path):
    """Without ``oracle/_ref`` (no reference install was built) the arm must print the reason and exit 0."""
    work = tmp_path / "repo"
    (work / "baseline").mkdir(parents=True)
    for name in ("bench.py",):
        (work / name).write_text((ROOT / name).read_text())
    out = subprocess.run([sys.executable, str(work / "bench.py"), "--impl", "reference"], capture_output=True, text=True, timeout=120,
                         env={**os.environ, "PYTHONPATH": str(ROOT)})
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [line for line in out.stdout.splitlines() if line.strip()]
    assert len(lines) == 1
    record = json.loads(lines[0])
    assert record["impl"] == "reference" and "unavailable" in record and "\n" not in record["unavailable"]


def test_steps_must_be_positive(monkeypatch, capsys):
    bench = _bench()
    monkeypatch.setattr(sys, "argv", ["bench.py", "--steps", "0"])
    try:
        bench.parse_args()
    except SystemExit as exc:
        assert exc.code == 2
    else:
        raise AssertionError("--steps 0 was accepted")
    monkeypatch.setattr(sys, "argv", ["bench.py", "--steps", "7"])
    assert bench.parse_args().steps == 7


def test_dump_outputs_writes_float32_loss_and_a_fixed_parameter_sample(tmp_path):
    import numpy as np
    import torch

    bench = _bench()
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(300, 200), torch.nn.LayerNorm(200)).bfloat16()
    loss = torch.tensor([2.5])
    bench.dump_outputs(str(tmp_path / "a"), loss, model)
    bench.dump_outputs(str(tmp_path / "b"), loss, model)
    got_loss = np.load(tmp_path / "a" / "loss.npy")
    sample = np.load(tmp_path / "a" / "params_sample.npy")
    assert got_loss.dtype == np.float32 and got_loss.tolist() == [2.5]
    sizes = [p.numel() for p in model.parameters()]
    assert sample.dtype == np.float32 and sample.size == sum(min(n, bench.DUMP_SAMPLES_PER_PARAM) for n in sizes)
    np.testing.assert_array_equal(sample, np.load(tmp_path / "b" / "params_sample.npy"))  # same positions every time
    params = dict(model.named_parameters())  # written in name order: 0.bias (whole), 0.weight (sampled), 1.bias, 1.weight
    bias = params["0.bias"].detach().float().numpy()
    np.testing.assert_array_equal(sample[: bias.size], bias)
    weight = sample[bias.size : bias.size + bench.DUMP_SAMPLES_PER_PARAM]
    assert set(weight.tolist()) <= set(params["0.weight"].detach().float().reshape(-1).numpy().tolist())


def test_graft_entry_exposes_build_and_smoke():
    import importlib.util

    spec = importlib.util.spec_from_file_location("graft_entry_under_test", ROOT / "__graft_entry__.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert callable(mod.build) and callable(mod.smoke)


def test_end_to_end_arm_plumbing_runs_on_cpu(tmp_path, monkeypatch):
    """The Trainer job ``bench.py`` times for its ``e2e`` number (providers, loader, optimizer, loss logging), dry-run on CPU with
    a tiny model: the timing itself needs CUDA events, the plumbing does not."""
    import types

    import d9d_b200.bench_support as support
    from d9d_b200.module.model.qwen3_moe import Qwen3MoEForCausalLMParameters, Qwen3MoELayerParameters, Qwen3MoEParameters

    original = support.trainer_config_for_bench

    def without_pinned_memory(*a, **k):
        cfg = original(*a, **k)
        cfg["data_loading"]["pin_memory"] = False  # pinning needs a CUDA runtime
        return cfg

    monkeypatch.setattr(support, "trainer_config_for_bench", without_pinned_memory)
    args = types.SimpleNamespace(warmup=1, steps=2, accum=2, microbatch=2, seq_len=32, layout="dp", dp_impl="nvlink", checkpointing=False)
    params = Qwen3MoEForCausalLMParameters(model=Qwen3MoEParameters(
        layer=Qwen3MoELayerParameters(hidden_size=64, intermediate_size=32, num_experts=4, experts_top_k=2, num_attention_heads=4,
                                      num_key_value_heads=2, rms_norm_eps=1e-6, head_dim=16),
        num_hidden_layers=2, rope_base=10000, max_position_ids=64, split_vocab_size={"regular": 200, "special": 24},
        split_vocab_order=["regular", "special"]))
    job = support.TrainerEndToEnd(args, 1, params, 224, str(tmp_path))
    job.trainer.train()
    assert job.trainer.state.stepper.current_step == 3
    assert 0 < float(job.trainer.state.logger.last_loss) < 10

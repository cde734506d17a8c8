"""Every parallelism on real GPUs (NCCL / NVLink), mirroring the reference's distributed tier
(``test/d9d_test/modules/model/meshes.py`` - 10 meshes on 8 GPUs - and ``test/d9d_test/pipelining/test_e2e.py``).

* whole-model checks: the model is parallelised over a mesh, one step runs through the gradient machinery and every
  parameter's global gradient is compared (direction + norm, bf16 kernels) with the single-GPU gradient over the global
  batch - ``benchmarks/validate_parallelism_gpu.py`` under ``torchrun`` at the largest world size the box offers;
* pipeline schedules end to end over NCCL p2p.

Skipped on boxes with fewer than 2 GPUs.
"""

import os
import subprocess
import sys

import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus() -> int:
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _torchrun(world: int, script_args: list[str], timeout: int = 420, env: dict[str, str] | None = None) -> None:
    port = 29800 + (os.getpid() % 150)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), *script_args]
    res = subprocess.run(cmd, cwd=REPO, capture_output=True, text=True, timeout=timeout, env={**os.environ, **(env or {})})
    tail = (res.stdout[-6000:] + "\n" + res.stderr[-3000:])
    log_dir = os.path.join(REPO, "gpurun_out")
    os.makedirs(log_dir, exist_ok=True)
    with open(os.path.join(log_dir, f"validate_parallelism_w{world}.log"), "a") as f:
        f.write(res.stdout)
    assert res.returncode == 0, tail


@pytest.mark.parametrize("world", [2, 4, 8])
def test_model_gradients_match_single_gpu_over_meshes(world):
    if _gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    if world != max(w for w in (2, 4, 8) if w <= _gpus()) and os.environ.get("D9D_TEST_ALL_WORLDS", "0") != "1":
        pytest.skip("only the largest world size the box offers runs by default (D9D_TEST_ALL_WORLDS=1 for all)")
    _torchrun(world, ["benchmarks/validate_parallelism_gpu.py"])


def test_fsdp_collectives_over_peer_memory():
    """FSDP / HSDP meshes with FSDP's all-gather / reduce-scatter replaced by pulls over NVLink peer memory
    (``D9D_FSDP_COMM=peer``, ``module/parallelism/api/_peer_memory_fsdp.py``): same gradient check as the NCCL run."""
    world = max((w for w in (2, 4, 8) if w <= _gpus()), default=0)
    if world < 2:
        pytest.skip("needs >= 2 GPUs")
    meshes = {2: ["dps2"], 4: ["dps4", "dpr2_dps2"], 8: ["dps8", "dpr2_dps4"]}[world]
    _torchrun(world, ["benchmarks/validate_parallelism_gpu.py", "--skip-attention", "--meshes", *meshes], env={"D9D_FSDP_COMM": "peer"})


def _pp_gpu_worker(rank, world, cases):
    from tests.test_pipelining import _pp_worker

    torch.cuda.set_device(rank)
    _pp_worker(rank, world, cases)


def test_pipeline_schedules_end_to_end_over_nccl():
    """All schedules on 4 (or 2) pipeline ranks with NCCL send / recv between the stages' GPUs."""
    from tests.dist_utils import run_distributed
    from tests.test_pipelining import _PP_CASES

    world = 4 if _gpus() >= 4 else 2
    if _gpus() < world:
        pytest.skip("needs >= 2 GPUs")
    cases = _PP_CASES if world == 4 else [c for c in _PP_CASES if "_v" not in c[0]]
    run_distributed(_pp_gpu_worker, world, cases)

#!/usr/bin/env bash
# Run a subset of the GPU kernel tests under NVIDIA compute-sanitizer (needs an H100; one GPU).
#
#   tools/sanitize.sh memcheck            # out-of-bounds / misaligned accesses, leaks
#   tools/sanitize.sh racecheck           # shared-memory hazards between warps (TMA / mbarrier protocols)
#   tools/sanitize.sh synccheck           # invalid barrier usage
#   tools/sanitize.sh initcheck           # reads of uninitialised global memory
#
# Optional second argument: a pytest -k expression (default: the GEMM, norm and MoE kernel tests; the full suite takes
# hours under the sanitizer).  Reports go to gpurun_out/sanitizer-<tool>.log so that `gpurun` brings them back.
set -euo pipefail
tool="${1:-memcheck}"
select="${2:-gemm or rms or moe or router or silu}"
mkdir -p gpurun_out
export D9D_NATIVE_ATTENTION=1 PYTORCH_NO_CUDA_MEMORY_CACHING=1   # exact allocation bounds for memcheck
exec compute-sanitizer --tool "$tool" --error-exitcode 1 --launch-timeout 0 --log-file "gpurun_out/sanitizer-$tool.log" \
    python -m pytest tests/test_ops_gpu.py -x -q -m gpu -k "$select"

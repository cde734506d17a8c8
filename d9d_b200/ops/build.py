"""In-tree build of the native sm_90a (H100) extension.

* ``*.cu`` translation units are compiled with ``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` and do
  not include torch headers (seconds per file).
* ``bindings.cpp`` (TORCH_LIBRARY registration) is compiled with the host compiler against torch.
* The result is ``d9d_b200/ops/_lib/d9d_b200_ops.so`` – it lives in-tree so it travels with the repo snapshot to
  the GPU box.  A content hash of all sources + flags is stored next to it; ``load()`` only rebuilds when it
  changes.
"""

from __future__ import annotations

import hashlib
import json
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

_HERE = Path(__file__).resolve().parent
CSRC = _HERE / "csrc"
BUILD_DIR = _HERE / "_build"
LIB_DIR = _HERE / "_lib"
LIB_PATH = LIB_DIR / "d9d_b200_ops.so"
STAMP_PATH = LIB_DIR / "d9d_b200_ops.stamp.json"

NVCC_FLAGS = [
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-O3",
    "-std=c++17",
    "--use_fast_math",
    "-Xcompiler",
    "-fPIC",
    "--expt-relaxed-constexpr",
]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-Wno-deprecated-declarations"]


def _cuda_home() -> Path:
    for cand in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if cand and Path(cand, "bin", "nvcc").exists():
            return Path(cand)
    nvcc = shutil.which("nvcc")
    if nvcc:
        return Path(nvcc).resolve().parent.parent
    raise RuntimeError("d9d_b200: nvcc not found (set CUDA_HOME)")


def cuda_sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def cpp_sources() -> list[Path]:
    return sorted(CSRC.glob("*.cpp"))


def _headers() -> list[Path]:
    return sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")))


def source_hash() -> str:
    h = hashlib.sha256()
    for p in cuda_sources() + cpp_sources() + _headers():
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS + CXX_FLAGS).encode())
    try:
        import torch

        h.update(torch.__version__.encode())
    except Exception:  # pragma: no cover
        pass
    return h.hexdigest()


def is_up_to_date() -> bool:
    if not LIB_PATH.exists() or not STAMP_PATH.exists():
        return False
    try:
        return json.loads(STAMP_PATH.read_text())["hash"] == source_hash()
    except Exception:
        return False


def _obj_hash(src: Path, flags: list[str]) -> str:
    h = hashlib.sha256()
    h.update(src.read_bytes())
    for hd in _headers():
        h.update(hd.read_bytes())
    h.update(" ".join(flags).encode())
    return h.hexdigest()


def _compile_one(cmd: list[str], src: Path, obj: Path, flags: list[str], verbose: bool) -> None:
    stamp = obj.with_suffix(obj.suffix + ".hash")
    want = _obj_hash(src, flags)
    if obj.exists() and stamp.exists() and stamp.read_text() == want:
        return
    if verbose:
        print(f"[d9d_b200.build] compiling {src.name}", flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"compilation of {src} failed:\n{' '.join(cmd)}\n{res.stdout}\n{res.stderr}")
    stamp.write_text(want)


def build(verbose: bool = True, force: bool = False) -> Path:
    """Compile every CUDA/C++ source for sm_90a and link the extension. Returns the .so path."""
    import torch
    from torch.utils import cpp_extension

    if not force and is_up_to_date():
        return LIB_PATH

    cuda_home = _cuda_home()
    nvcc = str(cuda_home / "bin" / "nvcc")
    cxx = os.environ.get("CXX", "g++")
    BUILD_DIR.mkdir(exist_ok=True)
    LIB_DIR.mkdir(exist_ok=True)

    jobs = []
    objs = []
    for src in cuda_sources():
        obj = BUILD_DIR / (src.stem + ".cu.o")
        objs.append(obj)
        flags = NVCC_FLAGS + [f"-I{CSRC}"]
        jobs.append(([nvcc, *flags, "-c", str(src), "-o", str(obj)], src, obj, flags))

    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    inc = [f"-I{p}" for p in cpp_extension.include_paths()] + [f"-I{cuda_home / 'include'}", f"-I{CSRC}"]
    import sysconfig

    inc.append(f"-I{sysconfig.get_paths()['include']}")
    for src in cpp_sources():
        obj = BUILD_DIR / (src.stem + ".cpp.o")
        objs.append(obj)
        flags = CXX_FLAGS + inc + [f"-D_GLIBCXX_USE_CXX11_ABI={abi}", "-DTORCH_API_INCLUDE_EXTENSION_H"]
        jobs.append(([cxx, *flags, "-c", str(src), "-o", str(obj)], src, obj, flags))

    workers = max(1, min(len(jobs), (os.cpu_count() or 4)))
    with ThreadPoolExecutor(workers) as pool:
        futs = [pool.submit(_compile_one, *job, verbose) for job in jobs]
        for f in futs:
            f.result()

    torch_lib = Path(torch.__file__).parent / "lib"
    link = [
        cxx,
        "-shared",
        "-o",
        str(LIB_PATH),
        *map(str, objs),
        f"-L{torch_lib}",
        f"-L{cuda_home / 'lib64'}",
        "-lc10",
        "-lc10_cuda",
        "-ltorch_cpu",
        "-ltorch_cuda",
        "-ltorch",
        "-lcudart",
        f"-Wl,-rpath,{torch_lib}",
        f"-Wl,-rpath,{cuda_home / 'lib64'}",
    ]
    if verbose:
        print("[d9d_b200.build] linking", LIB_PATH.name, flush=True)
    res = subprocess.run(link, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{' '.join(link)}\n{res.stdout}\n{res.stderr}")
    STAMP_PATH.write_text(json.dumps({"hash": source_hash()}))
    return LIB_PATH


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv)
    print(LIB_PATH)

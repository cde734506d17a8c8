"""Register, stack and spill report of every bf16 and fp8 wgmma GEMM instance, or of the flash attention kernels (no GPU needed).

Compiles the GEMM translation units (or ``flash_attn.cu`` with ``--units attention``) for sm_90a with ``-Xptxas -v`` (the
flags of ``d9d_b200/ops/build.py``) and prints one row per kernel instance: registers, stack frame, spill stores / loads,
and the wgmma serialisation advisories C7512 / C7515 ptxas raised for it.  Attention instances are named fwd / dkv / dq
with their (qk, v) head dims.

Exits non-zero when a GEMM instance spills or is serialised, so it doubles as a check.  For attention it fails on
serialised wgmma and on spills of the forward and dQ kernels; the dK/dV kernels' spill is reported (an open item at head
dim 128, see NOTES.md).

    python benchmarks/ptxas_gemm_report.py [--units gemm|attention] [--jobs N] [--all-kernels]
"""

from __future__ import annotations

import argparse
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from d9d_b200.ops import build as ops_build  # noqa: E402

UNITS = ["gemm_dense.cu", "gemm_dense_pair.cu", "gemm_grouped.cu", "gemm_ce.cu", "gemm_comm_fwd.cu", "gemm_comm_wgrad.cu",
         "gemm_fp8.cu"]
MODES = {0: "DENSE", 1: "GROUPED_M", 2: "GROUPED_K"}
EPIS = {0: "BF16", 1: "F32", 2: "F32_ACC", 3: "BF16_ACC", 4: "CE_LSE", 5: "CE_DLOGITS", 6: "CE_LSE_SUM",
        7: "CE_DLOGITS_REG"}
COMMS = {0: "-", 1: "AG_A", 2: "RS_D", 3: "AG_KA", 4: "AG_KB", 5: "WAIT_A"}
_GEMM = re.compile(r"gemm_kernelILi(\d+)ELi(\d+)ELb([01])ELb([01])ELi(\d+)ELi(\d+)ELi(\d+)EE")
_FP8 = re.compile(r"gemm_fp8_kernelILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)EE")
SCALINGS = {0: "ROWCOL", 1: "MX", 2: "BLOCK"}
_ATTN_FWD = re.compile(r"flash_attn_fwd_kernelILi(\d+)ELi(\d+)EE")
_ATTN_BWD = re.compile(r"flash_attn_bwd_kernelILi(\d+)ELi(\d+)ELb([01])EE")


def _name(mangled: str) -> str | None:
    m = _FP8.search(mangled)
    if m is not None:
        bn, scaling, mode, epi = (int(x) for x in m.groups())
        return f"fp8 {MODES[mode]:<9} BN {bn:<3} {SCALINGS[scaling]:<6} {EPIS[epi]}"
    m = _GEMM.search(mangled)
    if m is None:
        return None
    mode, bn, a_mn, b_mn, epi, comm, ctas = (int(x) for x in m.groups())
    layout = ("MN" if a_mn else "K") + "/" + ("MN" if b_mn else "K")
    return f"{MODES[mode]:<9} BN {bn:<3} A/B {layout:<5} {EPIS[epi]:<14} comm {COMMS[comm]:<6} ctas {ctas}"


def _attn_name(mangled: str) -> str | None:
    m = _ATTN_FWD.search(mangled)
    if m is not None:
        return f"fwd (DQK, DV) = ({m.group(1)}, {m.group(2)})"
    m = _ATTN_BWD.search(mangled)
    if m is not None:
        return f"{'dkv' if m.group(3) == '1' else 'dq':<3} (DQK, DV) = ({m.group(1)}, {m.group(2)})"
    return None


def _flagged(r: dict, name: str | None, units: str) -> bool:
    """GEMM: any spill or serialised wgmma.  Attention: serialised wgmma, or a spill outside the dK/dV kernels."""
    if name is None:
        return False
    if r["adv"] & {"C7512", "C7515"}:
        return True
    spills = bool(r["st"] or r["ld"])
    return spills and (units == "gemm" or not name.startswith("dkv"))


def compile_unit(unit: str, out_dir: Path) -> str:
    flags = [f for f in ops_build.NVCC_FLAGS if f not in ("-Xcompiler", "-fPIC")]
    nvcc = str(ops_build._cuda_home() / "bin" / "nvcc")
    cmd = [nvcc, *flags, f"-I{ops_build.CSRC}", "-Xptxas", "-v", "-cubin", "-o", str(out_dir / (unit + ".cubin")),
           str(ops_build.CSRC / unit)]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"compilation of {unit} failed:\n{res.stdout}\n{res.stderr}")
    return res.stdout + res.stderr


def parse(log: str) -> list[dict]:
    """One record per compiled entry function: registers, stack, spills and the advisories that name it."""
    rows: dict[str, dict] = {}
    cur = None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = rows.setdefault(m.group(1), {"fn": m.group(1), "regs": 0, "stack": 0, "st": 0, "ld": 0, "adv": set()})
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            cur["stack"], cur["st"], cur["ld"] = (int(x) for x in m.groups())
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and cur is not None:
            cur["regs"] = int(m.group(1))
            continue
        m = re.search(r"\((C75\d\d)\)", line)
        if m:
            # the advisory names its function; fall back to the one being compiled
            fn = re.search(r"'(_Z[^']+)'", line)
            target = rows.get(fn.group(1)) if fn else cur
            if target is not None:
                target["adv"].add(m.group(1))
    return list(rows.values())


def main() -> int:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--units", default="gemm", choices=["gemm", "attention"], help="GEMM translation units or flash_attn.cu")
    ap.add_argument("--jobs", type=int, default=len(UNITS))
    ap.add_argument("--all-kernels", action="store_true", help="also list the other kernels of these units")
    args = ap.parse_args()
    units, namer = (UNITS, _name) if args.units == "gemm" else (["flash_attn.cu"], _attn_name)
    with tempfile.TemporaryDirectory(prefix="d9d_ptxas_") as tmp:
        with ThreadPoolExecutor(max(1, args.jobs)) as pool:
            logs = list(pool.map(lambda u: compile_unit(u, Path(tmp)), units))
    bad = 0
    n = 0
    print(f"{'unit':<20} {'instance':<62} {'regs':>4} {'stack':>6} {'spill st':>9} {'spill ld':>9}  advisories")
    for unit, log in zip(units, logs):
        for r in sorted(parse(log), key=lambda r: namer(r["fn"]) or r["fn"]):
            name = namer(r["fn"])
            if name is None and not args.all_kernels:
                continue
            n += 1
            adv = ",".join(sorted(r["adv"])) or "-"
            flag = _flagged(r, name, args.units)
            bad += bool(flag)
            print(f"{unit:<20} {name or r['fn']:<62} {r['regs']:>4} {r['stack']:>6} {r['st']:>9} {r['ld']:>9}  {adv}"
                  + ("   <-- spills / serialised" if flag else ""))
    print(f"{n} instances, {bad} with spills or serialised wgmma")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())

"""In-tree build of the native pieces.

* ``learningorchestra_b200/lib/libloexec.so`` — the product: sm_90a kernels + C ABI
  (``include/loexec.h``), compiled with nvcc (cross-compiles without a GPU).
* ``oracle/_build/liboracle.so`` — the CPU oracle's C restatement (test infrastructure,
  gcc + OpenMP).  Building the checker is not using it: nothing in this package loads it.

Run ``python -m learningorchestra_b200.build`` or call :func:`build_all`.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "learningorchestra_b200" / "csrc"
LIB_DIR = ROOT / "learningorchestra_b200" / "lib"
LIB_PATH = LIB_DIR / "libloexec.so"
ORACLE_SRC = ROOT / "oracle" / "bsem.c"
ORACLE_LIB = ROOT / "oracle" / "_build" / "liboracle.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-O2,-Wall",
    "-shared", "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; libloexec cannot be built (there is no CPU fallback)")


def _stale(target: Path, sources: list[Path]) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(s.stat().st_mtime > t for s in sources)


def build_native(force: bool = False, verbose: bool = False) -> Path:
    sources = [CSRC / "loexec.cu", CSRC / "group.inc", CSRC / "kernels.cuh", CSRC / "naive_bayes.cuh", CSRC / "parse_number.cuh", CSRC / "pow5_table.inc",
               CSRC / "format_number.cuh", CSRC / "ryu_pow5.inc", CSRC / "ryu_pow5_inv.inc", CSRC / "csv.inc", CSRC / "csv_reader.cuh",
               ROOT / "include" / "loexec.h"]
    if not force and not _stale(LIB_PATH, sources):
        return LIB_PATH
    LIB_DIR.mkdir(parents=True, exist_ok=True)
    cmd = [_nvcc(), *NVCC_FLAGS, "-I", str(ROOT / "include"), "-I", str(CSRC)]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    tmp = LIB_PATH.with_suffix(f".so.tmp{os.getpid()}")
    cmd += ["-o", str(tmp), str(CSRC / "loexec.cu")]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        tmp.unlink(missing_ok=True)
        raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{proc.stdout}\n{proc.stderr}")
    os.replace(tmp, LIB_PATH)               # atomic: a concurrent loader sees the old or the new file, never half
    if verbose:
        print(proc.stderr, file=sys.stderr)
    return LIB_PATH


def build_oracle(force: bool = False) -> Path:
    if not force and not _stale(ORACLE_LIB, [ORACLE_SRC]):
        return ORACLE_LIB
    ORACLE_LIB.parent.mkdir(parents=True, exist_ok=True)
    # -ffp-contract=off: the oracle's fp32/fp64 arithmetic must be one IEEE operation per
    # C operator (no FMA fusion), -fno-fast-math is the default and stays.
    tmp = ORACLE_LIB.with_suffix(f".so.tmp{os.getpid()}")
    cmd = ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off",
           "-Wall", "-o", str(tmp), str(ORACLE_SRC), "-lm"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        tmp.unlink(missing_ok=True)
        raise RuntimeError(f"gcc failed:\n{' '.join(cmd)}\n{proc.stdout}\n{proc.stderr}")
    os.replace(tmp, ORACLE_LIB)
    return ORACLE_LIB


def build_all(force: bool = False, verbose: bool = False) -> None:
    build_native(force=force, verbose=verbose)
    build_oracle(force=force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(LIB_PATH)
    print(ORACLE_LIB)

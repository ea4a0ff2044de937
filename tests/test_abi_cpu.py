"""CPU: libloexec.so builds for sm_90a, loads, and exports exactly what include/loexec.h declares.
No compute calls are made here (there is no GPU and no CPU fallback)."""
import ctypes
import re
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
HEADER = ROOT / "include" / "loexec.h"


def _declared_functions():
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(lo_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported_and_bound(built):
    from learningorchestra_b200 import _native
    lib = _native.load()
    declared = _declared_functions()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in loexec.h but not exported by libloexec.so"
    assert sorted(_native.SIGNATURES) == declared, "ctypes SIGNATURES out of sync with include/loexec.h"
    assert lib.lo_abi_version() == _native.LO_ABI_VERSION


def test_library_is_sm90a_native_code(built):
    from learningorchestra_b200 import _native
    out = subprocess.run(["cuobjdump", "-lelf", str(_native.LIB_PATH)], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out
    full = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True).stdout
    sass = full.split("Function : _ZN2lo19k_project_cast_histILi1ELb1ELb1ELb1EEE")[1].split("Function :")[0]
    assert "LDG.E.NA.128" in sass                               # 128-bit streaming loads
    assert "STS.U8" in sass and "LDS.U8" in sass                # private byte-counter histogram, no ATOMS
    assert "ATOMS" not in sass
    assert "RED.E.ADD.64.STRONG.SYS" in sass or "REDG.E.ADD.64.STRONG.SYS" in sass    # in-kernel merge: pushes at system scope


def test_lane_slot_kernels_issue_one_shared_atomic_per_element(built):
    """The shipped byte-histogram kernel is the lane-slot form: per 64 input bytes 64 PRMT (the counter address straight from
    the input word) and 64 shared-memory atomics with the reserved-smem base in the immediate, 128-bit streaming loads, a
    RED.64 flush; the wide-bin kernel counts with shared atomics too and streams with 128-bit loads."""
    from learningorchestra_b200 import _native
    sass = subprocess.run(["cuobjdump", "-sass", str(_native.LIB_PATH)], capture_output=True, text=True).stdout
    lanes = sass.split("Function : _ZN2lo20k_hist_u8_cols_lanesILb1EEE")[1].split("Function :")[0]
    atoms = [l for l in lanes.splitlines() if "ATOMS" in l]
    assert len(atoms) >= 128 and all("+0x400]" in l for l in atoms if "POPC.INC" in l)
    assert lanes.count("PRMT") >= 128 and "LDG.E.NA.128" in lanes or "LDG.E.128" in lanes
    assert "LDS.U8" not in lanes and "STS.U8" not in lanes
    assert "REDG.E.ADD.64.STRONG.GPU" in lanes or "RED.E.ADD.64.STRONG.GPU" in lanes
    bins = sass.split("Function : _ZN2lo24k_project_cast_hist_binsILi1ELb1EEE")[1].split("Function :")[0]
    assert "ATOMS" in bins and "F2F.F32.F64" in bins and "LDG.E.NA.128" in bins


def test_no_gpu_means_loud_failure_not_fallback(built):
    """On a CPU-only host every entry that would compute must fail with LO_ERR_NO_DEVICE."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible")
    from learningorchestra_b200 import _native
    from learningorchestra_b200.engine import Engine
    with pytest.raises(_native.LoexecError) as e:
        Engine(0)
    assert e.value.code == _native.LO_ERR_NO_DEVICE
    assert "no CPU fallback" in e.value.message or "no CUDA device" in e.value.message
    n = ctypes.c_int(-1)
    rc = _native.load().lo_device_count(ctypes.byref(n))
    assert rc in (_native.LO_OK, _native.LO_ERR_NO_DEVICE) and n.value == 0


def test_package_never_imports_the_oracle():
    """The product must not import, link or execute anything under oracle/."""
    pkg = ROOT / "learningorchestra_b200"
    for path in pkg.rglob("*"):
        if path.suffix in (".py", ".cu", ".cuh", ".h") and path.name != "build.py":
            text = path.read_text()
            assert "oracle" not in text.lower() or all(
                "import" not in line and "dlopen" not in line and "CDLL" not in line
                for line in text.splitlines() if "oracle" in line.lower()), path


def _build_c_consumer(out_dir: Path) -> Path:
    """Compile tests/native/abi_smoke.c into ``out_dir`` (a temporary directory: the checkout may be read-only)."""
    from learningorchestra_b200 import _native
    exe = out_dir / "abi_smoke"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-O1", "-I", str(ROOT / "include"),
                    str(ROOT / "tests" / "native" / "abi_smoke.c"), "-o", str(exe),
                    "-L", str(_native.LIB_PATH.parent), "-lloexec", f"-Wl,-rpath,{_native.LIB_PATH.parent}"], check=True)
    return exe


def test_plain_c_program_links_against_the_abi(built, tmp_path):
    """include/loexec.h is plain C99 and the .so links without any C++ / CUDA / torch on the consumer side."""
    import torch
    exe = _build_c_consumer(tmp_path)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    if torch.cuda.is_available():
        assert out.returncode == 0, out.stderr
    else:
        assert out.returncode == 3 and "no CUDA device" in out.stderr      # loud, documented failure


def test_ctypes_mirror_matches_the_header_constants_and_struct_layouts(tmp_path):
    """Every ``#define LO_*`` integer of include/loexec.h that ``_native`` mirrors has the same value there, and the two
    structs that cross the boundary by pointer have the same size and field offsets (compiled with gcc, no library needed)."""
    from learningorchestra_b200 import _native
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    names = [n for n in re.findall(r"#define\s+(LO_[A-Z0-9_]+)\s+-?\d", text) if hasattr(_native, n)]
    assert len(names) >= 30 and "LO_ABI_VERSION" in names and "LO_MAX_BINS" in names
    src = tmp_path / "layout.c"
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "loexec.h"', 'int main(void) {']
    lines += [f'    printf("{n} %lld\\n", (long long)({n}));' for n in names]
    for struct, fields in (("lo_host_timing", ["total_ms", "h2d_bytes", "d2h_bytes", "launches", "kernel_ms"]),
                           ("lo_hist_spec", ["nbins", "flags", "lo", "hi"])):
        lines.append(f'    printf("sizeof.{struct} %zu\\n", sizeof({struct}));')
        lines += [f'    printf("offsetof.{struct}.{f} %zu\\n", offsetof({struct}, {f}));' for f in fields]
    lines += ['    return 0;', '}']
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", str(ROOT / "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    for n in names:
        assert int(got[n]) == getattr(_native, n), n
    for struct, mirror in (("lo_host_timing", _native.HostTiming), ("lo_hist_spec", _native.HistSpec)):
        assert int(got[f"sizeof.{struct}"]) == ctypes.sizeof(mirror), struct
        for f, _t in mirror._fields_:
            assert int(got[f"offsetof.{struct}.{f}"]) == getattr(mirror, f).offset, f"{struct}.{f}"


def test_output_column_array_has_one_entry_per_input_column():
    """The *project_cast_hist_host calls read k out_cols entries: a short ``out`` list leaves NULL entries, which the
    library rejects ("out_cols[j] is NULL"); a longer one is refused before any call."""
    import numpy as np
    from learningorchestra_b200.engine import _out_cols
    o = np.zeros(4, np.float32)
    arr = _out_cols([o], 3, 4)
    assert len(arr) == 3 and arr[0] == o.ctypes.data and arr[1] is None and arr[2] is None
    with pytest.raises(IndexError):
        _out_cols([o, o], 1, 4)

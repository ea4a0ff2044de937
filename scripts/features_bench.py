"""Time ``Engine.assemble_rows`` (lo_assemble_rows, the feature matrix of ``DeviceFrame.features``) against the torch
composition a consumer would otherwise write, ``torch.stack(cols, 1).to(torch.float32)``, on the same resident columns.

Workloads: 10 M rows x (16 f64 slabs + 4 int32 code columns) -> f32, the shape of a tabular dataset's frame, and
100 M rows x 32 f64 slabs -> f32, the size of the project's headline bench table.  The two are alternated in one
process after warm-ups; each iteration's outputs are compared.  Times: the library's own kernel time (CUDA events
around its kernels, lo_host_timing.kernel_ms), the whole call (allocation of the result included), and torch's
composition between CUDA events.  Bytes are algorithmic: every source byte read once plus the matrix written; the
skip mode reads the sources twice (validity pass, then write pass), reported beside it.

    python scripts/features_bench.py [--iters 20] [--warmup 3] [--small-only]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

PEAK_TBS = 3.35          # H100 SXM data-sheet HBM3 bandwidth


def card():
    import torch
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                          "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(), "nvidia_smi": out.stdout.strip()}


def run(eng, n, nf, ncodes, iters, warmup):
    import numpy as np
    import torch
    from learningorchestra_b200 import _native as N
    dev = f"cuda:{eng.device}"
    slabs = eng.table("f64", n, nf).fill_synthetic(N.LO_SYNTH_UNIFORM, 20261017)
    codes = [torch.randint(0, 1000, (n,), dtype=torch.int32, device=dev) for _ in range(ncodes)]
    ctabs = [eng.wrap("i32", n, 1, c.data_ptr(), 4 * n, keepalive=c) for c in codes]
    sources = [(slabs, j) for j in range(nf)] + [(t, 0) for t in ctabs]
    cols = [torch.as_tensor(slabs.column_view(j), device=dev) for j in range(nf)] + codes
    eng.sync()

    def ours(mode="error"):
        t = {}
        w0 = time.perf_counter()
        res = eng.assemble_rows(sources, dtype="float32", handle_invalid=mode, timing=t)
        return res, t["kernel_ms"], (time.perf_counter() - w0) * 1e3

    def theirs():
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = torch.stack(cols, 1).to(torch.float32)
        b.record()
        b.synchronize()
        return out, a.elapsed_time(b)

    k_ms, call_ms, torch_ms, equal = [], [], [], True
    for i in range(warmup + iters):
        res, kms, cms = ours()
        ref, tms = theirs()
        equal = equal and bool(torch.equal(torch.as_tensor(res.matrix(), device=dev), ref))
        res.free()
        del ref
        torch.cuda.empty_cache()
        if i >= warmup:
            k_ms.append(kms), call_ms.append(cms), torch_ms.append(tms)
    skip_ms = []
    for i in range(warmup + max(iters // 4, 3)):
        res, kms, _ = ours("skip")
        assert res.nkept == n
        res.free()
        if i >= warmup:
            skip_ms.append(kms)
    src_bytes = n * (8 * nf + 4 * ncodes)
    alg = src_bytes + n * 4 * (nf + ncodes)
    med = lambda v: float(np.median(v))
    r = {"rows": n, "f64_slabs": nf, "code_columns": ncodes, "dtype": "float32", "mode": "error", "equal": equal,
         "kernel_ms": med(k_ms), "kernel_ms_min": min(k_ms), "kernel_ms_max": max(k_ms), "call_ms": med(call_ms),
         "torch_ms": med(torch_ms), "torch_ms_min": min(torch_ms), "torch_ms_max": max(torch_ms),
         "algorithmic_bytes": alg, "kernel_tb_s": alg / med(k_ms) / 1e9, "kernel_share_of_peak": alg / med(k_ms) / 1e9 / PEAK_TBS,
         "torch_share_of_peak": alg / med(torch_ms) / 1e9 / PEAK_TBS, "speedup_vs_torch": med(torch_ms) / med(k_ms),
         "skip_kernel_ms": med(skip_ms), "skip_actual_bytes": 2 * src_bytes + n * 4 * (nf + ncodes) + n // 8 + 8 * n,
         "iters": iters}
    r["skip_share_of_peak"] = r["skip_actual_bytes"] / r["skip_kernel_ms"] / 1e9 / PEAK_TBS
    for t in ctabs:
        t.free()
    slabs.free()
    del cols, codes
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--small-only", action="store_true")
    a = ap.parse_args()
    import torch
    from learningorchestra_b200.build import build_all
    from learningorchestra_b200.engine import Engine
    build_all()
    torch.cuda.init()
    info = card()
    with Engine(0) as eng:
        results = [run(eng, 10_000_000, 16, 4, a.iters, a.warmup)]
        if not a.small_only:
            results.append(run(eng, 100_000_000, 32, 0, a.iters, a.warmup))
    for r in results:
        print(json.dumps({**info, **r}))
    print(json.dumps({**card(), "note": "card read again after the runs"}))


if __name__ == "__main__":
    main()

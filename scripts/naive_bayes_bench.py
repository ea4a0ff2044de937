"""Times NaiveBayes fit, transform and evaluate on the feature matrix in HBM (lo_nb_fit / lo_nb_predict) against a torch
composition on the same device, alternated in one process, and checks that the two agree.  Prints the card and its power
limit beside the figures.  Kernel time = the call's kernels between CUDA events (lo_host_timing.kernel_ms); call time =
CUDA events around the whole Python call.  Algorithmic bytes: fit and evaluate read n (4k + 4), transform reads n 4k and writes
n 8 (C + 1).  Workloads: 10 M x 20 f32 with C = 2 (Titanic-wide) and 100 M x 32 f32 with C = 10 (DESIGN.md §3.6.2)."""
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from learningorchestra_b200.engine import AssembledRows, Engine  # noqa: E402
from learningorchestra_b200.classifier import model_arrays  # noqa: E402

PEAK = 3.35e12


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        ev[0].record()
        fn()
        ev[1].record()
        torch.cuda.synchronize()
        ms.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(ms))


def run(eng, n, k, nclasses, reps):
    g = torch.Generator(device="cuda").manual_seed(n + k)
    y = torch.randint(0, nclasses, (n,), device="cuda", generator=g).to(torch.float32)
    rates = torch.rand((nclasses, k), device="cuda", generator=g) * 5 + 0.5
    x = torch.poisson(rates[y.long()], generator=g).to(torch.float32)
    xt = eng.wrap("f32", n * k, 1, x.data_ptr(), n * k * 4, keepalive=x)
    yt = eng.wrap("f32", n, 1, y.data_ptr(), n * 4, keepalive=y)
    part = AssembledRows(xt, yt, None, k, n)
    classes = eng.nb_labels(part)
    sums, counts = eng.nb_fit(part, classes)
    pi, theta = model_arrays(sums, counts, 1.0)
    pi_t, th_t = torch.tensor(pi, device="cuda"), torch.tensor(theta, device="cuda")

    def t_fit():
        s = torch.zeros((nclasses, k), dtype=torch.float64, device="cuda").index_add_(0, y.long(), x.double())
        return s, torch.bincount(y.long(), minlength=nclasses)

    def t_transform():
        r = x.double() @ th_t.T + pi_t
        p = torch.softmax(r, 1)
        return p, p.argmax(1)

    def t_eval():
        pred = (x.double() @ th_t.T + pi_t).argmax(1)
        return torch.bincount(y.long() * nclasses + pred, minlength=nclasses * nclasses)

    ts, tc = t_fit()
    assert np.allclose(ts.cpu().numpy(), sums, rtol=1e-12) and np.array_equal(tc.cpu().numpy(), counts)
    conf = eng.nb_predict(part, pi, theta, labels=classes)
    tconf = t_eval().cpu().numpy().reshape(nclasses, nclasses)
    agree_eval = int(np.abs(conf - tconf).sum())
    out = eng.nb_predict(part, pi, theta)
    agree_pred = int((torch.as_tensor(out.prediction(), device="cuda") != t_transform()[1].double()).sum())
    out.free()
    res = {"n": n, "k": k, "C": nclasses, "eval_pairs_differing": agree_eval, "predictions_differing": agree_pred}
    kernel_ms = []

    def timing():
        tm = {}
        kernel_ms.append(tm)
        return tm

    for name, ours, theirs, nbytes in (
            ("fit", lambda: eng.nb_fit(part, classes, timing=timing()), t_fit, n * (4 * k + 4)),
            ("transform", lambda: eng.nb_predict(part, pi, theta, timing=timing()).free(), t_transform,
             n * 4 * k + n * 8 * (nclasses + 1)),
            ("evaluate", lambda: eng.nb_predict(part, pi, theta, labels=classes, timing=timing()), t_eval,
             n * (4 * k + 4))):
        a, b = [], []
        kernel_ms.clear()
        for _ in range(3):                     # alternate the two in one process
            a.append(timed(ours, reps))
            b.append(timed(theirs, reps))
        ms, kms = min(a), float(np.median([t["kernel_ms"] for t in kernel_ms]))
        res[name] = {"kernel_ms": round(kms, 3), "call_ms": round(ms, 3), "torch_ms": round(min(b), 3), "bytes": nbytes,
                     "kernel_share_of_3.35TBps_peak": round(nbytes / (kms * 1e-3) / PEAK, 3),
                     "call_share_of_3.35TBps_peak": round(nbytes / (ms * 1e-3) / PEAK, 3)}
    return res


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    eng = Engine(0)
    results = [run(eng, 10_000_000, 20, 2, reps), run(eng, 100_000_000, 32, 10, reps)]
    print(json.dumps({"gpu": q, "results": results}))


if __name__ == "__main__":
    main()
